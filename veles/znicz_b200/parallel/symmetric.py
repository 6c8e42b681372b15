"""Symmetric (peer-mapped) gradient buffers for the fused reduce+update kernel.

Each GD unit's fp32 gradient staging buffers (split-K wgrad partials, bias column-sum
partials) are allocated in CUDA symmetric memory (``torch.distributed._symmetric_memory``:
VMM allocations exported to every rank of the node and mapped over NVLink/NVSwitch). The
rendezvous is only *plumbing* — handle exchange — the data path is our own kernel
(``csrc/update.cu::fused_update_k<true>``), which reads every rank's gradient tile through
the peer pointers, reduces in fixed rank order, applies the SGD step and synchronises with
flag words that also live in symmetric memory. No NCCL call is issued per step.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

MAX_BLOCKS = 592     # csrc/update.cu::MU_MAX_PEER_BLOCKS


class _Buf(object):
    __slots__ = ("tensor", "handle", "ptrs", "flags", "flag_ptrs", "epoch", "blocks")


class SymmetricGradients(object):
    def __init__(self, dp, gds):
        import torch.distributed._symmetric_memory as symm_mem
        self.symm_mem = symm_mem
        self.dp = dp
        self.device = dp.device.torch_device
        self.group = dist.group.WORLD
        self._bufs = {}
        self.bytes = 0

    def _alloc(self, numel, dtype):
        t = self.symm_mem.empty(numel, dtype=dtype, device=self.device)
        h = self.symm_mem.rendezvous(t, self.group)
        return t, h

    def buffer(self, unit, name, shape):
        """fp32 tensor of ``shape`` in symmetric memory (allocated once per (unit, name);
        all ranks call this in the same order, outside graph capture)."""
        key = (id(unit), name)
        b = self._bufs.get(key)
        numel = 1
        for s in shape:
            numel *= int(s)
        if b is not None and b.tensor.numel() == numel:
            return b.tensor.view(*shape)
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("symmetric buffers must be created before graph capture")
        b = _Buf()
        b.tensor, b.handle = self._alloc(numel, torch.float32)
        b.tensor.zero_()
        b.ptrs = [int(p) for p in b.handle.buffer_ptrs]
        b.flags, fh = self._alloc(MAX_BLOCKS * 8, torch.int32)
        b.flags.zero_()
        b.flag_ptrs = [int(p) for p in fh.buffer_ptrs]
        b.epoch = torch.zeros(MAX_BLOCKS, dtype=torch.int32, device=self.device)
        b.blocks = 0
        self._bufs[key] = b
        self._bufs[b.tensor.data_ptr()] = b
        self.bytes += numel * 4
        torch.cuda.synchronize()
        dist.barrier()
        return b.tensor.view(*shape)

    def reduction_buffer(self, key, numel, with_multicast=False):
        """fp32 buffer of ``numel`` elements in symmetric memory → per-rank base pointers
        (and, with ``with_multicast``, the NVLS multicast address of the same memory: 0 when
        the platform has no multicast support)."""
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("symmetric buffers must be created before graph capture")
        t, h = self._alloc(numel, torch.float32)
        t.zero_()
        self._bufs[("red", key, numel)] = (t, h)
        self.bytes += numel * 4
        torch.cuda.synchronize()
        dist.barrier()
        ptrs = [int(p) for p in h.buffer_ptrs]
        if not with_multicast:
            return ptrs
        mc = 0
        try:
            mc = int(h.multicast_ptr or 0)
        except Exception:        # pragma: no cover - older torch / no NVSwitch
            mc = 0
        return ptrs, mc

    def sync_state(self, key):
        """(flag ptrs per rank, local epoch ptr) for a kernel that synchronises across
        ranks on its own (the whole-network FusedStep)."""
        b = self._bufs.get(("sync", key))
        if b is None:
            b = _Buf()
            b.flags, fh = self._alloc(MAX_BLOCKS * 8, torch.int32)
            b.flags.zero_()
            b.flag_ptrs = [int(p) for p in fh.buffer_ptrs]
            b.epoch = torch.zeros(MAX_BLOCKS, dtype=torch.int32, device=self.device)
            self._bufs[("sync", key)] = b
            torch.cuda.synchronize()
            dist.barrier()
        return b.flag_ptrs, b.epoch.data_ptr()

    def peers(self, unit, grad_buf):
        """(grad ptrs per rank, flag ptrs per rank, local epoch ptr, blocks)."""
        b = self._bufs[grad_buf.data_ptr()]
        return b.ptrs, b.flag_ptrs, b.epoch.data_ptr(), 0
