"""Whole-network optimizer step: one kernel launch per training step.

The reference launches one weights_update + one bias_update kernel per layer
(/root/reference/nn_units.py:560-642, cuda/gradient_descent_common.cu) and, when
distributed, ships every layer's weights through the master
(/root/reference/nn_units.py:644-694). Here every GD unit only *produces* its local
gradient (split-K partials of the wgmma wgrad kernels, column-sum partials for the
bias); a ``FusedStep`` attached to the workflow collects the parameter tensors into a
descriptor table in HBM and, right after the last GD unit of the backward chain, launches
``csrc/update.cu::multi_update_k`` once: cross-GPU reduction over NVLink peer pointers +
split-K reduction + L1/L2/ortho regularisation + accumulation + momentum + apply + bf16
operand shadows for *all* tensors, with a single cross-GPU flag barrier per step.

Deferring the updates to the end of the chain is numerically identical to the reference
order because every layer's err_input is computed from pre-update weights in both.
"""
from __future__ import annotations

import torch

from ..kernels import api


def _desc_key(desc):
    """What the packed table holds of an ``api.UpdateDesc``: buffer addresses and the scalars."""
    return tuple(v.data_ptr() if isinstance(v, torch.Tensor) else v for v in desc)


class _Entry(object):
    __slots__ = ("unit", "is_bias", "desc", "touched")


class FusedStep(object):
    def __init__(self, device, dp=None):
        self.device = device
        self.dp = dp
        self.entries = []
        self.index = {}
        self.table = None
        self.total_tiles = 0
        self.has_ortho = False
        self.dirty = True
        self.enabled = []
        self.tables = []
        self.chunks = []
        self.red_ptrs = []
        self.red_numel = 0
        self.gridsync = torch.zeros(2, dtype=torch.int32, device=device.torch_device)
        self.flag_ptrs, self.epoch_ptr = [], 0
        self.launches = 0
        self.sync = []            # per chunk: (flag ptrs per rank, local epoch ptr)
        self.sum_ptrs, self.mc_red, self.mc_sum = [], 0, 0
        self.algo = 0
        self.algo_name = "single"
        self.max_blocks = 0       # > 0 only in fake-peer tests (several "ranks" share one GPU)

    # -- wiring ------------------------------------------------------------------------------
    @classmethod
    def attach(cls, workflow, dp=None):
        """Defer the updates of every CUDA GD unit of ``workflow`` and flush them after the
        last unit of the backward chain."""
        from .nn_units import GradientDescentBase
        chain = [u for u in reversed(workflow.gds) if u is not None]
        if not chain or not all(getattr(u, "on_cuda", False) for u in chain):
            return None
        fs = cls(workflow.device, dp)
        shared = cls.units_sharing_weights(chain)
        for u in chain:
            if isinstance(u, GradientDescentBase) and u.weights:
                # Tied weights (GDDeconv + the GD unit of its Conv in the auto-encoders) would be
                # two entries of ONE launch updating the same tensor concurrently: those units
                # keep the immediate, stream-ordered per-tensor update - the reference's order
                # (/root/reference/gd_deconv.py:306-365 updates right away as well)
                u.step_ = None if id(u) in shared else fs
        last = chain[-1]
        inner = last._backend_run_

        def run_and_flush():
            inner()
            fs.flush()
        last.__dict__["_backend_run_"] = run_and_flush
        fs.last_unit = last
        return fs

    @staticmethod
    def units_sharing_weights(chain):
        """ids of the GD units whose ``weights`` (or ``bias``) Array is also updated by another
        unit of the chain."""
        owners = {}
        for u in chain:
            for name in ("weights", "bias"):
                arr = getattr(u, name, None)
                if arr is not None and arr:
                    owners.setdefault(id(arr), []).append(u)
        return {id(u) for us in owners.values() if len(us) > 1 for u in us}

    # -- registration (called by api._update in deferred mode) -----------------------------------
    def submit(self, unit, is_bias, desc):
        """Step ``desc`` (an ``api.UpdateDesc``, which also keeps its buffers alive) in the next
        flush."""
        key = (id(unit), bool(is_bias))
        e = self.index.get(key)
        if e is None:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("FusedStep: new tensor registered during graph capture")
            e = _Entry()
            e.unit, e.is_bias = unit, bool(is_bias)
            self.index[key] = e
            self.entries.append(e)
            e.desc = None
        if e.desc is None or _desc_key(e.desc) != _desc_key(desc):
            if e.desc is not None and torch.cuda.is_current_stream_capturing():
                raise RuntimeError("FusedStep: %s changed buffers during graph capture" % unit)
            self.dirty = True
        e.desc = desc
        e.touched = True

    def refresh_flags(self, unit):
        """Host-side hook (GD ``cuda_prepare``): flags are baked into the table."""
        for is_bias in (False, True):
            e = self.index.get((id(unit), is_bias))
            if e is not None and e.desc is not None:
                f = unit.update_flags(for_bias=is_bias)
                if e.desc.flags != f:
                    e.desc = e.desc._replace(flags=f)
                    self.dirty = True
        if self.dirty and self.table is not None and not torch.cuda.is_current_stream_capturing():
            self._upload()

    def _upload(self):
        """(Re)build the descriptor table(s); more than ``multi_update_max_tensors`` tensors
        are split over several launches."""
        ext = self.device.ext
        cap = int(ext.multi_update_max_tensors())
        descs = [e.desc for e in self.entries]
        enabled = [bool(e.touched) for e in self.entries]
        self.chunks = []
        red = 0
        for i in range(0, len(descs), cap):
            part = descs[i:i + cap]
            packed, tiles, red, ortho = ext.multi_update_table(part, enabled[i:i + cap], red)
            old = self.tables[len(self.chunks)] if len(self.chunks) < len(self.tables) else None
            if old is None or old.numel() != packed.numel():
                old = torch.empty(packed.numel(), dtype=torch.uint8,
                                  device=self.device.torch_device)
            old.copy_(packed)
            self.chunks.append((old, len(part), int(tiles), ortho))
        self.tables = [c[0] for c in self.chunks]
        self.table = self.tables[0] if self.tables else None
        symm = self.dp.symm if self.dp is not None else None
        if symm is not None:
            # every chunk (launch) of a step has its own flag / epoch arrays: the chunks' grids
            # differ in size, a shared per-block epoch would advance unevenly (ADVICE r1)
            while len(self.sync) < len(self.chunks):
                self.sync.append(symm.sync_state("fused_step_%d" % len(self.sync)))
        if symm is not None and red > self.red_numel:
            # one fp32 slot per parameter in symmetric memory: ranks publish their locally
            # reduced gradients here, peers read them over NVLink (collective allocation:
            # all ranks build identical tables in the same step)
            # double buffered: step parity selects the half, so no trailing barrier is needed
            self.red_ptrs, self.mc_red = symm.reduction_buffer(
                "fused_step_red", 2 * int(red), with_multicast=True)
            self.red_numel = int(red)
            self._pick_algo(symm, int(red))
        self.enabled = enabled
        self.dirty = False

    def _pick_algo(self, symm, numel):
        """ZNICZ_DP_ALGO: auto | oneshot (N peer loads per element) | twoshot (owner reduce +
        broadcast, NVLS multimem when the platform has multicast) | twoshot_peer (same without
        multimem) | nvls1 (every rank multimem.ld_reduce-s everything, one barrier)."""
        import os
        name = os.environ.get("ZNICZ_DP_ALGO", "auto")
        have_mc = bool(self.mc_red)
        if name == "auto":
            # Small models are latency bound: ONE flag barrier per step, every rank reduces every
            # element itself (one multimem.ld_reduce per float4 with NVLS, N peer loads without).
            # Measured at 2 GPUs on the CIFAR net (0.36 MB of parameters, driver's 20-step run):
            # nvls1 0.2172 / oneshot 0.2165 / twoshot 0.2336 ms per step (1 GPU: 0.2042).
            # Large models are bandwidth bound: two-shot moves ~2 P floats per rank instead of
            # (N - 1) P and pays one more barrier.
            if numel >= (1 << 22):
                name = "twoshot" if have_mc else "twoshot_peer"
            else:
                name = "nvls1" if have_mc else "oneshot"
        if name == "twoshot" and not have_mc:
            name = "twoshot_peer"
        if name == "nvls1" and not have_mc:
            raise RuntimeError("ZNICZ_DP_ALGO=nvls1 needs multicast support")
        self.algo_name = name
        self.algo = {"oneshot": 0, "twoshot": 1, "twoshot_peer": 1, "nvls1": 2}[name]
        self.sum_ptrs, self.mc_sum = [], 0
        if self.algo == 1:
            self.sum_ptrs, self.mc_sum = symm.reduction_buffer(
                "fused_step_sum", 2 * numel, with_multicast=True)
            if name == "twoshot_peer" or not self.mc_sum:
                self.mc_sum = 0
        mc_red = self.mc_red if name in ("twoshot", "nvls1") else 0
        if name == "twoshot" and not self.mc_sum:
            mc_red = 0
            self.algo_name = "twoshot_peer"
        self.mc_red_used = mc_red

    # -- the launch ------------------------------------------------------------------------------
    def flush(self):
        if not self.entries:
            return
        touched = [bool(e.touched) for e in self.entries]
        if not any(touched):
            return
        if self.dirty or touched != self.enabled:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("FusedStep: table changed during graph capture")
            self._upload()
        api.join_side(self.device)      # wgrad kernels of the side-stream branch
        dp = self.dp
        if dp is not None and dp.world_size > 1 and dp.symm is None:
            # NCCL *baseline* mode (ZNICZ_DP_MODE=nccl): one library all-reduce per gradient
            # buffer, then the single-GPU update - what the fused peer-memory path is
            # measured against
            import torch.distributed as dist
            for e in self.entries:
                if e.touched:
                    dist.all_reduce(e.desc.grad, op=dist.ReduceOp.SUM)
        for ci, (table, n, tiles, ortho) in enumerate(self.chunks):
            flags, epoch = self.sync[ci] if self.sync else (self.flag_ptrs, self.epoch_ptr)
            self.device.ext.multi_update(table, n, tiles, ortho, flags, epoch,
                                         dp.rank if dp is not None else 0, self.gridsync,
                                         self.red_ptrs, self.red_numel if self.red_ptrs else 0, 1,
                                         self.sum_ptrs, getattr(self, "mc_red_used", 0),
                                         self.mc_sum, self.algo, self.max_blocks)
            api._launch()
        # fp8 layers: their e4m3 weight copies follow the updated fp32 masters (inside the
        # captured step graph)
        for e in self.entries:
            fwd = getattr(e.unit, "forward_unit", None)
            if e.touched and not e.is_bias and getattr(fwd, "weights_q_", None) is not None:
                api.requantize_weights(fwd)
        self.launches += 1
        for e in self.entries:
            e.touched = False
