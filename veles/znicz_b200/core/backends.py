"""Devices: ``NumpyDevice`` (CPU oracle) and ``CUDADevice`` (one H100, sm_90a).

Fresh design for ``veles.backends``. There is exactly one accelerator backend:
no OpenCL, no multi-vendor dispatch (SURVEY "five facts" #2). A CUDADevice owns a
compute stream, a side stream for the fused all-reduce/update kernels, and a copy
stream for loader H2D double-buffering.
"""
from __future__ import annotations

import numpy

from .config import root


class Device(object):
    is_cuda = False
    backend_name = "none"

    def sync(self):
        pass

    def __repr__(self):
        return "<%s>" % type(self).__name__


def _restore_device(backend):
    """Unpickle hook: devices are process-local; re-acquire by backend name."""
    if backend == "cuda":
        try:
            return get_device("cuda")
        except Exception:
            return NumpyDevice()
    return NumpyDevice()


class NumpyDevice(Device):
    backend_name = "numpy"

    def __reduce__(self):
        return (_restore_device, ("numpy",))

    def alloc_like(self, mem, dev_dtype=None):
        return None


class CUDADevice(Device):
    """One H100. The sm_90a extension is loaded eagerly and a missing/unloadable
    extension is a hard error (never a silent fallback to eager PyTorch)."""
    is_cuda = True
    backend_name = "cuda"

    def __init__(self, index=None):
        import os
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("CUDADevice requested but no CUDA device is visible")
        if index is None:
            index = int(os.environ.get("LOCAL_RANK", "0"))
        self.index = index
        self.torch_device = torch.device("cuda", index)
        torch.cuda.set_device(self.torch_device)
        props = torch.cuda.get_device_properties(index)
        self.name = props.name
        self.sm_count = props.multi_processor_count
        self.cc = (props.major, props.minor)
        self.total_memory = props.total_memory
        from ..kernels import load_extension
        self.ext = load_extension(required=True)
        self.stream = torch.cuda.current_stream(self.torch_device)
        self.side_stream = torch.cuda.Stream(self.torch_device)
        self.copy_stream = torch.cuda.Stream(self.torch_device)

    def __reduce__(self):
        return (_restore_device, ("cuda",))

    def alloc_like(self, mem, dev_dtype=None):
        import torch
        dt = dev_dtype
        if dt is None:
            dt = torch.from_numpy(numpy.zeros(0, dtype=mem.dtype)).dtype
        return torch.empty(mem.shape, dtype=dt, device=self.torch_device)

    def zeros(self, shape, dtype):
        import torch
        return torch.zeros(shape, dtype=dtype, device=self.torch_device)

    def empty(self, shape, dtype):
        import torch
        return torch.empty(shape, dtype=dtype, device=self.torch_device)

    def sync(self):
        import torch
        torch.cuda.synchronize(self.torch_device)

    def __repr__(self):
        return "<CUDADevice %d %s sm_%d%d %d SMs>" % (
            self.index, self.name, self.cc[0], self.cc[1], self.sm_count)


_auto_device = None


def get_device(backend=None):
    """``backend``: "numpy" | "cuda" | "auto"/None (= root.common.engine.backend)."""
    global _auto_device
    backend = backend or root.common.engine.get("backend", "auto")
    if backend == "numpy":
        return NumpyDevice()
    if backend == "cuda":
        if _auto_device is None or not _auto_device.is_cuda:
            _auto_device = CUDADevice()
        return _auto_device
    if backend in ("auto", None):
        try:
            import torch
            has = torch.cuda.is_available()
        except Exception:  # pragma: no cover
            has = False
        if has:
            return get_device("cuda")
        return NumpyDevice()
    raise ValueError("Unknown backend %r (only numpy and cuda exist)" % (backend,))
