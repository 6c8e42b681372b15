"""Array: a host numpy buffer paired with a device tensor.

Fresh design for ``veles.memory.Array`` (SURVEY §8 "Array protocol"; usages
/root/reference/nn_units.py:145,157-160,196-205,375, /root/reference/all2all.py:262,
/root/reference/evaluator.py:506-513). ``.mem`` is the numpy view, ``.devmem`` is a
``torch.Tensor`` living in H100 HBM. The map_read/map_write/map_invalidate/unmap
API is kept as a thin coherence state machine:

    MAPPED_READ   host valid, device valid
    MAPPED_WRITE  host valid, device stale   (unmap() uploads)
    UNMAPPED      device owns the data       (map_read() downloads)

H100 departures: the device copy may use a narrower dtype than the host copy
(``dev_dtype`` = bf16 activations while ``.mem`` stays float32), and all device
buffers are ordinary torch allocations so CUDA graphs can capture kernels that
read and write them.
"""
from __future__ import annotations

import numpy

_MAPPED_READ, _MAPPED_WRITE, _UNMAPPED = 0, 1, 2


def _graphs_recorder():
    from . import graphs
    return graphs._active_recorder


def roundup(num, align):
    d = num % align
    return num if d == 0 else num + (align - d)


def reshape(arr, shape):
    """Reshape without copying (raises if a copy would be needed)."""
    v = arr.view()
    v.shape = shape
    return v


def ravel(arr):
    return reshape(arr, (arr.size,))


def reshape_transposed(w):
    """View a row-major [a, b] matrix stored transposed as [b, a] and transpose it
    back *logically* (access-order flip only; /root/reference/all2all.py:75-77)."""
    a = w.reshape(w.shape[1], w.shape[0]) if w.ndim == 2 else w
    return a.transpose()


def eq_addr(a, b):
    return a.__array_interface__["data"][0] == b.__array_interface__["data"][0]


def assert_addr(a, b):
    if not eq_addr(a, b):
        raise ValueError("Addresses of the arrays are not equal.")


def interleave(arr):
    """CHW-like [n, c, h, w] (or [c, h, w]) → NHWC."""
    if arr.ndim == 4:
        return numpy.ascontiguousarray(arr.transpose(0, 2, 3, 1))
    if arr.ndim == 3:
        return numpy.ascontiguousarray(arr.transpose(1, 2, 0))
    raise ValueError("Unsupported number of dimensions %d" % arr.ndim)


class NumDiff(object):
    """Numeric differentiation helper (5-point stencil) used by the numdiff tests
    (/root/reference/tests/unit/gd_numdiff.py:43-156)."""

    def __init__(self):
        self.h = 1.0e-6
        self.points = (2.0 * self.h, self.h, -self.h, -2.0 * self.h)
        self.coeffs = numpy.array([-1.0, 8.0, -8.0, 1.0], dtype=numpy.float64)
        self.divizor = 12.0 * self.h
        self.errs = numpy.zeros_like(self.points)

    @property
    def derivative(self):
        return (self.errs * self.coeffs).sum() / self.divizor

    @staticmethod
    def check_diff(x, y, max_diff, logging_info, assertLess, error_text):
        mx = numpy.fabs(x - y).max()
        logging_info("max_diff = %.6f", mx)
        assertLess(mx, max_diff, error_text)


class Array(object):
    """Host+device array with explicit coherence."""

    def __init__(self, data=None, shallow_pickle=False, dev_dtype=None):
        self._mem = None
        self._devmem_ = None
        self._device_ = None
        self._state = _MAPPED_WRITE
        self.shallow_pickle = shallow_pickle
        self.dev_dtype = dev_dtype      # torch dtype or None (= same as host)
        self.max_supposed = 1.0
        self.supposed_max_value = 1.0
        if data is not None:
            self.reset(data)

    # -- pickling ---------------------------------------------------------------
    def __getstate__(self):
        if self._mem is not None and self._devmem_ is not None:
            self.map_read()
        st = {"shallow_pickle": self.shallow_pickle, "dev_dtype": None,
              "max_supposed": self.max_supposed,
              "supposed_max_value": self.supposed_max_value,
              "dev_dtype_name": str(self.dev_dtype) if self.dev_dtype is not None else None}
        if self.shallow_pickle and self._mem is not None:
            st["shape"] = self._mem.shape
            st["dtype"] = self._mem.dtype.str
            st["mem"] = None
        else:
            st["mem"] = self._mem
        return st

    def __setstate__(self, st):
        self.shallow_pickle = st["shallow_pickle"]
        self.max_supposed = st.get("max_supposed", 1.0)
        self.supposed_max_value = st.get("supposed_max_value", 1.0)
        self._devmem_ = None
        self._device_ = None
        self._state = _MAPPED_WRITE
        self.dev_dtype = None
        name = st.get("dev_dtype_name")
        if name:
            import torch
            self.dev_dtype = getattr(torch, name.split(".")[-1])
        if st.get("mem") is None and "shape" in st:
            self._mem = numpy.zeros(st["shape"], dtype=numpy.dtype(st["dtype"]))
        else:
            self._mem = st.get("mem")

    # -- basic protocol -----------------------------------------------------------
    def __bool__(self):
        return self._mem is not None and self._mem.size > 0

    __nonzero__ = __bool__

    def __len__(self):
        return 0 if self._mem is None else len(self._mem)

    def __getitem__(self, key):
        return self.mem[key]

    def __setitem__(self, key, value):
        self.mem[key] = value

    def __repr__(self):
        if self._mem is None:
            return "<Array empty>"
        return "<Array %s %s%s>" % (self._mem.shape, self._mem.dtype,
                                    " +dev" if self._devmem_ is not None else "")

    @property
    def mem(self):
        return self._mem

    @mem.setter
    def mem(self, value):
        if self._devmem_ is not None and value is not None and (
                self._mem is None or value.shape != self._mem.shape):
            raise ValueError("Use reset() to change the shape of an initialized Array")
        self._mem = value
        self._state = _MAPPED_WRITE

    @property
    def devmem(self):
        return self._devmem_

    @property
    def device(self):
        return self._device_

    @property
    def shape(self):
        return self._mem.shape

    @shape.setter
    def shape(self, value):
        self._mem = reshape(self._mem, value)
        if self._devmem_ is not None:
            self._devmem_ = self._devmem_.view(*self._mem.shape)

    @property
    def size(self):
        return 0 if self._mem is None else self._mem.size

    @property
    def dtype(self):
        return self._mem.dtype

    @property
    def itemsize(self):
        return self._mem.itemsize

    @property
    def nbytes(self):
        return self._mem.nbytes

    @property
    def sample_size(self):
        return self._mem.size // self._mem.shape[0]

    @property
    def matrix(self):
        return reshape(self._mem, (self._mem.shape[0], self.sample_size))

    @property
    def plain(self):
        return ravel(self._mem)

    # -- (re)allocation -------------------------------------------------------------
    def reset(self, new_mem=None):
        """Drop the device copy and adopt ``new_mem`` (None = become empty)."""
        self._devmem_ = None
        self._mem = None if new_mem is None else numpy.ascontiguousarray(new_mem)
        self._state = _MAPPED_WRITE
        return self

    def initialize(self, device):
        """Create the device copy (no-op for the numpy device)."""
        if self._mem is None:
            return self
        self._device_ = device
        if device is None or not device.is_cuda:
            return self
        if self._devmem_ is not None and tuple(self._devmem_.shape) == self._mem.shape:
            if self._state == _MAPPED_WRITE:
                self._upload()
                self._state = _MAPPED_READ
            return self
        self._devmem_ = device.alloc_like(self._mem, self.dev_dtype)
        self._upload()
        self._state = _MAPPED_READ
        return self

    def _upload(self):
        """Host → device through a persistent pinned staging buffer (asynchronous w.r.t.
        the host, so run-ahead of the launch queue is preserved; the staging buffer is
        only rewritten after the previous copy out of it has completed)."""
        import torch
        src = torch.from_numpy(self._mem)
        pin = self.__dict__.get("_pin_")
        if pin is None or pin.shape != src.shape or pin.dtype != src.dtype:
            if src.numel() * src.element_size() > (64 << 20):
                self._devmem_.copy_(src)      # huge one-off uploads: plain copy
                return
            pin = torch.empty(src.shape, dtype=src.dtype).pin_memory()
            self.__dict__["_pin_"] = pin
            self.__dict__["_pin_evt_"] = torch.cuda.Event()
        else:
            self.__dict__["_pin_evt_"].synchronize()
        pin.copy_(src)
        dev = self._devmem_
        if dev.dtype != pin.dtype:
            dev.copy_(pin.to(dev.device, non_blocking=True))
        else:
            dev.copy_(pin, non_blocking=True)
        self.__dict__["_pin_evt_"].record()

    def _download(self):
        import torch
        dev = self._devmem_
        dst = torch.from_numpy(self._mem)
        if dev.dtype != dst.dtype:
            dst.copy_(dev.to(dst.dtype))
        else:
            dst.copy_(dev)

    # -- coherence ------------------------------------------------------------------
    def map_read(self):
        if self._devmem_ is not None and self._state == _UNMAPPED:
            self._download()
            self._state = _MAPPED_READ
        return self

    def map_write(self):
        if self._devmem_ is not None and self._state == _UNMAPPED:
            self._download()
        self._state = _MAPPED_WRITE
        return self

    def map_invalidate(self):
        self._state = _MAPPED_WRITE
        return self

    def unmap(self):
        if self._devmem_ is None:
            return self
        if self._state == _MAPPED_WRITE:
            self._upload()
        self._state = _UNMAPPED
        return self

    @property
    def dev(self):
        """Device tensor, made current (the common call in ``cuda_run``)."""
        if self._state == _MAPPED_WRITE:
            self._upload()
            self._state = _MAPPED_READ
        rec = _graphs_recorder()
        if rec is not None:
            rec.read(self)
        return self._devmem_

    def dev_written(self):
        """Mark that a kernel wrote the device copy (host copy is now stale)."""
        self._state = _UNMAPPED
        rec = _graphs_recorder()
        if rec is not None:
            rec.write(self)

    @property
    def dev_out(self):
        """Device tensor about to be fully overwritten by a kernel."""
        self.dev_written()
        return self._devmem_


class ScalarUploader(object):
    """A few per-step host scalars → a fixed device tensor (read by captured kernels).

    Each upload takes the next of ``depth`` pinned slots and is carried out by the
    ``pull_from_host`` kernel (the SMs read the pinned slot; no copy-engine operation enters the
    stream, which on the benchmark platform costs ~100 us per engine switch). The ring makes the
    upload safe while the host runs a few steps ahead of the device (a single pinned buffer would
    be overwritten before the asynchronous transfer of the previous step had read it)."""

    def __init__(self, device, n, dtype, depth=8):
        import torch
        self.dev = torch.zeros(max(n, 4), dtype=dtype, device=device.torch_device)
        self.slots = [torch.zeros(max(n, 4), dtype=dtype).pin_memory() for _ in range(depth)]
        self.i = 0
        ext = getattr(device, "ext", None)
        self.ext = ext if ext is not None and hasattr(ext, "pull_from_host") else None

    def upload(self, values):
        s = self.slots[self.i]
        self.i = (self.i + 1) % len(self.slots)
        for k, v in enumerate(values):
            s[k] = v
        if self.ext is not None:
            self.ext.pull_from_host(s, self.dev)
        else:
            self.dev.copy_(s, non_blocking=True)
        return self.dev
