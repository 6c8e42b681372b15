"""cuda4py-compatible surface (the reference imports ``cuda4py`` / ``cuda4py.blas``; the real
package is absent offline). Implemented on NVIDIA's own ``cuda-python`` bindings: NVRTC for
the run-time compilation of the reference's ``cuda/*.cu`` sources, the driver API for memory,
module loading and kernel launches. Only what the Veles core shim and the reference call."""
import ctypes
import os

import numpy

# CUDA4PY_DRY=1: no GPU is touched (host buffers stand in for device memory, launches and GEMMs
# are counted but not executed) - lets the whole cuda_init / cuda_run control flow of the
# reference be exercised on a CPU-only box; NVRTC compilation is real in both modes.
DRY = bool(os.environ.get("CUDA4PY_DRY"))
dry_stats = {"launches": 0, "gemms": 0, "kernels": {}}

from cuda.bindings import driver as _drv
from cuda.bindings import nvrtc as _nvrtc


class CUDARuntimeError(RuntimeError):
    pass


def _ck(res):
    err = res[0]
    if int(err) != 0:
        name = getattr(err, "name", str(err))
        raise CUDARuntimeError("CUDA driver error: %s" % name)
    return res[1] if len(res) == 2 else res[1:] if len(res) > 2 else None


def _nck(res, prog=None):
    err = res[0]
    if int(err) != 0:
        log = ""
        if prog is not None:
            try:
                _, n = _nvrtc.nvrtcGetProgramLogSize(prog)
                buf = b" " * n
                _nvrtc.nvrtcGetProgramLog(prog, buf)
                log = buf.decode(errors="replace")
            except Exception:
                pass
        raise CUDARuntimeError("NVRTC error %s\n%s" % (getattr(err, "name", err), log))
    return res[1] if len(res) == 2 else res[1:] if len(res) > 2 else None


_inited = False


def _init():
    global _inited
    if DRY:
        return
    if not _inited:
        _ck(_drv.cuInit(0))
        _inited = True


class Device(object):
    def __init__(self, index):
        _init()
        self.index = index
        if DRY:
            self.handle, self.name, self.compute_capability = None, "dry", (9, 0)
            self.multiprocessor_count, self.total_mem = 132, 80 << 30
            return
        self.handle = _ck(_drv.cuDeviceGet(index))
        name = _ck(_drv.cuDeviceGetName(128, self.handle))
        self.name = bytes(name).split(b"\0")[0].decode()
        A = _drv.CUdevice_attribute
        self.compute_capability = (
            _ck(_drv.cuDeviceGetAttribute(A.CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MAJOR, self.handle)),
            _ck(_drv.cuDeviceGetAttribute(A.CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MINOR, self.handle)))
        self.multiprocessor_count = _ck(_drv.cuDeviceGetAttribute(
            A.CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, self.handle))
        self.total_mem = _ck(_drv.cuDeviceTotalMem(self.handle))


class Devices(object):
    def __init__(self):
        _init()
        n = 8 if DRY else _ck(_drv.cuDeviceGetCount())
        self.devices = [Device(i) for i in range(n)]

    def __len__(self):
        return len(self.devices)

    def __getitem__(self, i):
        return self.devices[i]

    def create_some_context(self):
        return Context(self.devices[0])


class MemAlloc(object):
    """Device buffer. ``int(mem)`` is the device pointer (the reference does pointer arithmetic
    on it: /root/reference/conv.py:279-281)."""

    def __init__(self, context, size):
        self.context = context
        self.size = int(size)
        if DRY:
            self._host = numpy.zeros(max(self.size, 1), numpy.uint8)
            self.handle = self._host.ctypes.data
            return
        self.handle = int(_ck(_drv.cuMemAlloc(max(self.size, 1))))

    def __int__(self):
        return self.handle

    __index__ = __int__

    def to_device(self, arr, offs=0, size=None):
        arr = numpy.ascontiguousarray(arr)
        n = arr.nbytes if size is None else size
        if DRY:
            ctypes.memmove(self.handle + offs, arr.ctypes.data, n)
            return
        _ck(_drv.cuMemcpyHtoD(self.handle + offs, arr.ctypes.data, n))

    def to_device_async(self, arr, offs=0, size=None, stream=0):
        n = arr.nbytes if size is None else size
        _ck(_drv.cuMemcpyHtoDAsync(self.handle + offs, arr.ctypes.data, n, stream))

    def to_host(self, arr, offs=0, size=None):
        n = arr.nbytes if size is None else size
        if DRY:
            ctypes.memmove(arr.ctypes.data, self.handle + offs, n)
            return
        _ck(_drv.cuMemcpyDtoH(arr.ctypes.data, self.handle + offs, n))

    def to_host_async(self, arr, offs=0, size=None, stream=0):
        n = arr.nbytes if size is None else size
        _ck(_drv.cuMemcpyDtoHAsync(arr.ctypes.data, self.handle + offs, n, stream))

    def from_device(self, src, size=None, src_offs=0, dst_offs=0):
        n = min(self.size - dst_offs, int(getattr(src, "size", 1 << 62)) - src_offs) if size is None else size
        _ck(_drv.cuMemcpyDtoD(self.handle + dst_offs, int(src) + src_offs, n))

    def from_device_async(self, src, size=None, src_offs=0, dst_offs=0, stream=0):
        n = min(self.size - dst_offs, int(getattr(src, "size", 1 << 62)) - src_offs) if size is None else size
        _ck(_drv.cuMemcpyDtoDAsync(self.handle + dst_offs, int(src) + src_offs, n, stream))

    def memset32_async(self, value=0, offs=0, size=None, stream=0):
        n = (self.size - offs) // 4 if size is None else size
        if n > 0 and DRY:
            ctypes.memset(self.handle + offs, 0, n * 4)
        elif n > 0:
            _ck(_drv.cuMemsetD32Async(self.handle + offs, value, n, stream))

    def release(self):
        if DRY:
            return
        if self.handle:
            try:
                _drv.cuMemFree(self.handle)
            except Exception:
                pass
            self.handle = 0

    def __del__(self):
        self.release()


class Context(object):
    def __init__(self, device):
        self.device = device
        self.handle = None if DRY else _ck(_drv.cuDevicePrimaryCtxRetain(device.handle))
        self.set_current()

    def set_current(self):
        if not DRY:
            _ck(_drv.cuCtxSetCurrent(self.handle))

    push_current = set_current

    def mem_alloc(self, size, flags=0):
        return MemAlloc(self, size)

    def synchronize(self):
        if not DRY:
            _ck(_drv.cuCtxSynchronize())


class _Skip(object):
    def __init__(self, n):
        self.n = n


def skip(n=1):
    return _Skip(n)


class Function(object):
    """Kernel handle with cuda4py call conventions: ``set_args(*args)``, ``set_arg(i, a)``,
    ``fn(grid, block)``. Arguments: device buffers / python ints (64-bit pointers), None
    (NULL), 1-element numpy arrays and numpy scalars (passed by value with their dtype)."""
    MAX_ARGS = 64

    def __init__(self, module, name):
        self.module = module
        self.name = name
        if DRY:
            if ("%s" % name).encode() not in module.binary:
                raise CUDARuntimeError("kernel %s not found in module" % name)
            self.handle = None
        else:
            self.handle = _ck(_drv.cuModuleGetFunction(module.handle, name.encode()))
        self._slots = [None] * self.MAX_ARGS          # ctypes buffers (kept alive)
        self._ptrs = (ctypes.c_void_p * self.MAX_ARGS)()
        self._refs = [None] * self.MAX_ARGS           # keeps MemAlloc objects alive
        self._n = 0

    def _store(self, i, arg):
        if hasattr(arg, "devmem"):                    # veles.memory.Array
            arg = arg.devmem
        if arg is None:
            raw = (0).to_bytes(8, "little")
        elif isinstance(arg, MemAlloc):
            self._refs[i] = arg
            raw = arg.handle.to_bytes(8, "little")
        elif isinstance(arg, numpy.ndarray):
            if arg.size != 1:
                raise ValueError("kernel scalar argument must have exactly one element")
            raw = arg.tobytes()
        elif isinstance(arg, numpy.generic):
            raw = arg.tobytes()
        elif isinstance(arg, int):
            raw = int(arg).to_bytes(8, "little", signed=arg < 0)
        elif isinstance(arg, float):
            raise TypeError("python float kernel argument is ambiguous (use a numpy scalar)")
        else:
            raw = int(arg).to_bytes(8, "little")
        buf = self._slots[i]
        if buf is None or len(buf) != len(raw):
            buf = ctypes.create_string_buffer(len(raw), len(raw))
            self._slots[i] = buf
            self._ptrs[i] = ctypes.addressof(buf)
        ctypes.memmove(buf, raw, len(raw))
        if i + 1 > self._n:
            self._n = i + 1

    def set_arg(self, i, arg):
        self._store(i, arg)

    def set_args(self, *args):
        i = 0
        for a in args:
            if isinstance(a, _Skip):
                i += a.n
                continue
            self._store(i, a)
            i += 1

    def __call__(self, grid_dims, block_dims=(1, 1, 1), args_tuple=None, shared_mem=0, stream=0):
        if args_tuple is not None:
            self.set_args(*args_tuple)
        g = tuple(grid_dims) + (1,) * (3 - len(grid_dims))
        b = tuple(block_dims) + (1,) * (3 - len(block_dims))
        if DRY:
            dry_stats["launches"] += 1
            dry_stats["kernels"][self.name] = dry_stats["kernels"].get(self.name, 0) + 1
            assert all(int(v) > 0 for v in g + b), (self.name, g, b)
            if self.name == "evaluate_softmax":      # keep the decision logic alive: fake errors
                ptr = int.from_bytes(bytes(self._slots[5]), "little")
                (ctypes.c_int32 * 2).from_address(ptr)[0] += 50
                (ctypes.c_int32 * 2).from_address(ptr)[1] += 100
            return
        dry_stats["launches"] += 1
        _ck(_drv.cuLaunchKernel(self.handle, int(g[0]), int(g[1]), int(g[2]), int(b[0]), int(b[1]),
                                int(b[2]), shared_mem, stream, ctypes.addressof(self._ptrs), 0))

    def max_active_blocks_per_multiprocessor(self, block_size, dynamic_smem_size=0):
        if DRY:
            return 2048 // block_size
        return int(_ck(_drv.cuOccupancyMaxActiveBlocksPerMultiprocessor(
            self.handle, block_size, dynamic_smem_size)))

    def max_potential_block_size(self, dynamic_smem_size=0, block_size_limit=0):
        """(min grid size, block size) with the occupancy API's rule: the largest block size
        that reaches the maximum number of resident threads per SM."""
        lim = 1024 if DRY else int(_ck(_drv.cuFuncGetAttribute(
            _drv.CUfunction_attribute.CU_FUNC_ATTRIBUTE_MAX_THREADS_PER_BLOCK, self.handle)))
        if block_size_limit:
            lim = min(lim, block_size_limit)
        best, best_threads = 32, -1
        bs = (lim // 32) * 32
        while bs >= 32:
            t = self.max_active_blocks_per_multiprocessor(bs, dynamic_smem_size) * bs
            if t > best_threads:
                best, best_threads = bs, t
            bs -= 32
        sms = self.module.context.device.multiprocessor_count
        return sms * max(best_threads // best, 1), best


class Module(object):
    """NVRTC-compiled module. ``source`` is CUDA C; ``include_dirs`` are searched by #include."""

    def __init__(self, context, ptx=None, source=None, source_file=None, include_dirs=(),
                 options=(), nvcc_path=None):
        self.context = context
        if source is None and source_file is not None:
            with open(source_file) as f:
                source = f.read()
        if source is None:
            raise ValueError("source is required")
        cc = context.device.compute_capability if context is not None else (9, 0)
        self.binary = compile_source(source, include_dirs, options, cc)
        if context is not None and not DRY:
            context.set_current()
            self.handle = _ck(_drv.cuModuleLoadData(self.binary))
        else:
            self.handle = None

    def create_function(self, name):
        return Function(self, name)

    get_function = create_function


def compile_source(source, include_dirs=(), options=(), cc=(9, 0), name="veles_program.cu"):
    """CUDA C -> cubin for sm_<cc> with NVRTC (works without a GPU)."""
    prog = _nck(_nvrtc.nvrtcCreateProgram(source.encode(), name.encode(), 0, [], []))
    opts = [("--gpu-architecture=sm_%d%d" % tuple(cc)).encode(), b"--std=c++14",
            b"-default-device"]
    opts += [("-I" + d).encode() for d in include_dirs]
    opts += [o.encode() if isinstance(o, str) else o for o in options]
    try:
        _nck(_nvrtc.nvrtcCompileProgram(prog, len(opts), opts), prog)
        n = _nck(_nvrtc.nvrtcGetCUBINSize(prog))
        buf = b" " * n
        _nck(_nvrtc.nvrtcGetCUBIN(prog, buf))
        return buf
    finally:
        _nvrtc.nvrtcDestroyProgram(prog)


class Event(object):
    """CUDA event on the legacy default stream (where every launch of this shim goes)."""

    def __init__(self):
        self.handle = None if DRY else _ck(_drv.cuEventCreate(0))
        self._t = 0.0

    def record(self, stream=0):
        if DRY:
            import time
            self._t = time.perf_counter()
            return
        _ck(_drv.cuEventRecord(self.handle, stream))

    def synchronize(self):
        if not DRY:
            _ck(_drv.cuEventSynchronize(self.handle))

    def elapsed_ms(self, end):
        if DRY:
            return (end._t - self._t) * 1e3
        end.synchronize()
        return float(_ck(_drv.cuEventElapsedTime(self.handle, end.handle)))
