"""Native (C++) forward-only runtime — python binding over the C ABI (ctypes)."""
from __future__ import annotations

import ctypes
import os

import numpy

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def load_library():
    global _lib
    if _lib is not None:
        return _lib
    path = os.path.join(HERE, "libznicz_native.so")
    if not os.path.exists(path):
        from . import build
        build.build(verbose=False)
    lib = ctypes.CDLL(path)
    lib.znicz_engine_create.restype = ctypes.c_void_p
    lib.znicz_engine_create.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int]
    lib.znicz_engine_destroy.argtypes = [ctypes.c_void_p]
    lib.znicz_engine_num_units.argtypes = [ctypes.c_void_p]
    lib.znicz_engine_infer.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int),
                                       ctypes.POINTER(ctypes.c_int)]
    lib.znicz_engine_run.argtypes = [
        ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_float),
        ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_float), ctypes.c_longlong,
        ctypes.c_char_p, ctypes.c_int]
    lib.znicz_engine_tc_launches.restype = ctypes.c_longlong
    lib.znicz_engine_tc_launches.argtypes = [ctypes.c_void_p]
    _lib = lib
    return lib


def cuda_available():
    return bool(load_library().znicz_cuda_available())


class NativeEngine(object):
    """``NativeEngine("mnist.zip").run(x)`` — x: [n, features] or NHWC float array."""

    def __init__(self, package_path):
        lib = load_library()
        err = ctypes.create_string_buffer(512)
        self._h = lib.znicz_engine_create(str(package_path).encode(), err, 512)
        if not self._h:
            raise RuntimeError("native engine: %s" % err.value.decode())
        self._lib = lib

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._lib.znicz_engine_destroy(h)
            self._h = None

    @property
    def num_units(self):
        return self._lib.znicz_engine_num_units(self._h)

    @property
    def tensor_core_launches(self):
        """wgmma GEMM / conv launches issued by the CUDA executor so far."""
        return int(self._lib.znicz_engine_tc_launches(self._h))

    @staticmethod
    def _shape4(x):
        if x.ndim == 2:
            return (x.shape[0], 1, 1, x.shape[1])
        if x.ndim == 4:
            return tuple(x.shape)
        if x.ndim == 3:
            return tuple(x.shape) + (1,)
        raise ValueError("input must be [n, features] or NHWC")

    def run(self, x, backend="cpu"):
        x = numpy.ascontiguousarray(x, dtype=numpy.float32)
        s4 = (ctypes.c_int * 4)(*self._shape4(x))
        o4 = (ctypes.c_int * 4)()
        if self._lib.znicz_engine_infer(self._h, s4, o4):
            raise ValueError("input shape %s does not fit the packaged model" % (x.shape,))
        out = numpy.empty(tuple(o4), dtype=numpy.float32)
        err = ctypes.create_string_buffer(512)
        rc = self._lib.znicz_engine_run(
            self._h, 1 if backend == "cuda" else 0,
            x.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), s4,
            out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), out.size, err, 512)
        if rc:
            raise RuntimeError("native engine: %s" % err.value.decode())
        if out.shape[1] == 1 and out.shape[2] == 1:
            out = out.reshape(out.shape[0], out.shape[3])
        return out
