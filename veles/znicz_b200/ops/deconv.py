"""Deconv: transposed convolution sharing weights with a Conv (no bias).

Parity: /root/reference/deconv.py (Deconv :55, ``compute_padding`` :91,
``check_padding_is_safe`` :101, ``hits`` overlap counter :185-190). The reference has no
numpy path (:347-348); the oracle here is ``col2im(input · W)`` scaled by the overlap count.

``output = col2im(input[N,oy,ox,F] · W[F, ky·kx·C]) / overlap`` where overlap is
``(kx/slide_x)·(ky/slide_y)`` for safe paddings, otherwise the per-pixel number of windows
(``hits``) — a *static* map of the geometry, computed once on the host (the reference
counts it with ``atomicAdd`` every run, /root/reference/cuda/conv/gradient_descent/
err_input_update.cu:31, cuda/deconv/forward.cu:12).

H100: the transposed conv *is* the conv dgrad gather kernel (no atomics), with the
overlap scaling folded into ``alpha`` (safe) or applied as a reciprocal-hits multiply.
"""
from __future__ import annotations

import numpy

from ..core.distributable import TriviallyDistributable
from ..core.memory import Array
from . import nn_units
from .conv import ConvolutionalBase, col2im, conv_output_size


def overlap_hits(sy, sx, ky, kx, padding, sliding):
    """[sy, sx] map: how many kernel applications cover each pixel."""
    left, top, right, bottom = padding
    oy = conv_output_size(sy, ky, top, bottom, sliding[1])
    ox = conv_output_size(sx, kx, left, right, sliding[0])
    hp = numpy.zeros((sy + top + bottom, sx + left + right), dtype=numpy.int32)
    for i in range(oy):
        for j in range(ox):
            hp[i * sliding[1]:i * sliding[1] + ky, j * sliding[0]:j * sliding[0] + kx] += 1
    return hp[top:top + sy, left:left + sx]


class Deconv(TriviallyDistributable, ConvolutionalBase, nn_units.Forward):
    MAPPING = {"deconv"}

    @staticmethod
    def compute_padding(sx, sy, kx, ky, sliding):
        """Padding that makes ``Conv(padding)`` map (sy, sx) onto the deconv input."""
        return (kx - sliding[1], ky - sliding[0],
                kx - sx % sliding[1] if sx % sliding[1] != 0 else kx - sliding[1],
                ky - sy % sliding[0] if sy % sliding[0] != 0 else ky - sliding[0])

    @staticmethod
    def check_padding_is_safe(kx, ky, sliding):
        if sliding[0] > (ky >> 1) or sliding[1] > (kx >> 1):
            raise ValueError("sliding should not be greater than half of the kernel size")
        if kx % sliding[0] != 0 or kx % sliding[1] != 0:
            raise ValueError("Kernel size should be multiple of sliding")

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.unsafe_padding = kwargs.get("unsafe_padding", False)
        self.hits = Array()
        self.include_bias = False
        self.bias = None
        self.output_shape_source = None
        for a in ("n_kernels", "kx", "ky", "padding", "sliding"):
            if a in kwargs and getattr(self, a, None) is None:
                setattr(self, a, kwargs[a])
        self.demand("n_kernels", "kx", "ky", "sliding", "input", "weights",
                    "output_shape_source")
        self.undemand("padding", "unpack_size")

    def init_unpickled(self):
        super().init_unpickled()
        self.rhits_dev_ = None

    def initialize(self, device=None, **kwargs):
        if not self.input or not self.weights or not self.output_shape_source:
            return True
        super().initialize(device=device, **kwargs)
        self.weights_shape = (tuple(reversed(self.weights.shape))
                              if self.weights_transposed else tuple(self.weights.shape))
        if len(self.input.shape) != 4 or self.input.shape[3] != self.n_kernels:
            raise ValueError("Incorrectly shaped input encountered")
        if (len(self.weights_shape) != 2 or self.weights_shape[0] != self.n_kernels or
                self.weights_shape[1] % (self.kx * self.ky) != 0):
            raise ValueError("Incorrectly shaped weights encountered")
        output_shape = tuple(self.output_shape_source.shape)
        if len(output_shape) != 4:
            raise ValueError("Incorrect output_shape_source shape")
        if output_shape[0] != self.input.shape[0]:
            raise ValueError("output_shape_source.shape[0] != input.shape[0]")
        self.sliding = tuple(self.sliding)
        use_hits = False
        try:
            self.check_padding_is_safe(self.kx, self.ky, self.sliding)
        except ValueError:
            if not self.unsafe_padding:
                raise
            self.warning("The padding will be unsafe")
            use_hits = True
        padding = Deconv.compute_padding(output_shape[2], output_shape[1], self.kx, self.ky,
                                         self.sliding)
        if getattr(self, "padding", None) is None:
            self.padding = padding
        elif tuple(self.padding) != tuple(padding):
            if not self.unsafe_padding:
                raise ValueError("Expected padding %s but got %s" % (padding, self.padding))
            use_hits = True
        self.padding = tuple(self.padding)
        self._output_shape = output_shape
        self._sy, self._sx, self._n_channels = output_shape[1:]
        self._kernel_size = self.kx * self.ky * self._n_channels
        oy = conv_output_size(self._sy, self.ky, self.padding[1], self.padding[3],
                              self.sliding[1])
        ox = conv_output_size(self._sx, self.kx, self.padding[0], self.padding[2],
                              self.sliding[0])
        if (oy, ox) != tuple(self.input.shape[1:3]):
            raise ValueError("input %s does not match the geometry (%d, %d)" % (
                self.input.shape, oy, ox))
        if use_hits:
            h = overlap_hits(self._sy, self._sx, self.ky, self.kx, self.padding, self.sliding)
            full = numpy.broadcast_to(h[None, :, :, None], output_shape)
            self.hits.reset(numpy.ascontiguousarray(full, dtype=numpy.int32))
        self.make_output(output_shape, self.input.dtype)
        self.output.dev_dtype = self.input.dev_dtype
        self.init_vectors(self.input, self.weights, self.output, self.hits)
        return None

    @property
    def scale(self):
        """Overlap normalisation for safe geometries."""
        return 1.0 / ((self.kx // self.sliding[0]) * (self.ky // self.sliding[1]))

    def numpy_run(self):
        self.input.map_read()
        self.weights.map_read()
        self.output.map_invalidate()
        w = self.weights.mem.transpose() if self.weights_transposed else self.weights.mem
        cols = self.input.mem.reshape(-1, self.n_kernels).dot(w)
        out = col2im(cols, self._output_shape, self.ky, self.kx, self.padding, self.sliding)
        if self.hits:
            out = out / numpy.maximum(self.hits.mem, 1)
        else:
            out = out * self.scale
        self.output.mem[...] = out

    def cuda_run(self):
        from ..kernels import api
        api.deconv_forward(self)
