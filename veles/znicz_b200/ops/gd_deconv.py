"""Gradient descent for Deconv.

Parity: /root/reference/gd_deconv.py:53-409 (divide err_output by hits or the constant
overlap; ``err_input = im2col(err_output) · Wᵀ``; ``gradW += inputᵀ · im2col(err_output)``;
shared fused weights update; no bias). numpy oracle written fresh (reference :408-409 has
none).

H100: err_input is the conv *fprop* kernel applied to the scaled err_output, wgrad is the
conv wgrad kernel with (image = scaled err_output, errors = deconv input).
"""
from __future__ import annotations

import numpy

from . import nn_units
from .conv import ConvolutionalBase, im2col
from .gd import GDCommon


class GDDeconv(ConvolutionalBase, GDCommon):
    MAPPING = {"deconv"}

    def __init__(self, workflow, **kwargs):
        kwargs["include_bias"] = False
        super().__init__(workflow, **kwargs)
        self.hits = None
        self.undemand("bias", "unpack_size")
        self.demand("weights")

    @property
    def channels_number(self):
        sy, sx = self.err_output.shape[1:3]
        return self.err_output.size // (self.err_output.shape[0] * sx * sy)

    @property
    def unsafe_padding(self):
        return self.hits is not None and bool(self.hits)

    def initialize(self, device=None, **kwargs):
        if not self.input or not self.err_output or not self.weights:
            return True
        super().initialize(device=device, **kwargs)
        self.sliding = tuple(self.sliding)
        self.padding = tuple(self.padding)
        self._n_channels = self.channels_number
        self._kernel_size = self.kx * self.ky * self._n_channels
        self._sy, self._sx = self.err_output.shape[1:3]
        self._batch_size = self.err_output.shape[0]
        self._ky_app, self._kx_app = self.input.shape[1:3]
        if self.weights.size != self.n_kernels * self._kernel_size:
            raise ValueError("Incorrectly shaped weights encountered")
        if self.hits is not None and self.hits:
            self.init_vectors(self.hits)
        return None

    @property
    def scale(self):
        return 1.0 / ((self.kx // self.sliding[0]) * (self.ky // self.sliding[1]))

    def numpy_run(self):
        self.err_output.map_write()
        self.input.map_read()
        self.weights.map_read()
        eo = self.err_output.mem
        if self.unsafe_padding:
            self.hits.map_read()
            eo /= numpy.maximum(self.hits.mem, 1)
        else:
            eo *= self.scale
        cols = im2col(eo.reshape(self._batch_size, self._sy, self._sx, self._n_channels),
                      self.ky, self.kx, self.padding, self.sliding) \
            .reshape(-1, self._kernel_size)
        w = self.weights.mem.transpose() if self.weights_transposed else self.weights.mem
        if self.need_err_input:
            self.err_input.map_write()
            bp = cols.dot(w.transpose()).reshape(self.err_input.shape) * self.err_input_alpha
            if self.err_input_beta:
                self.err_input.mem *= self.err_input_beta
                self.err_input.mem += bp
            else:
                self.err_input.mem[...] = bp
        if self.need_gradient_weights:
            self.gradient_weights.map_invalidate()
            g = self.input.mem.reshape(-1, self.n_kernels).transpose().dot(cols)
            if self.weights_transposed:
                g = g.transpose()
            self.gradient_weights.mem[...] = g.reshape(self.gradient_weights.shape)
            self.numpy_update("weights")
        if self.on_cuda_forward_shadow():
            self.forward_unit.refresh_shadows()

    def cuda_run(self):
        from ..kernels import api
        api.deconv_backward(self)
