"""Gradient descent for convolutional layers.

Parity: /root/reference/gd_conv.py (GradientDescentConv :60, GDTanhConv :645,
GDSigmoidConv :675, GDRELUConv :701, GDStrictRELUConv :726): dgrad
(``err_input``), wgrad (``gradient_weights``), bias gradient = Σ over batch·pixels,
then the shared fused SGD step.

H100 path: dgrad is a *gather* implicit GEMM over the transposed filters (no
``atomicAdd`` col2im scatter → deterministic), wgrad is a split-K implicit GEMM
over batch·pixels whose per-CTA partials are summed in fixed order by the fused
update kernel (reference: per-16-image Unpack1D + cuBLAS β=1 accumulation and an
atomic ``DirectPack`` scatter, /root/reference/gd_conv.py:313-423).
"""
from __future__ import annotations

from . import nn_units
from .conv import ConvolutionalBase, im2col, col2im, conv_output_size
from .gd import GDCommon
from .nn_units import (ACT_LINEAR, ACT_TANH, ACT_RELU, ACT_STRICT_RELU, ACT_SIGMOID)


class GradientDescentConv(ConvolutionalBase, GDCommon):
    MAPPING = {"conv"}
    ACT = ACT_LINEAR

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.demand("weights")
        if self.include_bias:
            self.demand("bias")

    def initialize(self, device=None, **kwargs):
        if not self.input or not self.err_output:
            return True
        super().initialize(device=device, **kwargs)
        shp = self.input.shape
        if len(shp) == 3:
            shp = shp + (1,)
        self._batch_size, self._sy, self._sx = shp[0], shp[1], shp[2]
        self._n_channels = self.input.size // (self._batch_size * self._sx * self._sy)
        self._kernel_size = self.kx * self.ky * self._n_channels
        self._kx_app = conv_output_size(self._sx, self.kx, self.padding[0],
                                        self.padding[2], self.sliding[0])
        self._ky_app = conv_output_size(self._sy, self.ky, self.padding[1],
                                        self.padding[3], self.sliding[1])
        self._kernel_app_per_image = self._kx_app * self._ky_app
        self._kernel_app_total = self._batch_size * self._kernel_app_per_image
        n_weights = self.n_kernels * self._kernel_size
        if self.weights.size != n_weights:
            raise ValueError("Expected number of weights to match input, n_kernels, "
                             "kx, ky parameters")
        if self.include_bias and self.bias and self.bias.size != self.n_kernels:
            raise ValueError("Expected bias to match n_kernels")
        return None

    @property
    def input_nhwc(self):
        return (self._batch_size, self._sy, self._sx, self._n_channels)

    # -- numpy oracle -----------------------------------------------------------------
    def numpy_err_input_update(self):
        if not self.need_err_input:
            return
        self.err_input.map_write()
        self.err_output.map_read()
        self.weights.map_read()
        w = self.weights.mem.transpose() if self.weights_transposed else self.weights.mem
        eo = self.err_output.mem.reshape(-1, self.n_kernels)
        cols = eo.dot(w)
        bp = col2im(cols, self.input_nhwc, self.ky, self.kx, self.padding, self.sliding)
        bp = bp.reshape(self.err_input.shape) * self.err_input_alpha
        if self.err_input_beta:
            self.err_input.mem *= self.err_input_beta
            self.err_input.mem += bp
        else:
            self.err_input.mem[...] = bp

    def numpy_weights_update(self):
        if not self.need_gradient_weights:
            return
        self.input.map_read()
        self.err_output.map_read()
        x = self.input.mem.reshape(self.input_nhwc)
        cols = im2col(x, self.ky, self.kx, self.padding, self.sliding) \
            .reshape(-1, self._kernel_size)
        eo = self.err_output.mem.reshape(-1, self.n_kernels)
        self.gradient_weights.map_invalidate()
        g = eo.transpose().dot(cols)
        if self.weights_transposed:
            g = g.transpose()
        self.gradient_weights.mem[...] = g.reshape(self.gradient_weights.shape)
        self.numpy_update("weights")

    def numpy_bias_update(self):
        if not self.need_gradient_weights or not self.include_bias:
            return
        self.err_output.map_read()
        self.gradient_bias.map_invalidate()
        self.gradient_bias.mem[:] = self.err_output.mem.reshape(
            -1, self.n_kernels).sum(axis=0)
        self.numpy_update("bias")

    def numpy_run(self):
        self.numpy_err_output_update()
        self.numpy_err_input_update()
        self.numpy_weights_update()
        self.numpy_bias_update()
        if self.on_cuda_forward_shadow():
            self.forward_unit.refresh_shadows()

    # -- sm_90a ------------------------------------------------------------------------
    def cuda_run(self):
        from ..kernels import api
        api.conv_backward(self)


class GDTanhConv(nn_units.GradientDescentWithActivation, GradientDescentConv):
    MAPPING = {"conv_tanh"}
    ACT = ACT_TANH


class GDSigmoidConv(nn_units.GradientDescentWithActivation, GradientDescentConv):
    MAPPING = {"conv_sigmoid"}
    ACT = ACT_SIGMOID


class GDRELUConv(nn_units.GradientDescentWithActivation, GradientDescentConv):
    MAPPING = {"conv_relu"}
    ACT = ACT_RELU


class GDStrictRELUConv(nn_units.GradientDescentWithActivation, GradientDescentConv):
    MAPPING = {"conv_str"}
    ACT = ACT_STRICT_RELU
