"""Convolutional forward units (NHWC, implicit GEMM).

Parity: /root/reference/conv.py (ConvolutionalBase :57, Conv :71-476, ConvTanh :478,
ConvSigmoid :500, ConvRELU :522 (softplus), ConvStrictRELU :547).
``padding=(left, top, right, bottom)``, ``sliding=(x, y)``; output size
``1 + (S − K + pad) // slide`` (:161-166); weights ``[n_kernels, ky·kx·C]`` row-major
with (ky, kx, C) order; default magnitude ``min(1/(max·sqrt(ky·kx·C)), 0.05)``.

H100 path: no im2col buffer exists. ``conv_fprop`` is an implicit-GEMM wgmma
kernel: producer warps gather the NHWC patches straight into 128B-swizzled shared
memory (zero fill for the padding), one warpgroup issues ``wgmma.mma_async`` into
register accumulators and the epilogue adds bias and applies the activation
(reference: 16-image ``Unpack1D`` + cuBLAS + a bias/activation kernel,
/root/reference/conv.py:268-297).
"""
from __future__ import annotations

import numpy

from ..core.memory import Array
from ..core.units import Unit
from . import nn_units
from .all2all import apply_activation_numpy
from .nn_units import (ACT_LINEAR, ACT_TANH, ACT_RELU, ACT_STRICT_RELU, ACT_SIGMOID)


def conv_output_size(s, k, pad_a, pad_b, slide):
    return 1 + (s - k + pad_a + pad_b) // slide


def im2col(x, ky, kx, padding, sliding):
    """NHWC ``x`` → ``[n, oy, ox, ky*kx*C]`` patches (zero padded). numpy oracle."""
    n, sy, sx, c = x.shape
    left, top, right, bottom = padding
    slx, sly = sliding
    oy = conv_output_size(sy, ky, top, bottom, sly)
    ox = conv_output_size(sx, kx, left, right, slx)
    xp = numpy.zeros((n, sy + top + bottom, sx + left + right, c), dtype=x.dtype)
    xp[:, top:top + sy, left:left + sx] = x
    cols = numpy.empty((n, oy, ox, ky, kx, c), dtype=x.dtype)
    for i in range(ky):
        for j in range(kx):
            cols[:, :, :, i, j, :] = xp[:, i:i + (oy - 1) * sly + 1:sly,
                                        j:j + (ox - 1) * slx + 1:slx, :]
    return cols.reshape(n, oy, ox, ky * kx * c)


def col2im(cols, x_shape, ky, kx, padding, sliding):
    """Adjoint of :func:`im2col` (overlapping patches are summed)."""
    n, sy, sx, c = x_shape
    left, top, right, bottom = padding
    slx, sly = sliding
    oy = conv_output_size(sy, ky, top, bottom, sly)
    ox = conv_output_size(sx, kx, left, right, slx)
    cols = cols.reshape(n, oy, ox, ky, kx, c)
    xp = numpy.zeros((n, sy + top + bottom, sx + left + right, c), dtype=cols.dtype)
    for i in range(ky):
        for j in range(kx):
            xp[:, i:i + (oy - 1) * sly + 1:sly, j:j + (ox - 1) * slx + 1:slx, :] += \
                cols[:, :, :, i, j, :]
    return xp[:, top:top + sy, left:left + sx]


class ConvolutionalBase(Unit):
    hide_from_registry = True
    CONV_ATTRS = ("n_kernels", "kx", "ky", "sliding", "padding", "unpack_size")

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.demand(*self.CONV_ATTRS)
        for attr in self.CONV_ATTRS:     # GD units may get them as kwargs or by link
            if attr in kwargs:
                v = kwargs[attr]
                setattr(self, attr, tuple(v) if attr in ("sliding", "padding") else v)
        if getattr(self, "unpack_size", None) is None:
            self.unpack_size = 16

    def link_conv_attrs(self, other):
        self.link_attrs(other, *self.CONV_ATTRS)
        return self


class Conv(ConvolutionalBase, nn_units.NNLayerBase):
    """Convolution with linear activation."""
    MAPPING = {"conv"}
    ACT = ACT_LINEAR

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        try:
            self.n_kernels = kwargs["n_kernels"]
            self.kx = kwargs["kx"]
            self.ky = kwargs["ky"]
        except KeyError:
            raise KeyError("n_kernels, kx and ky are required parameters") from None
        self.padding = tuple(kwargs.get("padding", (0, 0, 0, 0)))   # L T R B
        self.sliding = tuple(kwargs.get("sliding", (1, 1)))         # X Y
        if len(self.padding) != 4 or len(self.sliding) != 2:
            raise ValueError("padding must have 4 and sliding 2 elements")
        self.activation_mode = "ACTIVATION_LINEAR"
        self.exports.extend(("activation_mode", "kx", "ky", "n_kernels",
                             "padding", "sliding"))
        self.unpack_size = kwargs.get("unpack_size", 16)  # API parity; unused on H100
        self.weights_shape = None

    def get_weights_magnitude(self):
        n_channels = self.input.size // (self.input.shape[0] * self.input.shape[1] *
                                         self.input.shape[2])
        vle = (1.0 / self.input.max_supposed /
               numpy.sqrt(self.kx * self.ky * n_channels))
        if self.weights_filling == "gaussian":
            vle /= 3
        return vle

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        super().initialize(device=device, **kwargs)
        if self.weights_stddev is None:
            self.weights_stddev = min(self.get_weights_magnitude(), 0.05)
        if self.bias_stddev is None:
            self.bias_stddev = self.weights_stddev
        shp = self.input.shape
        if len(shp) == 3:   # single-channel images without the C axis
            shp = shp + (1,)
        self._batch_size, self._sy, self._sx = shp[0], shp[1], shp[2]
        self._n_channels = self.input.size // (self._batch_size * self._sx * self._sy)
        self._kx_app = conv_output_size(self._sx, self.kx, self.padding[0],
                                        self.padding[2], self.sliding[0])
        self._ky_app = conv_output_size(self._sy, self.ky, self.padding[1],
                                        self.padding[3], self.sliding[1])
        if self._kx_app < 1 or self._ky_app < 1:
            raise ValueError("%s: kernel does not fit into the padded input" % self)
        self._kernel_app_per_image = self._kx_app * self._ky_app
        self._kernel_size = self.kx * self.ky * self._n_channels
        self._fill_weights()
        self._fill_biases()
        output_shape = (self._batch_size, self._ky_app, self._kx_app, self.n_kernels)
        self.make_output(output_shape, self.input.dtype)
        self.init_vectors(self.input, self.output, self.weights, self.bias)
        if self.on_cuda:
            self.refresh_shadows()
        return None

    @property
    def input_nhwc(self):
        return (self._batch_size, self._sy, self._sx, self._n_channels)

    def _fill_array(self, filling_type, mem, stddev):
        if filling_type == "gabor":
            self._fill_with_gabor_filters(self.n_kernels, (self.ky, self.kx), stddev)
        else:
            self.fill_array(filling_type, mem, stddev)

    def _fill_weights(self):
        self.weights_shape = (self.n_kernels, self._kernel_size)
        weights_shape_t = tuple(reversed(self.weights_shape))
        if not self.weights:
            self.weights.reset(numpy.zeros(self.weights_shape, dtype=self.input.dtype))
            self._fill_array(self.weights_filling, self.weights.mem, self.weights_stddev)
            if self.weights_transposed:
                a = self.weights.mem.transpose().copy()
                self.weights.reset(a)
        else:
            expect = weights_shape_t if self.weights_transposed else self.weights_shape
            if tuple(self.weights.shape) != expect:
                raise ValueError("%s: weights shape %s != %s" % (
                    self, self.weights.shape, expect))

    def _fill_biases(self):
        if not self.include_bias:
            return
        if not self.bias:
            self.bias.reset(numpy.zeros(self.n_kernels, self.input.dtype))
            self._fill_array(self.bias_filling, self.bias.mem, self.bias_stddev)
        elif self.bias.size != self.n_kernels:
            raise ValueError("%s: bias size mismatch" % self)

    def _fill_with_gabor_filters(self, n_filters, shape, stddev):
        """Gabor bank (4 orientations × 2 phases × wavelength/σ ladder); the rest
        is white noise (/root/reference/conv.py:425-476). Pure numpy (no cv2)."""
        ky, kx = shape
        size = min(shape)
        c = self._n_channels
        w = self.weights.mem.reshape(self.n_kernels, ky, kx, c)
        ys, xs = numpy.mgrid[0:ky, 0:kx].astype(numpy.float64)
        ys -= (ky - 1) / 2.0
        xs -= (kx - 1) / 2.0
        count = 0
        for wavelen_ratio in range(1, 4):
            for dev_ratio in range(1, 2 * wavelen_ratio + 1):
                for ori in (0, numpy.pi / 4, numpy.pi / 2, 3 * numpy.pi / 4):
                    for phase in (0, numpy.pi):
                        sigma = size / dev_ratio / 2.0
                        lambd = size / float(wavelen_ratio)
                        xr = xs * numpy.cos(ori) + ys * numpy.sin(ori)
                        yr = -xs * numpy.sin(ori) + ys * numpy.cos(ori)
                        g = numpy.exp(-(xr ** 2 + yr ** 2) / (2 * sigma ** 2)) * \
                            numpy.cos(2 * numpy.pi * xr / lambd + phase)
                        g -= g.min()
                        mx = g.max()
                        if mx:
                            g /= mx
                        g = (g * 2.0 - 1.0) * stddev
                        w[count] = g[:, :, None]
                        count += 1
                        if count == n_filters:
                            return
        rest = self.weights.mem.reshape(self.n_kernels, -1)[count:]
        self.rand.fill_normal_real(rest, 0, stddev)

    # -- numpy oracle -----------------------------------------------------------------
    def numpy_run(self):
        self.input.map_read()
        self.weights.map_read()
        self.output.map_invalidate()
        x = self.input.mem.reshape(self.input_nhwc)
        w = self.weights.mem.transpose() if self.weights_transposed else self.weights.mem
        cols = im2col(x, self.ky, self.kx, self.padding, self.sliding)
        out = cols.reshape(-1, self._kernel_size).dot(w.transpose())
        if self.include_bias:
            self.bias.map_read()
            out += self.bias.mem
        apply_activation_numpy(out, self.ACT)
        self.output.mem[...] = out.reshape(self.output.shape)

    # -- sm_90a ------------------------------------------------------------------------
    def refresh_shadows(self):
        from ..kernels import api
        api.refresh_weight_shadows(self)

    def cuda_run(self):
        from ..kernels import api
        api.conv_forward(self)


class ConvTanh(Conv):
    """Conv with scaled tanh: f(x) = 1.7159 · tanh(0.6666 · x)."""
    MAPPING = {"conv_tanh"}
    ACT = ACT_TANH

    def initialize(self, device=None, **kwargs):
        self.activation_mode = "ACTIVATION_TANH"
        r = super().initialize(device=device, **kwargs)
        self.output.max_supposed = 1.7159
        return r


class ConvSigmoid(Conv):
    MAPPING = {"conv_sigmoid"}
    ACT = ACT_SIGMOID

    def initialize(self, device=None, **kwargs):
        self.activation_mode = "ACTIVATION_SIGMOID"
        r = super().initialize(device=device, **kwargs)
        self.output.max_supposed = 1.0
        return r


class ConvRELU(Conv):
    """Conv with softplus ("RELU" in znicz): f(x) = log(1 + exp(x))."""
    MAPPING = {"conv_relu"}
    ACT = ACT_RELU

    def initialize(self, device=None, **kwargs):
        self.activation_mode = "ACTIVATION_RELU"
        r = super().initialize(device=device, **kwargs)
        self.output.max_supposed = 10
        return r


class ConvStrictRELU(Conv):
    """Conv with f(x) = max(x, 0) (like Caffe)."""
    MAPPING = {"conv_str"}
    ACT = ACT_STRICT_RELU

    def initialize(self, device=None, **kwargs):
        self.activation_mode = "ACTIVATION_STRICT_RELU"
        r = super().initialize(device=device, **kwargs)
        self.output.max_supposed = 10
        return r
