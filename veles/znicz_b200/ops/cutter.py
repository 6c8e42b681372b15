"""Cutter: crop an NHWC rectangle; GDCutter: its adjoint; Cutter1D: strided AXPBY.

Parity: /root/reference/cutter.py (Cutter :91, GDCutter :177, Cutter1D :263):
``padding=(left, top, right, bottom)`` is what gets cut *off*; backward = zero fill +
paste; ``Cutter1D``: ``y[:, o:o+L] = α·x[:, i:i+L] + β·y[:, o:o+L]`` (LSTM backward).
On H100 these are single strided-copy kernels (``crop_nhwc`` / ``axpby_2d``).
"""
from __future__ import annotations

import numpy

from ..core.accelerated_units import AcceleratedUnit
from ..core.memory import Array
from . import nn_units


class CutterBase(object):
    def _init_cutter(self, kwargs):
        self.padding = kwargs.get("padding", (0, 0, 0, 0))

    @property
    def padding(self):
        return self._padding

    @padding.setter
    def padding(self, value):
        if value is None:
            raise ValueError("padding may not be None")
        value = tuple(int(v) for v in value)
        if len(value) != 4:
            raise ValueError("padding must have 4 elements (left, top, right, bottom)")
        self._padding = value

    def cut_shape(self, shape):
        sh = list(shape)
        sh[2] -= self.padding[0] + self.padding[2]
        sh[1] -= self.padding[1] + self.padding[3]
        if sh[2] <= 0 or sh[1] <= 0:
            raise ValueError("Resulted output shape is empty")
        return tuple(sh)


class Cutter(nn_units.Forward, CutterBase):
    MAPPING = {"cutter"}

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._init_cutter(kwargs)
        self.exports.append("padding")

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        if len(self.input.shape) != 4:
            raise ValueError("input should have shape (n_samples, sy, sx, n_channels)")
        if self.padding[0] < 0 or self.padding[1] < 0:
            raise ValueError("padding[0], padding[1] should not be less than zero")
        super().initialize(device=device, **kwargs)
        self.output_shape = self.cut_shape(self.input.shape)
        self.make_output(self.output_shape, self.input.dtype)
        self.output.dev_dtype = self.input.dev_dtype
        self.init_vectors(self.input, self.output)
        return None

    def numpy_run(self):
        self.output.map_invalidate()
        self.input.map_read()
        l, t = self.padding[0], self.padding[1]
        sh = self.output_shape
        self.output.mem[...] = self.input.mem[:, t:t + sh[1], l:l + sh[2], :]

    def cuda_run(self):
        from ..kernels import api
        api.cutter_forward(self)


class GDCutter(nn_units.GradientDescentBase, CutterBase):
    MAPPING = {"cutter"}

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._init_cutter(kwargs)

    def initialize(self, device=None, **kwargs):
        if not self.input or not self.err_output:
            return True
        if len(self.input.shape) != 4:
            raise ValueError("input should have shape (n_samples, sy, sx, n_channels)")
        super().initialize(device=device, **kwargs)
        self.output_shape = self.cut_shape(self.input.shape)
        if self.err_output.size != int(numpy.prod(self.output_shape)):
            raise ValueError("Computed err_output size differs from an assigned one")
        return None

    def numpy_run(self):
        self.err_output.map_read()
        self.err_input.map_invalidate()
        l, t = self.padding[0], self.padding[1]
        sh = self.output_shape
        self.err_input.mem[...] = 0
        self.err_input.mem[:, t:t + sh[1], l:l + sh[2], :] = \
            self.err_output.mem.reshape(sh)

    def cuda_run(self):
        from ..kernels import api
        api.cutter_backward(self)


class Cutter1D(AcceleratedUnit):
    """y[:, oo:oo+L] = alpha * x[:, io:io+L] + beta * y[:, oo:oo+L]."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.alpha = kwargs.get("alpha")
        self.beta = kwargs.get("beta")
        self.input_offset = kwargs.get("input_offset", 0)
        self.output_offset = kwargs.get("output_offset", 0)
        self.length = kwargs.get("length")
        self.output = Array()
        self.demand("alpha", "beta", "input")

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        super().initialize(device=device, **kwargs)
        if self.length is None:
            self.length = self.input.sample_size - self.input_offset
        if not self.output or self.output.shape[0] != self.input.shape[0]:
            self.output.reset(numpy.zeros(
                (self.input.shape[0], self.output_offset + self.length),
                dtype=self.input.dtype))
            self.output.dev_dtype = self.input.dev_dtype
        elif self.output.sample_size < self.output_offset + self.length:
            raise ValueError("output is too small")
        self.init_vectors(self.input, self.output)
        return None

    def numpy_run(self):
        self.input.map_read()
        self.output.map_write()
        out = self.output.matrix[:, self.output_offset:self.output_offset + self.length]
        if self.beta:
            out *= self.beta
        else:
            out[:] = 0
        out += self.input.matrix[
            :, self.input_offset:self.input_offset + self.length] * self.alpha

    def cuda_run(self):
        from ..kernels import api
        api.cutter1d_forward(self)
