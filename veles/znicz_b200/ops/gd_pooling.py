"""Pooling backward units.

Parity: /root/reference/gd_pooling.py (GDPooling :58, GDMaxPooling :182 — also serves
stochastic and pool-depool :197-198, GDMaxAbsPooling :249, GDAvgPooling :255).
The reference has no numpy oracle for the base (:171-172); ours are vectorised.

H100: the scatter kernels skip the reference's separate memset when windows do not
overlap (every input element is written exactly once by a gather formulation) and
only fall back to zero-fill + atomics for overlapping windows.
"""
from __future__ import annotations

import numpy

from ..core.distributable import TriviallyDistributable
from . import nn_units
from .pooling import PoolingBase


class GDPooling(PoolingBase, nn_units.GradientDescentBase, TriviallyDistributable):
    MAPPING = set()
    hide_from_registry = True
    KERNEL = None

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.demand("input", "err_output", *self.POOL_ATTRS)
        for attr in self.POOL_ATTRS:
            if attr in kwargs:
                v = kwargs[attr]
                setattr(self, attr, tuple(v) if attr == "sliding" else v)

    def link_pool_attrs(self, other):
        self.link_attrs(other, *self.POOL_ATTRS)

    def initialize(self, device=None, **kwargs):
        if not self.input or not self.err_output:
            return True
        if self.err_output.size != self.output_size:
            raise ValueError("Size of err_output differs from the size computed based "
                             "on kx, ky, size of input.")
        return super().initialize(device=device, **kwargs)

    def cuda_run(self):
        from ..kernels import api
        api.pooling_backward(self)


class GDMaxPooling(GDPooling):
    MAPPING = {"max_pooling", "stochastic_pooling", "stochastic_pool_depool",
               "stochastic_abs_pool_depool"}
    KERNEL = "max"

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.input_offset = None
        self.demand("input_offset")

    def initialize(self, device=None, **kwargs):
        r = super().initialize(device=device, **kwargs)
        if r:
            return r
        if self.err_output.size != self.input_offset.size:
            raise ValueError("Shape of err_output differs from that of input_offset")
        self.init_vectors(self.input_offset)
        return None

    def numpy_run(self):
        self.err_output.map_read()
        self.input_offset.map_read()
        self.err_input.map_invalidate()
        self.err_input.mem[...] = 0
        numpy.add.at(self.err_input.mem.reshape(-1), self.input_offset.mem.ravel(),
                     self.err_output.mem.ravel())


class GDMaxAbsPooling(GDMaxPooling):
    MAPPING = {"maxabs_pooling", "stochastic_abs_pooling"}


class GDAvgPooling(GDPooling):
    MAPPING = {"avg_pooling"}
    KERNEL = "avg"

    def numpy_run(self):
        self.err_output.map_read()
        self.err_input.map_invalidate()
        ei = self.err_input.mem.reshape(self.input_nhwc)
        ei[...] = 0
        eo = self.err_output.mem.reshape(self.output_shape)
        ox, oy = self.out_sxy
        for y in range(oy):
            hy1 = y * self.sliding[1]
            hy2 = min(hy1 + self.ky, self.sy)
            for x in range(ox):
                hx1 = x * self.sliding[0]
                hx2 = min(hx1 + self.kx, self.sx)
                delta = eo[:, y, x, :] / ((hx2 - hx1) * (hy2 - hy1))
                ei[:, hy1:hy2, hx1:hx2, :] += delta[:, None, None, :]
