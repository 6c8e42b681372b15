"""RProp: sign-based per-weight learning rates.

Parity: /root/reference/rprop_gd.py:44-129. The reference discards the result of
``lrs * decrease_ratios`` (:87,113 — no decrease is ever applied, SURVEY §9); here the
decrease really happens. :func:`rprop_step` is the numpy oracle; on the GPU the same step
runs inside the fused update kernels (csrc/update.cu::step_elem, flag bit 256) on the
reduced gradient, with the previous gradient kept in ``gradient_weights`` /
``gradient_bias`` and the rates in ``weight_lrs`` / ``bias_lrs``.
"""
from __future__ import annotations

import numpy

from ..core.memory import Array
from .gd import GradientDescent


def rprop_step(weights, prev_gradient, lrs, gradient, increase, decrease, min_learning_rate,
               max_learning_rate, apply_gradient=True):
    """One RProp step, in place on ``weights``, ``prev_gradient`` and ``lrs``: rates grow by
    ``increase`` where the gradient kept its sign, shrink by ``decrease`` where it flipped, are
    clipped to [min, max]; ``weights -= sign(gradient) * lrs``; ``prev_gradient = gradient``.
    No learning rate, decay or momentum is involved."""
    sign = numpy.sign(gradient)
    delta = numpy.sign(prev_gradient * gradient)
    lrs *= numpy.where(delta > 0, increase, 1.0)
    lrs *= numpy.where(delta < 0, decrease, 1.0)
    numpy.clip(lrs, min_learning_rate, max_learning_rate, lrs)
    if apply_gradient:
        weights -= sign * lrs
    prev_gradient[...] = gradient


class GDRProp(GradientDescent):
    MAPPING = {"rprop_gd"}

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.initial_learning_rate = kwargs.get("initial_learning_rate", 0.01)
        self.min_learning_rate = kwargs.get("min_learning_rate", 1e-6)
        self.max_learning_rate = kwargs.get("max_learning_rate", 1.0)
        self.increase = kwargs.get("increase", 1.05)
        self.decrease = kwargs.get("decrease", 0.80)
        self.weight_lrs = Array()
        self.bias_lrs = Array()

    def initialize(self, device=None, **kwargs):
        r = super().initialize(device=device, **kwargs)
        if r:
            return r
        if self.weight_lrs.size != self.weights.size:
            self.weight_lrs.reset(numpy.full(self.weights.shape, self.initial_learning_rate,
                                             dtype=self.weights.dtype))
        if self.include_bias and self.bias and self.bias_lrs.size != self.bias.size:
            self.bias_lrs.reset(numpy.full(self.bias.shape, self.initial_learning_rate,
                                           dtype=self.bias.dtype))
        self.init_vectors(self.weight_lrs, self.bias_lrs)
        return None

    def forced_host_by_solvers(self):
        return True

    # -- fused update kernel: the RProp bit replaces the SGD step ---------------------------
    def update_flags(self, for_bias=False):
        f = self.FLAG_RPROP
        if self.apply_gradient:
            f |= self.FLAG_APPLY
        return f

    def solver_hyper_values(self):
        return (0.0,) * 4 + (self.increase, self.decrease, self.min_learning_rate,
                             self.max_learning_rate)

    def solver_arrays(self, for_bias=False):
        return (self.bias_lrs if for_bias else self.weight_lrs), None, None

    # -- numpy oracle -------------------------------------------------------------------
    def _step(self, vec, prev_grad, lrs, gradient):
        rprop_step(vec.mem, prev_grad.mem, lrs.mem, gradient, self.increase, self.decrease,
                   self.min_learning_rate, self.max_learning_rate, self.apply_gradient)

    def numpy_weights_update(self):
        if not self.need_gradient_weights:
            return
        self.input.map_read()
        self.err_output.map_read()
        self.weights.map_write()
        self.gradient_weights.map_write()
        self.weight_lrs.map_write()
        gradient = numpy.dot(self.err_output.matrix.transpose(), self.input.matrix)
        if self.weights_transposed:
            gradient = gradient.transpose()
        self._step(self.weights, self.gradient_weights, self.weight_lrs, gradient)

    def numpy_bias_update(self):
        if not self.need_gradient_weights or not self.include_bias:
            return
        self.err_output.map_read()
        self.bias.map_write()
        self.gradient_bias.map_write()
        self.bias_lrs.map_write()
        self._step(self.bias, self.gradient_bias, self.bias_lrs,
                   self.err_output.matrix.sum(axis=0))
