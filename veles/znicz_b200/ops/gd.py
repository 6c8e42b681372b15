"""Gradient descent units for the fully connected layers.

Parity: /root/reference/gd.py (GradientDescent :73, GDSoftmax :552, GDTanh :561,
GDRELU :594, GDStrictRELU :623, GDSigmoid :649):
``err_output *= f'(y)``; ``err_input = α·err_output·W + β·err_input``;
``gradW = err_outputᵀ·x``; ``gradb = Σ_batch err_output``; then the fused SGD step.
Extra numpy-only solvers of the reference (adagrad / adadelta / fast, :111,395-419)
are provided with the *intended* maths (SURVEY §9: the reference's adagrad
multiplies where it should divide).

H100 path (kernels/api.py): act-derivative is fused into the producer of the
two wgmma GEMMs' operand (one elementwise pass that also emits the column sums
= bias gradient), dgrad and wgrad GEMMs run on tensor cores, and weights+bias
are stepped by one fused update kernel (which is also the cross-GPU reduce).
"""
from __future__ import annotations

import numpy

from ..core.memory import Array, reshape
from . import nn_units
from .nn_units import (ACT_LINEAR, ACT_TANH, ACT_RELU, ACT_STRICT_RELU,
                       ACT_SIGMOID)


class GDCommon(nn_units.GradientDescentBase):
    """Solver plumbing + the numpy fused-step oracle shared by FC/conv/deconv GDs."""
    hide_from_registry = True
    MAPPING = set()
    SOLVERS = ("momentum", "adagrad", "adadelta", "fast")
    ACT = ACT_LINEAR

    def __init__(self, workflow, **kwargs):
        self._solvers = set()
        super().__init__(workflow, **kwargs)
        self.solvers = kwargs.get("solvers", set())
        self.demand("weights")
        if self.include_bias:
            self.demand("bias")
        self.variant_gradient = kwargs.get("variant_gradient", True)
        self.variant_moment_gradient = kwargs.get("variant_moment_gradient", True)
        self.last_minibatch = kwargs.get("last_minibatch", False)
        self.fast_learning_rate = kwargs.get("fast_learning_rate", 0.02)
        self.adadelta_momentum = kwargs.get("adadelta_momentum", 0.9)
        self.adadelta_adom = kwargs.get("adadelta_adom", 0.3)
        self.adadelta_epsilon = kwargs.get("adadelta_epsilon", 1e-8)
        self.adagrad_epsilon = kwargs.get("adagrad_epsilon", 1e-8)
        self.solver_state = {}

    @property
    def solvers(self):
        return self._solvers

    @solvers.setter
    def solvers(self, arr):
        arr = set(arr)
        if "adagrad" in arr and "adadelta" in arr:
            raise ValueError("adagrad and adadelta may not be combined")
        for value in arr:
            if value not in self.SOLVERS:
                raise ValueError("This solver is not supported: %s. Select one of %s."
                                 % (value, ", ".join(self.SOLVERS)))
        self._solvers = arr

    @property
    def extra_solvers(self):
        return self._solvers - {"momentum"}

    def initialize(self, device=None, **kwargs):
        if not self.input or not self.err_output:
            return True
        if self.extra_solvers:
            # host-only maths, like the reference (/root/reference/gd.py:111,395-419)
            self.force_numpy = True
        super().initialize(device=device, **kwargs)
        for s in self.extra_solvers:
            for part, ref in (("weights", self.weights), ("bias", self.bias)):
                if ref:
                    self.solver_state[(s, part)] = numpy.zeros_like(ref.mem)
                    if s == "adadelta":
                        self.solver_state[(s + "_g", part)] = numpy.zeros_like(ref.mem)
        if self.extra_solvers and not self.gradient_weights_with_moment:
            raise ValueError("Some of the solvers need moment vectors")
        return None

    # -- numpy oracle -------------------------------------------------------------------
    def moment_use(self, vec_old, grad, moment):
        if vec_old:
            if self.variant_moment_gradient:
                gradients = grad + vec_old.mem * moment
            else:
                gradients = (1 - moment) * grad + vec_old.mem * moment
            vec_old.mem[:] = gradients
            return gradients
        return grad

    def numpy_update(self, s):
        is_bias = s == "bias"
        vec = self.bias if is_bias else self.weights
        grad_vec = self.gradient_bias if is_bias else self.gradient_weights
        acc_vec = self.accumulated_gradient_bias if is_bias \
            else self.accumulated_gradient_weights
        vec_old = self.gradient_bias_with_moment if is_bias \
            else self.gradient_weights_with_moment
        for a in (vec, acc_vec, vec_old):
            if a:
                a.map_write()
        grad_vec.map_read()
        dp = self.dp_
        if dp is not None and dp.world_size > 1:
            # host-side counterpart of the fused cross-GPU reduction: sum over ranks
            grad_vec.map_write()
            dp.all_reduce_numpy(grad_vec.mem)
        lr = self.learning_rate_bias if is_bias else self.learning_rate
        factor_l12 = self.weights_decay_bias if is_bias else self.weights_decay
        l1_vs_l2 = self.l1_vs_l2_bias if is_bias else self.l1_vs_l2
        moment = self.gradient_moment_bias if is_bias else self.gradient_moment
        f_ortho = 0 if is_bias else self.factor_ortho
        v_trans = False if is_bias else self.weights_transposed
        step = nn_units.GradientDescentBase.numpy_gradient_step
        if self.variant_gradient:
            gradient = -step(vec.mem, grad_vec.mem, lr, factor_l12, l1_vs_l2,
                             f_ortho, v_trans)
            gradient = self.accumulate_gradient_f(acc_vec, gradient)
            gradient = self.moment_use(vec_old, gradient, moment)
        else:
            gradient = self.accumulate_gradient_f(acc_vec, grad_vec.mem.copy())
            gradient = self.moment_use(vec_old, gradient, moment)
            gradient = -step(vec.mem, gradient, lr, factor_l12, l1_vs_l2,
                             f_ortho, v_trans)
        if "adagrad" in self.solvers:
            h = self.solver_state[("adagrad", s)]
            h += gradient ** 2
            gradient = gradient / numpy.sqrt(h + self.adagrad_epsilon)
        if "adadelta" in self.solvers:
            eg = self.solver_state[("adadelta_g", s)]
            ed = self.solver_state[("adadelta", s)]
            rho = self.adadelta_momentum
            eg *= rho
            eg += (1 - rho) * gradient ** 2
            gradient = gradient * numpy.sqrt(ed + self.adadelta_epsilon) / \
                numpy.sqrt(eg + self.adadelta_epsilon)
            ed *= rho
            ed += (1 - rho) * gradient ** 2
        if "fast" in self.solvers:
            f = self.solver_state[("fast", s)]
            f *= 0.95
            if vec_old:
                f += self.fast_learning_rate * vec_old.mem
        if self.apply_gradient:
            vec.mem += gradient
            if "fast" in self.solvers and not v_trans:
                vec.mem -= self.solver_state[("fast", s)]

    def on_cuda_forward_shadow(self):
        fu = self.forward_unit
        return fu is not None and getattr(fu, "on_cuda", False)


class GradientDescent(GDCommon):
    """GD for :class:`All2All` (linear)."""
    MAPPING = {"all2all"}

    def numpy_weights_update(self):
        if not self.need_gradient_weights:
            return
        self.input.map_read()
        self.err_output.map_read()
        err_output = self.err_output.matrix
        inp = self.input.matrix
        self.gradient_weights.map_invalidate()
        from ..utils import mxfp8
        if mxfp8.enabled():      # reduction over the batch: quantise both operands along it
            inp, err_output = mxfp8.operand(inp, 0), mxfp8.operand(err_output, 0)
        if self.weights_transposed:
            numpy.dot(inp.transpose(), err_output, self.gradient_weights.mem)
        else:
            numpy.dot(err_output.transpose(), inp, self.gradient_weights.mem)
        self.numpy_update("weights")

    def numpy_bias_update(self):
        if not self.need_gradient_weights or not self.include_bias:
            return
        self.err_output.map_read()
        self.gradient_bias.map_invalidate()
        self.gradient_bias.mem[:] = self.err_output.matrix.sum(axis=0)
        self.numpy_update("bias")

    def numpy_err_input_update(self):
        if not self.need_err_input:
            return
        self.err_input.map_write()
        self.err_output.map_read()
        self.weights.map_read()
        err_output = self.err_output.matrix
        err_input = self.err_input.matrix
        from ..utils import mxfp8
        w = self.weights.mem.transpose() if self.weights_transposed else self.weights.mem
        bp = numpy.dot(mxfp8.operand(err_output, 1), mxfp8.operand(w, 0, tile=True))
        bp *= self.err_input_alpha
        if self.err_input_beta:
            err_input *= self.err_input_beta
            err_input += bp
        else:
            err_input[:] = bp

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
        api.fc_backward(self)


class GDSoftmax(GradientDescent):
    """Cross-entropy + softmax: the evaluator already produced dL/ds."""
    MAPPING = {"softmax"}


class GDTanh(nn_units.GradientDescentWithActivation, GradientDescent):
    """f'(s) = y² · (−0.388484177) + 1.14381894 (/root/reference/gd.py:561-591)."""
    MAPPING = {"all2all_tanh"}
    ACT = ACT_TANH


class GDRELU(nn_units.GradientDescentWithActivation, GradientDescent):
    """softplus: f'(s) = 1 − exp(−y)."""
    MAPPING = {"all2all_relu"}
    ACT = ACT_RELU


class GDStrictRELU(nn_units.GradientDescentWithActivation, GradientDescent):
    """f'(s) = [y > 0]."""
    MAPPING = {"all2all_str"}
    ACT = ACT_STRICT_RELU


class GDSigmoid(nn_units.GradientDescentWithActivation, GradientDescent):
    """f'(s) = y (1 − y)."""
    MAPPING = {"all2all_sigmoid"}
    ACT = ACT_SIGMOID
