"""Gradient descent units for the fully connected layers.

Parity: /root/reference/gd.py (GradientDescent :73, GDSoftmax :552, GDTanh :561,
GDRELU :594, GDStrictRELU :623, GDSigmoid :649):
``err_output *= f'(y)``; ``err_input = α·err_output·W + β·err_input``;
``gradW = err_outputᵀ·x``; ``gradb = Σ_batch err_output``; then the fused SGD step.
The reference's extra solvers (adagrad / adadelta / fast, :111,395-419, numpy-only
there) are provided with the *intended* maths (SURVEY §9: the reference's adagrad
multiplies where it should divide). :func:`solver_step` is their numpy oracle; on
the GPU they run inside the fused update kernels (csrc/update.cu::step_elem) on
per-parameter state kept in device memory.

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


# solver state arrays of one parameter tensor, by name (GDCommon.solver_state keys (name, part))
#   adagrad     h       = sum of squared steps
#   adadelta    E[dx²]  (running mean of the squared adapted steps)
#   adadelta_g  E[g²]   (running mean of the squared steps)
#   fast        f       (fast weights)
SOLVER_STATE = {"adagrad": ("adagrad",), "adadelta": ("adadelta", "adadelta_g"),
                "fast": ("fast",)}
# flag bits of the fused update kernel (GradientDescentBase.update_flags)
SOLVER_FLAGS = {"adagrad": 32, "adadelta": 64, "fast": 128}


def solver_step(weights, gradient, velocity, state, solvers, adagrad_epsilon=1e-8,
                adadelta_momentum=0.9, adadelta_epsilon=1e-8, fast_learning_rate=0.02,
                apply_gradient=True, weights_transposed=False):
    """The solver half of one update, in place on ``weights`` and the ``state`` arrays.

    ``gradient`` is the step after regularisation, accumulation and momentum (it is also what
    ``velocity`` holds when there is one; the velocity keeps that pre-solver value). Adagrad or
    adadelta rescale it, ``fast`` decays its fast weights and adds ``fast_learning_rate * velocity``,
    then ``weights += gradient`` and, for non-transposed weights, ``weights -= f``. ``state`` maps
    the names of :data:`SOLVER_STATE` to arrays shaped like the weights. Returns the final step.
    The fused update kernel (csrc/update.cu::step_elem) computes the same in the same order."""
    if "adagrad" in solvers:
        h = state["adagrad"]
        h += gradient ** 2
        gradient = gradient / numpy.sqrt(h + adagrad_epsilon)
    if "adadelta" in solvers:
        eg = state["adadelta_g"]
        ed = state["adadelta"]
        rho = adadelta_momentum
        eg *= rho
        eg += (1 - rho) * gradient ** 2
        gradient = gradient * numpy.sqrt(ed + adadelta_epsilon) / \
            numpy.sqrt(eg + adadelta_epsilon)
        ed *= rho
        ed += (1 - rho) * gradient ** 2
    if "fast" in solvers:
        f = state["fast"]
        f *= 0.95
        if velocity is not None:
            f += fast_learning_rate * velocity
    if apply_gradient:
        weights += gradient
        if "fast" in solvers and not weights_transposed:
            weights -= state["fast"]
    return gradient


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
        # marks units built by a version whose update kernels run the solvers (see initialize)
        self.solvers_on_device = True

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
        if "solvers_on_device" not in self.__dict__:
            # restored from a snapshot of an earlier version, which sent every unit with an extra
            # solver (and every RProp unit) to the host by setting force_numpy: that flag did not
            # come from the user, the unit goes back to the device
            if self.forced_host_by_solvers():
                self.force_numpy = False
            self.solvers_on_device = True
        if self.extra_solvers and not (self.variant_gradient and self.variant_moment_gradient):
            # the update kernels implement the default gradient / momentum variants only; the
            # other variants keep the host maths of the numpy oracle (as before the solvers ran
            # on the device)
            self.force_numpy = True
        super().initialize(device=device, **kwargs)
        self.init_solver_state()
        if self.extra_solvers and not self.gradient_weights_with_moment:
            raise ValueError("Some of the solvers need moment vectors")
        return None

    def init_solver_state(self):
        """One :class:`Array` per solver state tensor, kept across re-initialisation. A snapshot
        may carry the state as plain numpy arrays (the form of earlier versions): their values are
        adopted."""
        for s in self.extra_solvers:
            for part, ref in (("weights", self.weights), ("bias", self.bias)):
                if not ref:
                    continue
                for name in SOLVER_STATE[s]:
                    old = self.solver_state.get((name, part))
                    if isinstance(old, Array) and old.size == ref.size:
                        continue
                    if isinstance(old, numpy.ndarray) and old.size == ref.size:
                        arr = Array(old.reshape(ref.shape).astype(ref.dtype))
                    else:
                        arr = Array(numpy.zeros_like(ref.mem))
                    self.solver_state[(name, part)] = arr
        self.init_vectors(*self.solver_state.values())

    def forced_host_by_solvers(self):
        """Whether earlier versions forced this unit onto the host because of its solvers."""
        return bool(self.extra_solvers)

    def solver_flags(self, for_bias=False):
        f = 0
        for s in self.extra_solvers:
            f |= SOLVER_FLAGS[s]
        return f

    def solver_hyper_values(self):
        return (self.adagrad_epsilon, self.adadelta_momentum, self.adadelta_epsilon,
                self.fast_learning_rate) + (0.0,) * 4

    def solver_arrays(self, for_bias=False):
        """(s0, s1, s2) state of the fused update kernel: s0 adagrad h or adadelta E[dx²],
        s1 adadelta E[g²], s2 fast f."""
        part = "bias" if for_bias else "weights"
        get = lambda name: self.solver_state.get((name, part))  # noqa: E731
        s0 = get("adagrad") if "adagrad" in self.solvers else (
            get("adadelta") if "adadelta" in self.solvers else None)
        s1 = get("adadelta_g") if "adadelta" in self.solvers else None
        s2 = get("fast") if "fast" in self.solvers else None
        return s0, s1, s2

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
        state = {}
        for (name, part), arr in self.solver_state.items():
            if part == s:
                arr.map_write()
                state[name] = arr.mem
        solver_step(vec.mem, gradient, vec_old.mem if vec_old else None, state,
                    self.extra_solvers, self.adagrad_epsilon, self.adadelta_momentum,
                    self.adadelta_epsilon, self.fast_learning_rate, self.apply_gradient, v_trans)

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
