"""Base classes of the neural-network units + the layer registry.

Capability parity with /root/reference/nn_units.py (Forward :119, NNLayerBase :214,
FullyConnectedOutput :248, GradientDescentWithActivation :299,
GradientDescentBase :339-724, NNWorkflow :727, NNSnapshotter* :808-854), written
fresh for the H100 engine:

* the SGD step (L1/L2 mix, orthogonality term, gradient accumulation, momentum,
  apply) is ONE fused kernel for weights and one for bias on the device
  (``fused_update``), which in data-parallel mode also performs the cross-GPU
  gradient reduction through peer memory (see ``veles.znicz_b200.parallel``);
* hyper-parameters live in a small device tensor so a captured CUDA graph keeps
  working while ``LearningRateAdjust`` rewrites them every minibatch;
* master weights are fp32; when the compute type is bf16 the update kernel also
  emits the bf16 shadow copy used by the tensor-core GEMMs.
"""
from __future__ import annotations

import gc
import logging
import time

import numpy

from ..core import prng
from ..core.accelerated_units import AcceleratedUnit, AcceleratedWorkflow
from ..core.config import root
from ..core.distributable import IDistributable
from ..core.memory import Array, roundup, reshape_transposed
from ..core.mutable import Bool
from ..core.registry import Match, MatchingObject
from ..core.snapshotter import SnapshotterBase, SnapshotterToFile, SnapshotterToDB
from ..core.workflow import Repeater

# activation codes shared with the kernels (csrc/common.cuh)
ACT_LINEAR, ACT_TANH, ACT_RELU, ACT_STRICT_RELU, ACT_SIGMOID = 0, 1, 2, 3, 4
ACTIVATION_CODES = {
    "ACTIVATION_LINEAR": ACT_LINEAR, "ACTIVATION_TANH": ACT_TANH,
    "ACTIVATION_RELU": ACT_RELU, "ACTIVATION_STRICT_RELU": ACT_STRICT_RELU,
    "ACTIVATION_SIGMOID": ACT_SIGMOID}


def compute_dtype_name():
    return root.common.engine.get("compute_type", "fp32")


def torch_act_dtype():
    """Device dtype of activations/errors for the current compute type."""
    import torch
    return torch.bfloat16 if compute_dtype_name() in ("bf16", "fp8") else None


class ForwardBase(AcceleratedUnit, metaclass=MatchingObject):
    """Base class for forward propagation units."""
    hide_from_registry = True
    MAPPING = set()


Match.forward_base = ForwardBase


class Forward(ForwardBase):
    """Forward unit owning ``weights``/``bias``/``output``
    (/root/reference/nn_units.py:119-211)."""
    hide_from_registry = True
    MAPPING = set()

    def __init__(self, workflow, **kwargs):
        kwargs["view_group"] = kwargs.get("view_group", "WORKER")
        super().__init__(workflow, **kwargs)
        self.weights_stddev = kwargs.get("weights_stddev")
        self.bias_stddev = kwargs.get("bias_stddev", self.weights_stddev)
        self.weights_filling = kwargs.get("weights_filling", "uniform")
        self.bias_filling = kwargs.get("bias_filling", "uniform")
        self.rand = kwargs.get("rand", prng.get())
        self.weights_transposed = kwargs.get("weights_transposed", False)
        self.include_bias = kwargs.get("include_bias", True)
        self.demand("input")
        self.output = Array(shallow_pickle=True)
        self.weights = Array()
        self.bias = Array()
        self._forward_mode = False
        self.exports = ["weights", "bias", "include_bias", "weights_transposed"]

    def init_unpickled(self):
        super().init_unpickled()
        self.weights_lp_ = None     # bf16 shadow of weights (device)
        self.weights_lp_t_ = None   # transposed bf16 shadow (dgrad operand)
        self.weights_q_ = None      # fp8 codes W_q / W_qt and their scales (kernels/api.py)
        self.weights_qt_ = None
        self.weights_qs_ = None
        self.weights_qts_ = None

    # -- export ------------------------------------------------------------------------
    def package_export(self):
        data = {}
        for attr in self.exports:
            value = getattr(self, attr, None)
            if value is not None:
                if isinstance(value, Array):
                    if not value:
                        continue
                    value.map_read()
                    value = value.mem
                data[attr] = value
        return data

    @property
    def forward_mode(self):
        return self._forward_mode

    @forward_mode.setter
    def forward_mode(self, value):
        if not isinstance(value, bool):
            raise TypeError("forward_mode must be boolean (got %s)" % type(value))
        self._forward_mode = value

    def initialize(self, device=None, **kwargs):
        self.forward_mode = kwargs.get("forward_mode", self._forward_mode)
        return super().initialize(device=device, **kwargs)

    def fill_array(self, filling, array, stddev):
        if filling == "uniform":
            self.rand.fill(array, -stddev, stddev)
        elif filling == "gaussian":
            self.rand.fill_normal_real(array, 0, stddev)
        elif filling == "constant":
            array[:] = stddev
        else:
            raise ValueError("Invalid filling type %s" % filling)

    def make_output(self, shape, dtype):
        """(Re)allocate ``output`` with the compute-type device dtype."""
        if self.output and self.output.shape == tuple(shape):
            return
        self.output.reset(numpy.zeros(shape, dtype))
        self.output.dev_dtype = torch_act_dtype() if self.on_cuda else None

    def refresh_shadows(self):
        """Rebuild low-precision device copies after a host-side weight change."""
        pass

    # -- IDistributable (/root/reference/nn_units.py:178-211) ----------------------------
    def generate_data_for_slave(self, slave=None):
        if self.forward_mode:
            return None
        data = [None, None]
        if self.weights:
            self.weights.map_read()
            data[0] = self.weights.mem
        if self.bias:
            self.bias.map_read()
            data[1] = self.bias.mem
        return data

    def generate_data_for_master(self):
        return None

    def apply_data_from_master(self, data):
        if self.forward_mode or data is None:
            return
        for arr, d in ((self.weights, data[0]), (self.bias, data[1])):
            if d is None:
                continue
            if arr:
                arr.map_invalidate()
                numpy.copyto(arr.mem, d)
            else:
                arr.reset(numpy.array(d))
        if self.is_initialized and self.on_cuda:
            self.refresh_shadows()

    def apply_data_from_slave(self, data, slave=None):
        pass

    def drop_slave(self, slave=None):
        pass


class NNLayerBase(Forward):
    MAPPING = set()
    hide_from_registry = True

    def print_debug_data(self, t_start):
        if not self.logger.isEnabledFor(logging.DEBUG):
            return
        self.output.map_read()
        y = self.output.mem
        self.debug("%s: %d samples with %d weights in %.2f sec: y: min avg max: "
                   "%.6f %.6f %.6f", type(self).__name__, y.shape[0],
                   self.weights.size, time.time() - t_start,
                   y.min(), numpy.average(y), y.max())


class FullyConnectedOutput(object):
    """``output_sample_shape`` / ``output_samples_number`` / ``neurons_number``
    (/root/reference/nn_units.py:248-296)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._output_sample_shape = tuple()
        self._set_output_sample_shape(kwargs.get("output_sample_shape", tuple()))
        self.output_samples_number = kwargs.get("output_samples_number")
        self.output_dtype = kwargs.get("output_dtype")

    @property
    def output_sample_shape(self):
        return self._output_sample_shape

    @output_sample_shape.setter
    def output_sample_shape(self, value):
        if self.is_initialized:
            raise AssertionError(
                "Cannot set output_sample_shape after initialize() was called")
        self._set_output_sample_shape(value)

    def _set_output_sample_shape(self, value):
        if isinstance(value, (int, numpy.integer)):
            self._output_sample_shape = (int(value),)
        elif hasattr(value, "shape"):
            self._output_sample_shape = tuple(value.shape[1:])
        elif hasattr(value, "__iter__"):
            self._output_sample_shape = tuple(int(v) for v in value)
        else:
            raise TypeError("Unsupported output_sample_shape type: %s" % type(value))

    @property
    def output_samples_number(self):
        inp = getattr(self, "input", None)
        if inp:
            return inp.shape[0]
        return self._output_samples_number

    @output_samples_number.setter
    def output_samples_number(self, value):
        if value is not None and not isinstance(value, int):
            raise TypeError("output_samples_number must be an integer")
        self._output_samples_number = value

    @property
    def output_shape(self):
        return (self.output_samples_number,) + self.output_sample_shape

    @property
    def neurons_number(self):
        return int(numpy.prod(self.output_sample_shape))


class GradientDescentWithActivation(AcceleratedUnit):
    """Mixin: ``err_output *= f'(output)`` before the GD math
    (/root/reference/nn_units.py:299-334). ``ACT`` selects the derivative."""
    hide_from_registry = True
    ACT = ACT_LINEAR

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.demand("output")


class GradientDescentBase(AcceleratedUnit, metaclass=MatchingObject):
    """Base class for gradient descent units (/root/reference/nn_units.py:339-724)."""
    hide_from_registry = True
    MAPPING = set()
    REDUCE_SIZE = 64
    ACT = ACT_LINEAR
    # layout of the device hyper-parameter vector (csrc/update.cu::load_step_hyper); the kernel
    # reads slots from 13 on only when the flags select a solver
    HYPER_FIELDS = ("lr", "wd", "l1_vs_l2", "moment", "acc_alpha", "acc_beta",
                    "gd_alpha", "gd_beta", "factor_ortho", "lr_bias", "wd_bias",
                    "l1_vs_l2_bias", "moment_bias", "adagrad_epsilon", "adadelta_rho",
                    "adadelta_epsilon", "fast_lr", "rprop_increase", "rprop_decrease",
                    "rprop_min_lr", "rprop_max_lr", "reserved0", "reserved1", "reserved2")
    # flag bits of the fused update kernel (update_flags)
    FLAG_APPLY, FLAG_MOMENT, FLAG_ACC, FLAG_ORTHO, FLAG_TRANSPOSED = 1, 2, 4, 8, 16
    FLAG_ADAGRAD, FLAG_ADADELTA, FLAG_FAST, FLAG_RPROP = 32, 64, 128, 256

    def __init__(self, workflow, **kwargs):
        kwargs["view_group"] = kwargs.get("view_group", "TRAINER")
        super().__init__(workflow, **kwargs)
        self.err_input = Array(shallow_pickle=True)
        self.weights = None
        self.bias = None
        self.output = None
        self.demand("input", "err_output")
        self.learning_rate = kwargs.get("learning_rate", 0.01)
        self.learning_rate_bias = kwargs.get("learning_rate_bias", self.learning_rate)
        self.weights_decay = kwargs.get("weights_decay", 0.00005)
        self.weights_decay_bias = kwargs.get("weights_decay_bias", 0.0)
        self.l1_vs_l2 = kwargs.get("l1_vs_l2", 0)
        self.l1_vs_l2_bias = kwargs.get("l1_vs_l2_bias", self.l1_vs_l2)
        self.gradient_moment = kwargs.get("gradient_moment", 0)
        self.gradient_moment_bias = kwargs.get("gradient_moment_bias",
                                               self.gradient_moment)
        self.weights_transposed = kwargs.get("weights_transposed", False)
        # err_input = alpha * new_err_input + beta * err_input
        self.err_input_alpha = kwargs.get("err_input_alpha", 1.0)
        self.err_input_beta = kwargs.get("err_input_beta", 0.0)
        self.need_err_input = kwargs.get("need_err_input", True)
        self.need_gradient_weights = kwargs.get("need_gradient_weights", True)
        self.include_bias = kwargs.get("include_bias", True)
        self.factor_ortho = kwargs.get("factor_ortho", 0)
        self.col_sums = Array()
        self.gradient_weights = Array()
        self.gradient_bias = Array()
        self.accumulate_gradient = kwargs.get("accumulate_gradient", False)
        self.acc_alpha = kwargs.get("acc_alpha", 0.0)
        self.acc_beta = kwargs.get("acc_beta", 0.0)
        self.gd_alpha = kwargs.get("gd_alpha", 0.0)
        self.gd_beta = kwargs.get("gd_beta", 1.0)
        self.accumulated_gradient_weights = Array()
        self.accumulated_gradient_bias = Array()
        self.gradient_weights_with_moment = Array()
        self.gradient_bias_with_moment = Array()
        self.gradient_changed = False
        self.apply_gradient = kwargs.get(
            "apply_gradient", not (workflow.is_slave if workflow is not None else False))
        self.reduce_size = self.REDUCE_SIZE
        self.weights_shape = None
        self.forward_unit = None   # optional back-reference (shadow refresh)

    def init_unpickled(self):
        super().init_unpickled()
        self.hyper_dev_ = None
        self.hyper_host_ = None
        self.hyper_cache_ = None
        self.dp_ = None   # data-parallel context (parallel.DataParallel) or None
        self.step_ = None  # whole-network FusedStep collecting this unit's updates, or None

    @property
    def current_batch_size(self):
        batch_size = getattr(self, "batch_size", None)
        if batch_size is None:
            return self.err_output.shape[0]
        return int(batch_size)

    # -- allocation (/root/reference/nn_units.py:451-541) ----------------------------------
    def initialize(self, device=None, **kwargs):
        super().initialize(device=device, **kwargs)
        if self.weights:
            assert len(self.weights.shape) == 2
            self.weights_shape = (tuple(reversed(self.weights.shape))
                                  if self.weights_transposed else self.weights.shape)
        else:
            self.weights_shape = None
        for name in ("learning_rate", "weights_decay", "gradient_moment",
                     "learning_rate_bias", "weights_decay_bias",
                     "gradient_moment_bias"):
            if name in kwargs:
                setattr(self, name, kwargs[name])

        w_ok = self.need_gradient_weights and self.weights
        if w_ok:
            self._ensure_like(self.gradient_weights, self.weights)
            if self.accumulate_gradient:
                self._ensure_like(self.accumulated_gradient_weights, self.weights)
            if self.gradient_moment or not self.is_standalone:
                self._ensure_like(self.gradient_weights_with_moment, self.weights)
        if self.include_bias and not self.bias:
            # the forward unit was built with include_bias=False: nothing to train
            self.include_bias = False
        b_ok = self.need_gradient_weights and self.include_bias and self.bias
        if b_ok:
            self._ensure_like(self.gradient_bias, self.bias)
            if self.accumulate_gradient:
                self._ensure_like(self.accumulated_gradient_bias, self.bias)
            if self.gradient_moment_bias or not self.is_standalone:
                self._ensure_like(self.gradient_bias_with_moment, self.bias)

        dtype = self.err_output.dtype
        if self.need_err_input:
            if self.err_input:
                assert self.err_input.shape[1:] == self.input.shape[1:]
            if not self.err_input or self.err_input.shape[0] != self.input.shape[0]:
                self.err_input.reset(numpy.zeros(self.input.shape, dtype))
                self.err_input.dev_dtype = self.input.dev_dtype
        if w_ok:
            side = self.weights_shape[0]
            other = self.weights.size // side
            if self.factor_ortho:
                if not self.col_sums or self.col_sums.size != other:
                    self.col_sums.reset(numpy.zeros(other, dtype=self.weights.dtype))
            self.reduce_size = roundup(min(self.reduce_size, other), 32)
        self.init_vectors(
            self.err_output, self.weights, self.bias, self.input, self.output,
            self.err_input, self.gradient_weights, self.gradient_bias,
            self.accumulated_gradient_weights, self.accumulated_gradient_bias,
            self.gradient_weights_with_moment, self.gradient_bias_with_moment,
            self.col_sums)
        return None

    @staticmethod
    def _ensure_like(arr, ref):
        if not arr or arr.size != ref.size:
            arr.reset(numpy.zeros_like(ref.mem))

    # -- device hyper-parameters ---------------------------------------------------------
    def hyper_values(self):
        vals = (self.learning_rate, self.weights_decay, self.l1_vs_l2,
                self.gradient_moment, self.acc_alpha, self.acc_beta,
                self.gd_alpha, self.gd_beta, self.factor_ortho,
                self.learning_rate_bias, self.weights_decay_bias,
                self.l1_vs_l2_bias, self.gradient_moment_bias) + \
            tuple(self.solver_hyper_values())
        return vals + (0.0,) * (len(self.HYPER_FIELDS) - len(vals))

    # -- solvers beyond SGD + momentum (ops/gd.py, ops/rprop_gd.py) --------------------------
    def solver_hyper_values(self):
        """Hyper slots 13-20: adagrad eps, adadelta rho and eps, fast lr, RProp increase,
        decrease, min and max rate."""
        return (0.0,) * 8

    def solver_flags(self, for_bias=False):
        return 0

    def solver_arrays(self, for_bias=False):
        """Solver state Arrays (s0, s1, s2) the fused update kernel steps with the tensor."""
        return None, None, None

    def sync_hyper(self):
        """Push hyper-parameters to HBM when they changed (outside any graph)."""
        vals = self.hyper_values()
        if vals == self.hyper_cache_:
            return
        import torch
        if self.hyper_dev_ is None:
            n = len(self.HYPER_FIELDS)
            self.hyper_dev_ = torch.zeros(n, dtype=torch.float32,
                                          device=self.device.torch_device)
            # ring of pinned staging slots (per-iteration LR policies change the values every
            # step while the host runs ahead of the device: a single slot could be rewritten
            # before its queued async copy has executed)
            self.hyper_host_ = [torch.zeros(n, dtype=torch.float32).pin_memory() for _ in range(8)]
            self.__dict__["hyper_slot_"] = 0
        k = self.__dict__["hyper_slot_"] = (self.__dict__.get("hyper_slot_", 0) + 1) % 8
        host = self.hyper_host_[k]
        host.copy_(torch.tensor(vals, dtype=torch.float32))
        self.hyper_dev_.copy_(host, non_blocking=True)
        self.hyper_cache_ = vals

    def cuda_prepare(self):
        self.sync_hyper()
        if self.step_ is not None:
            self.step_.refresh_flags(self)

    def update_flags(self, for_bias=False):
        """Bit flags understood by the fused update kernel."""
        moment_arr = self.gradient_bias_with_moment if for_bias \
            else self.gradient_weights_with_moment
        acc_arr = self.accumulated_gradient_bias if for_bias \
            else self.accumulated_gradient_weights
        f = 0
        if self.apply_gradient:
            f |= 1
        if moment_arr:
            f |= 2
        if self.accumulate_gradient and acc_arr:
            f |= 4
        if self.factor_ortho and not for_bias:
            f |= 8
        if self.weights_transposed and not for_bias:
            f |= 16
        return f | self.solver_flags(for_bias)

    # -- numpy reference math (/root/reference/nn_units.py:696-719) -----------------------
    def accumulate_gradient_f(self, accumulated_gradient, gradient):
        if accumulated_gradient and self.accumulate_gradient:
            accumulated_gradient.mem[:] = (
                gradient * self.acc_alpha +
                (self.acc_beta * accumulated_gradient.mem if self.acc_beta else 0))
            gradient *= self.gd_beta
            gradient += self.gd_alpha * accumulated_gradient.mem
        return gradient

    @staticmethod
    def numpy_gradient_step(weight, gradient, lr, factor_l12, l1_vs_l2,
                            factor_ortho=0, weights_transposed=False):
        gradient = gradient.copy()
        gradient += factor_l12 * ((1.0 - l1_vs_l2) * weight +
                                  0.5 * l1_vs_l2 * numpy.sign(weight))
        if factor_ortho:
            col_sums = (reshape_transposed(weight).sum(axis=1)
                        if weights_transposed else weight.sum(axis=0))
            for i, row in enumerate(gradient):
                row += (col_sums - weight[i]) * factor_ortho / weight.shape[0]
        gradient *= lr
        return gradient

    def numpy_err_output_update(self):
        """err_output *= f'(output) for the unit's activation."""
        act = self.ACT
        if act == ACT_LINEAR:
            return
        self.output.map_read()
        self.err_output.map_write()
        y = self.output.mem
        e = self.err_output.mem
        if act == ACT_TANH:
            e *= y * y * (-0.388484177) + 1.14381894
        elif act == ACT_RELU:
            e *= 1.0 - numpy.exp(-y)
        elif act == ACT_STRICT_RELU:
            e *= numpy.greater(y, 0)
        elif act == ACT_SIGMOID:
            e *= y * (1.0 - y)

    # -- IDistributable (/root/reference/nn_units.py:644-694) -----------------------------
    def generate_data_for_slave(self, slave=None):
        return (self.learning_rate, self.weights_decay, self.gradient_moment,
                self.learning_rate_bias, self.weights_decay_bias,
                self.gradient_moment_bias)

    @staticmethod
    def fill_zeros(vector):
        if not vector:
            return
        vector.map_invalidate()
        vector.mem[:] = 0

    def apply_data_from_master(self, data):
        (self.learning_rate, self.weights_decay, self.gradient_moment,
         self.learning_rate_bias, self.weights_decay_bias,
         self.gradient_moment_bias) = data
        for v in (self.gradient_weights_with_moment, self.gradient_bias_with_moment,
                  self.gradient_weights, self.gradient_bias,
                  self.accumulated_gradient_weights, self.accumulated_gradient_bias):
            self.fill_zeros(v)

    def generate_data_for_master(self):
        if not self.gradient_changed:
            return None
        self.gradient_changed = False
        self.gradient_weights_with_moment.map_read()
        self.gradient_bias_with_moment.map_read()
        return (self.gradient_weights_with_moment.mem,
                self.gradient_bias_with_moment.mem)

    def apply_data_from_slave(self, data, slave=None):
        if self.weights:
            self.weights.map_write()
            self.gradient_weights_with_moment.map_write()
            self.gradient_weights_with_moment.mem *= self.gradient_moment
            self.gradient_weights_with_moment.mem += data[0]
            self.weights.mem += self.gradient_weights_with_moment.mem
        if self.bias:
            self.bias.map_write()
            self.gradient_bias_with_moment.map_write()
            self.gradient_bias_with_moment.mem *= self.gradient_moment_bias
            self.gradient_bias_with_moment.mem += data[1]
            self.bias.mem += self.gradient_bias_with_moment.mem

    def drop_slave(self, slave=None):
        pass

    def run(self):
        self.gradient_changed = True
        super().run()


class NNWorkflow(AcceleratedWorkflow):
    """Workflow with repeater/loader/forwards/evaluator/decision/gds slots
    (/root/reference/nn_units.py:727-805)."""
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._repeater = Repeater(self)
        self._loader = None
        self._forwards = []
        self._evaluator = None
        self._decision = None
        self._gds = []

    repeater = property(lambda self: self._repeater)
    forwards = property(lambda self: self._forwards)
    gds = property(lambda self: self._gds)

    @property
    def loader(self):
        if self._loader is None:
            raise AttributeError(
                "No loader unit currently exists. You must set it first.")
        return self._loader

    @loader.setter
    def loader(self, value):
        from ..loader.base import Loader
        from ..core.avatar import Avatar
        if not isinstance(value, (Loader, Avatar)):
            raise TypeError("Loader must be an instance of Loader")
        self._loader = value

    @property
    def decision(self):
        if self._decision is None:
            raise AttributeError(
                "No decision unit currently exists. You must set it first.")
        return self._decision

    @decision.setter
    def decision(self, value):
        from ..workflow.decision import DecisionBase
        if not isinstance(value, DecisionBase):
            raise TypeError("Decision must be an instance of DecisionBase")
        self._decision = value

    @property
    def evaluator(self):
        if self._evaluator is None:
            raise AttributeError(
                "No evaluator unit currently exists. You must set it first.")
        return self._evaluator

    @evaluator.setter
    def evaluator(self, value):
        from ..workflow.evaluator import EvaluatorBase
        if value is None:
            raise ValueError("Evaluator may not be None")
        if not isinstance(value, EvaluatorBase) and (
                not hasattr(value, "output") or "input" not in value.demanded):
            raise TypeError(
                "Evaluator must be either an EvaluatorBase or demand \"input\" and "
                "provide \"output\" (got %s)." % type(value))
        self._evaluator = value


class NNSnapshotterBase(SnapshotterBase):
    """Logs min/max/avg of every unit array and flags NaN/Inf
    (/root/reference/nn_units.py:808-846)."""
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.has_invalid_values = Bool(False)

    def _log_attr(self, unit, attr, logged):
        val = getattr(unit, attr, None)
        if val is None or not isinstance(val, Array) or not val:
            return
        val.map_read()
        mem = val.mem
        if id(mem) in logged:
            return
        bad = not numpy.isfinite(mem).all() if mem.dtype.kind == "f" else False
        self.has_invalid_values <<= bool(self.has_invalid_values) or bad
        args = ("%s: %s: min max avg: %.6f %.6f %.6f%s", type(unit).__name__, attr,
                float(mem.min()), float(mem.max()), float(numpy.average(mem)),
                " has invalid values" if bad else "")
        if bad:
            self.error(*args)
        else:
            self.debug(*args)
        logged.add(id(mem))

    def run(self):
        if not super().run():
            return False
        logged = set()
        for u in self.workflow.start_point.dependent_units():
            for attr in ("input", "weights", "bias", "output", "err_output",
                         "err_input"):
                self._log_attr(u, attr, logged)
        t0 = time.time()
        gc.collect()
        dt = time.time() - t0
        if dt > 1.0:
            self.warning("gc.collect() took %.1f sec", dt)
        return True


class NNSnapshotterToFile(NNSnapshotterBase, SnapshotterToFile):
    MAPPING = "nnfile"


class NNSnapshotterToDB(NNSnapshotterBase, SnapshotterToDB):
    MAPPING = "nnodbc"
