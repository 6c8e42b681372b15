"""Stand-alone activation units (forward + backward pairs).

Parity: /root/reference/activation.py (ActivationForward :59, ActivationBackward :126;
pairs Tanh :218/232, Sigmoid :247/259, Mul :272/342 with auto ``factor = 0.75/max|x|``
:328-335, RELU = softplus :385/403, StrictRELU :416/445, Log :477/499,
TanhLog :525/553, SinCos :589/609). Reference bugs are *not* reproduced: sigmoid is
the documented 1/(1+e^-x) (the CUDA kernel computes e^x, cuda/activation.cu:32),
StrictRELU selects from the input, Log/TanhLog work on the device.

H100: one vectorised elementwise kernel family (``act_forward`` / ``act_backward``,
16-byte accesses, bf16 or fp32 storage, fp32 math). In StandardWorkflow graphs the
activation that directly follows a conv/FC is normally folded into that GEMM's
epilogue; these units exist for the composable API.
"""
from __future__ import annotations

import numpy

from ..core.memory import Array
from .nn_units import Forward, GradientDescentBase

# kernel codes (csrc/common.cuh); 1..4 match nn_units.ACT_*
A_TANH, A_RELU, A_STRICT_RELU, A_SIGMOID, A_MUL, A_LOG, A_TANHLOG, A_SINCOS = \
    1, 2, 3, 4, 5, 6, 7, 8

TL_D, TL_A, TL_B = 3.0, 0.242528761112, 305.459953195


def act_forward_numpy(code, x, factor=1.0):
    if code == A_TANH:
        return 1.7159 * numpy.tanh(0.6666 * x)
    if code == A_RELU:
        return numpy.where(x > 15, x, numpy.log1p(numpy.exp(numpy.minimum(x, 15))))
    if code == A_STRICT_RELU:
        return numpy.maximum(x, 0)
    if code == A_SIGMOID:
        return 1.0 / (1.0 + numpy.exp(-x))
    if code == A_MUL:
        return x * factor
    if code == A_LOG:
        return numpy.log(x + numpy.sqrt(x * x + 1))
    if code == A_TANHLOG:
        ax = numpy.maximum(numpy.abs(x), 1e-30)
        big = numpy.sign(x) * numpy.log(ax * TL_B) * TL_A
        return numpy.where(numpy.abs(x) > TL_D, big, 1.7159 * numpy.tanh(0.6666 * x))
    if code == A_SINCOS:
        flat = x.reshape(-1)
        out = numpy.empty_like(flat)
        out[1::2] = numpy.sin(flat[1::2])
        out[0::2] = numpy.cos(flat[0::2])
        return out.reshape(x.shape)
    raise ValueError(code)


def act_backward_numpy(code, err, x, y, factor=1.0):
    """err_input = err · f'(·) expressed through the input x and/or output y."""
    if code == A_TANH:
        return err * (y * y * (-0.388484177) + 1.14381894)
    if code == A_RELU:
        return err * (1.0 - numpy.exp(-y))
    if code == A_STRICT_RELU:
        return err * (y > 0)
    if code == A_SIGMOID:
        return err * (y * (1.0 - y))
    if code == A_MUL:
        return err * factor
    if code == A_LOG:
        return err / numpy.sqrt(x * x + 1)
    if code == A_TANHLOG:
        ax = numpy.maximum(numpy.abs(x), 1e-30)
        return err * numpy.where(numpy.abs(x) > TL_D, TL_A / ax,
                                 y * y * (-0.388484177) + 1.14381894)
    if code == A_SINCOS:
        fe, fx = err.reshape(-1), x.reshape(-1)
        out = numpy.empty_like(fe)
        out[1::2] = fe[1::2] * numpy.cos(fx[1::2])
        out[0::2] = fe[0::2] * (-numpy.sin(fx[0::2]))
        return out.reshape(err.shape)
    raise ValueError(code)


class Activation(object):
    CODE = None
    NEEDS_INPUT = False     # backward needs x
    NEEDS_OUTPUT = True     # backward needs y


class ActivationForward(Forward, Activation):
    MAPPING = set()
    hide_from_registry = True

    def init_unpickled(self):
        super().init_unpickled()
        # set by workflow/fusion.py: the producing unit applies this activation in its own
        # kernel epilogue; this unit then only aliases ``output`` to ``input``
        self.fused_into_ = None

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        super().initialize(device=device, **kwargs)
        if self.fused_into_ is not None and self.on_cuda:
            self.output = self.input
            return None
        if self.output is self.input:       # restored from a snapshot of a fused run
            self.output = Array()
        self.make_output(self.input.shape, self.input.dtype)
        self.output.dev_dtype = self.input.dev_dtype
        self.init_vectors(self.input, self.output)
        return None

    @property
    def factor(self):
        return 1.0

    def numpy_run(self):
        self.input.map_read()
        self.output.map_invalidate()
        self.output.mem[...] = act_forward_numpy(self.CODE, self.input.mem, self.factor)

    def cuda_run(self):
        if self.fused_into_ is not None:
            return
        from ..kernels import api
        api.activation_forward(self)

    def generate_data_for_slave(self, slave=None):
        return None

    def apply_data_from_master(self, data):
        pass


class ActivationBackward(GradientDescentBase, Activation):
    """err_input = err_output · F'(output)."""
    MAPPING = set()
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.demand("output")

    def init_unpickled(self):
        super().init_unpickled()
        self.fused_into_ = None     # see ActivationForward.fused_into_

    def initialize(self, device=None, **kwargs):
        if not self.err_output or not self.input:
            return True
        if self.err_input is not None and self.err_input is self.err_output and \
                self.fused_into_ is None:
            self.err_input = Array()        # restored from a snapshot of a fused run
        r = super().initialize(device=device, **kwargs)
        if self.fused_into_ is not None and self.on_cuda:
            # the consumer GD unit multiplies by f'(y) itself: pass the error through
            self.err_input = self.err_output
        return r

    @property
    def factor(self):
        return 1.0

    def numpy_run(self):
        self.err_output.map_read()
        self.input.map_read()
        self.output.map_read()
        self.err_input.map_invalidate()
        self.err_input.mem[...] = act_backward_numpy(
            self.CODE, self.err_output.mem.reshape(self.err_input.shape),
            self.input.mem, self.output.mem.reshape(self.input.shape), self.factor)

    def cuda_run(self):
        if self.fused_into_ is not None:
            return
        from ..kernels import api
        api.activation_backward(self)

    def generate_data_for_slave(self, slave=None):
        return None

    def apply_data_from_master(self, data):
        pass

    def generate_data_for_master(self):
        return None

    def apply_data_from_slave(self, data, slave=None):
        pass


class ForwardTanh(ActivationForward):
    """y = 1.7159 · tanh(0.6666 · x)."""
    MAPPING = {"activation_tanh"}
    CODE = A_TANH


class BackwardTanh(ActivationBackward):
    MAPPING = {"activation_tanh"}
    CODE = A_TANH


class ForwardSigmoid(ActivationForward):
    """y = 1 / (1 + exp(−x))."""
    MAPPING = {"activation_sigmoid"}
    CODE = A_SIGMOID


class BackwardSigmoid(ActivationBackward):
    MAPPING = {"activation_sigmoid"}
    CODE = A_SIGMOID


class ForwardMul(ActivationForward):
    """y = k·x; k is auto-set to 0.75/max|x| on the first minibatch when not given
    (/root/reference/activation.py:328-335). Master keeps the min over slaves."""
    MAPPING = {"activation_mul"}
    CODE = A_MUL

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._factor = kwargs.get("factor")

    @property
    def factor(self):
        return self._factor

    @factor.setter
    def factor(self, value):
        self._factor = None if value is None else float(value)

    def run(self):
        if self._factor is None:
            self.input.map_read()
            mx = float(numpy.fabs(self.input.mem).max())
            dp = getattr(self, "dp_", None)
            self.factor = 0.75 / mx if mx else 0.75
            if dp is not None and dp.world_size > 1:
                self.factor = dp.all_reduce_scalar(self.factor, "min")
            self.info("Autosetting factor to %f", self.factor)
        super().run()

    def generate_data_for_slave(self, slave=None):
        return self.factor

    def apply_data_from_master(self, data):
        if data is not None and self.factor != data:
            self.factor = data

    def generate_data_for_master(self):
        return self.factor

    def apply_data_from_slave(self, data, slave=None):
        if data is None:
            return
        self.factor = data if self.factor is None else min(self.factor, data)


class BackwardMul(ActivationBackward):
    MAPPING = {"activation_mul"}
    CODE = A_MUL
    NEEDS_OUTPUT = False

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._factor = float(kwargs.get("factor", 1.0))

    @property
    def factor(self):
        return self._factor

    @factor.setter
    def factor(self, value):
        self._factor = float(value)


class ForwardRELU(ActivationForward):
    """y = log(1 + exp(x)) (softplus)."""
    MAPPING = {"activation_relu"}
    CODE = A_RELU


class BackwardRELU(ActivationBackward):
    MAPPING = {"activation_relu"}
    CODE = A_RELU


class ForwardStrictRELU(ActivationForward):
    """y = max(0, x)."""
    MAPPING = {"activation_str"}
    CODE = A_STRICT_RELU


class BackwardStrictRELU(ActivationBackward):
    MAPPING = {"activation_str"}
    CODE = A_STRICT_RELU


class ForwardLog(ActivationForward):
    """y = log(x + sqrt(x² + 1))."""
    MAPPING = {"activation_log"}
    CODE = A_LOG


class BackwardLog(ActivationBackward):
    MAPPING = {"activation_log"}
    CODE = A_LOG
    NEEDS_INPUT = True
    NEEDS_OUTPUT = False


class ForwardTanhLog(ActivationForward):
    """Hybrid: scaled tanh inside [−3, 3], ±a·log(±b·x) outside."""
    d, a, b = TL_D, TL_A, TL_B
    MAPPING = {"activation_tanhlog"}
    CODE = A_TANHLOG


class BackwardTanhLog(ActivationBackward):
    MAPPING = {"activation_tanhlog"}
    CODE = A_TANHLOG
    NEEDS_INPUT = True


class ForwardSinCos(ActivationForward):
    """y = sin(x) at odd flat indices, cos(x) at even ones."""
    MAPPING = {"activation_sincos"}
    CODE = A_SINCOS


class BackwardSinCos(ActivationBackward):
    MAPPING = {"activation_sincos"}
    CODE = A_SINCOS
    NEEDS_INPUT = True
    NEEDS_OUTPUT = False
