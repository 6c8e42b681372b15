"""Fully connected forward units: ``y = act(x · Wᵀ + b)``.

Parity: /root/reference/all2all.py (All2All :53, All2AllTanh :271, All2AllRELU :298
(softplus!), All2AllStrictRELU :320, All2AllSigmoid :343, All2AllSoftmax :370).
Weight init magnitude ``min(sqrt(C/(in+out)), 0.5)`` (:106-117,154-155); fill modes
uniform/gaussian/constant; FC weights are ``[neurons, input_size]`` and
``weights_transposed`` flips the storage to ``[input_size, neurons]``.

H100 path: one wgmma GEMM whose epilogue applies bias + activation to the
register accumulator tile (``gemm_bias_act``); softmax adds a row
kernel that also records ``max_idx``. No cuBLAS on this path.
"""
from __future__ import annotations

import numpy

from ..core.memory import Array, reshape
from . import nn_units
from .nn_units import (ACT_LINEAR, ACT_TANH, ACT_RELU, ACT_STRICT_RELU,
                       ACT_SIGMOID, ACTIVATION_CODES)


class All2All(nn_units.FullyConnectedOutput, nn_units.NNLayerBase):
    """Linear fully connected layer."""
    __id__ = "58a5eadf-ae1e-498f-bf35-7d93939c4c86"
    MAPPING = {"all2all"}
    C = 10
    ACT = ACT_LINEAR

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.activation_mode = "ACTIVATION_LINEAR"
        self.exports.append("activation_mode")
        self.demand("input", "output_sample_shape")
        self.weights_shape = None

    def get_weights_magnitude(self):
        """Range such that the activation is near its maximum when all inputs are
        at their supposed maximum."""
        vle = numpy.sqrt(self.C / (self.input.sample_size +
                                   numpy.prod(self.output_sample_shape)))
        if self.weights_filling == "gaussian":
            vle /= 3
        return vle

    def initialize(self, device=None, **kwargs):
        if not self.input:
            # two-stage init: input not allocated yet (/root/reference/all2all.py:130-152)
            if self.output_samples_number is not None and self.output_dtype is not None \
                    and self.output_sample_shape:
                if not self.output or self.output.shape != self.output_shape:
                    self.output.reset(numpy.zeros(self.output_shape, self.output_dtype))
            return True
        super().initialize(device=device, **kwargs)
        if not self.output_sample_shape:
            raise ValueError("%s: output_sample_shape is not set" % self)
        if self.weights_stddev is None:
            self.weights_stddev = min(self.get_weights_magnitude(), 0.5)
        if self.bias_stddev is None:
            self.bias_stddev = self.weights_stddev
        self.weights_shape = (self.neurons_number, self.input.sample_size)
        weights_shape_t = tuple(reversed(self.weights_shape))
        if not self.weights:
            self.weights.reset(numpy.zeros(self.weights_shape, dtype=self.input.dtype))
            self.fill_array(self.weights_filling, self.weights.mem, self.weights_stddev)
            if self.weights_transposed:
                self.weights.shape = weights_shape_t
        else:
            expect = weights_shape_t if self.weights_transposed else self.weights_shape
            if tuple(self.weights.shape) != expect:
                raise ValueError("%s: weights shape %s != expected %s" % (
                    self, self.weights.shape, expect))
        if self.include_bias:
            if not self.bias:
                self.bias.reset(numpy.zeros(self.neurons_number, self.input.dtype))
                self.fill_array(self.bias_filling, self.bias.mem, self.bias_stddev)
            elif self.bias.size != self.neurons_number:
                raise ValueError("%s: bias size mismatch" % self)
        self.make_output(self.output_shape, self.input.dtype)
        self.init_vectors(self.input, self.output, self.weights, self.bias)
        if self.on_cuda:
            self.refresh_shadows()
        return None

    # -- numpy oracle -----------------------------------------------------------------
    def numpy_linear(self):
        self.output.map_invalidate()
        self.input.map_read()
        self.weights.map_read()
        from ..utils import mxfp8
        w = self.weights.mem if self.weights_transposed else self.weights.mem.transpose()
        # (block-scaled fp8 emulation: both operands quantised along the reduction dimension)
        mem = numpy.dot(mxfp8.operand(self.input.matrix, 1), mxfp8.operand(w, 0, tile=True))
        if self.include_bias:
            self.bias.map_read()
            mem += self.bias.mem
        reshape(self.output.mem, mem.shape)[:] = mem

    def numpy_run(self):
        self.numpy_linear()
        apply_activation_numpy(self.output.mem, self.ACT)

    # -- sm_90a ------------------------------------------------------------------------
    def refresh_shadows(self):
        from ..kernels import api
        api.refresh_weight_shadows(self)

    def cuda_run(self):
        from ..kernels import api
        api.fc_forward(self)


def apply_activation_numpy(mem, act):
    if act == ACT_LINEAR:
        return
    if act == ACT_TANH:
        mem *= 0.6666
        numpy.tanh(mem, mem)
        mem *= 1.7159
    elif act == ACT_RELU:     # "RELU" in znicz = softplus
        mem[:] = numpy.where(mem > 15, mem, numpy.log(numpy.exp(numpy.minimum(mem, 15)) + 1.0))
    elif act == ACT_STRICT_RELU:
        numpy.clip(mem, 0.0, 1.0e30, mem)
    elif act == ACT_SIGMOID:
        mem[:] = 1.0 / (1.0 + numpy.exp(-mem))
    else:
        raise ValueError("unknown activation %r" % act)


class All2AllTanh(All2All):
    """f(x) = 1.7159 * tanh(0.6666 * x)."""
    __id__ = "b3a2bd5c-3c01-46ef-978a-fef22e008f31"
    A = 1.7159
    B = 0.6666
    C = 9.0
    MAPPING = {"all2all_tanh"}
    ACT = ACT_TANH

    def initialize(self, device=None, **kwargs):
        self.activation_mode = "ACTIVATION_TANH"
        retval = super().initialize(device=device, **kwargs)
        self.output.max_supposed = All2AllTanh.A
        return retval


class All2AllRELU(All2All):
    """f(x) = log(1 + exp(x)) (softplus; the reference calls it RELU)."""
    __id__ = "5b7f36d8-f8c8-4eb7-8af3-75eb3cfca3fe"
    MAPPING = {"all2all_relu"}
    ACT = ACT_RELU

    def initialize(self, device=None, **kwargs):
        self.activation_mode = "ACTIVATION_RELU"
        retval = super().initialize(device=device, **kwargs)
        self.output.max_supposed = 10
        return retval


class All2AllStrictRELU(All2All):
    """f(x) = max(x, 0)."""
    __id__ = "fe63baf0-4fe4-4cf3-bafb-ef1215bf27a8"
    MAPPING = {"all2all_str"}
    ACT = ACT_STRICT_RELU

    def initialize(self, device=None, **kwargs):
        self.activation_mode = "ACTIVATION_STRICT_RELU"
        retval = super().initialize(device=device, **kwargs)
        self.output.max_supposed = 10
        return retval


class All2AllSigmoid(All2All):
    """f(x) = 1 / (1 + exp(-x))."""
    __id__ = "a27974ec-1764-4944-925d-4862de237881"
    MAPPING = {"all2all_sigmoid"}
    C = 1
    ACT = ACT_SIGMOID

    def initialize(self, device=None, **kwargs):
        self.activation_mode = "ACTIVATION_SIGMOID"
        retval = super().initialize(device=device, **kwargs)
        self.output.supposed_max_value = 1
        return retval


class All2AllSoftmax(All2All):
    """Linear layer + row softmax; records ``max_idx`` (argmax per sample)."""
    __id__ = "420219fc-3e1a-45b1-87f8-aaa0c1540de4"
    MAPPING = {"softmax"}
    ACT = ACT_LINEAR

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.max_idx = Array()
        self.reduce_size = 256

    def initialize(self, device=None, **kwargs):
        retval = super().initialize(device=device, **kwargs)
        if retval:
            return retval
        if self.output.size // self.output.shape[0] <= 1:
            raise ValueError("Output sample size should be greater than 1 for SoftMax.")
        if not self.max_idx or self.max_idx.size != self.output.shape[0]:
            self.max_idx.reset(numpy.zeros(self.output.shape[0], dtype=numpy.int32))
        self.init_vectors(self.max_idx)
        return retval

    def make_output(self, shape, dtype):
        super().make_output(shape, dtype)
        # probabilities feed the loss: keep them fp32 on the device in every mode
        self.output.dev_dtype = None

    def numpy_apply_exp(self):
        self.output.map_write()
        self.max_idx.map_invalidate()
        out = self.output.matrix
        im = out.argmax(axis=1)
        self.max_idx.mem[:] = im
        out -= out[numpy.arange(out.shape[0]), im][:, None]
        numpy.exp(out, out)
        out /= out.sum(axis=1, keepdims=True)

    def numpy_run(self):
        self.numpy_linear()
        self.numpy_apply_exp()

    def cuda_run(self):
        from ..kernels import api
        api.fc_forward(self, softmax=True)
