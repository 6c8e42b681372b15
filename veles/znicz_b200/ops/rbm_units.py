"""Restricted Boltzmann machine units (contrastive divergence).

Parity: /root/reference/rbm_units.py (Binarization :72, IterationCounter :155,
BatchWeights :182, GradientsCalculator :261, WeightsUpdater :338, MemCpy :366,
GradientRBM :441 — CD-k Gibbs chain as a nested workflow, EvaluatorRBM :518). The numpy
paths are the reference's host statistics (``EmptyDeviceMethodsMixin`` :54-68 ran them on
the host in every backend).

H100: the whole CD-k step stays on the device. Binarization draws from a counter-based hash
of (seed, counter, element) (csrc/rbm.cu; ``binarize_twin`` is its exact numpy twin), the
batch statistics run on the GEMM and column-sum kernels, GradientsCalculator on ``axpby_2d``
and WeightsUpdater is one launch (``rbm_apply_k``), after which the forward units that read
the updated weights through a bf16 / fp8 copy rebuild it.
"""
from __future__ import annotations

import numpy

from ..core import prng
from ..core.accelerated_units import AcceleratedUnit, AcceleratedWorkflow
from ..core.memory import Array
from ..core.mutable import Bool
from ..core.normalization import NoneNormalizer
from ..core.units import Unit
from ..core.workflow import Repeater, Workflow
from ..workflow.evaluator import EvaluatorMSE
from .all2all import All2AllSigmoid
from .nn_units import Forward
from .pooling import hash_u32


def binarize_twin(p, batch_size, seed, counter):
    """The device sampler's rule in numpy: for flat index i of the first ``batch_size`` rows,
    1 when (hash_u32(seed, counter, i) >> 8) * 2^-24 < p[i] (p as fp32), else 0; the other
    rows are copied."""
    p = numpy.asarray(p, dtype=numpy.float32)
    out = p.copy()
    n = int(batch_size) * (p.size // p.shape[0])
    u = (hash_u32(seed, counter, numpy.arange(n, dtype=numpy.uint64)) >> numpy.uint32(8)).astype(
        numpy.float32) * numpy.float32(2.0 ** -24)
    out.reshape(-1)[:n] = (u < p.reshape(-1)[:n]).astype(numpy.float32)
    return out


class Binarization(AcceleratedUnit):
    """output(i, j) = 1 with probability input(i, j), else 0 (first batch_size rows).

    numpy: ``matlab_binornd`` on ``rand``. CUDA: the hash sampler of ``binarize_twin``, with a
    ``seed`` drawn from ``rand`` at initialize and a ``rng_counter`` that advances once per run;
    both are pickled, so a workflow restored from a snapshot continues the same sample stream."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.output = Array()
        self.rand = kwargs.get("rand", prng.get())
        self.seed = kwargs.get("seed")
        self.rng_counter = 0
        self.demand("input", "batch_size")

    def init_unpickled(self):
        super().init_unpickled()
        self.rng_up_ = None

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        super().initialize(device=device, **kwargs)
        if not self.output or self.output.shape != self.input.shape:
            self.output.reset(numpy.zeros_like(self.input.mem))
        # 0 / 1 are exact in bf16: a bf16 sample keeps the next GEMM on the tensor cores (and the
        # device copy a consumer makes of a host sample matches the device units around it)
        self.output.dev_dtype = self.input.dev_dtype
        if self.on_cuda and self.seed is None:
            self.seed = int(self.rand.randint(1, 2 ** 31 - 1))
        self.init_vectors(self.input, self.output)
        return None

    def matlab_binornd(self, n, p_in):
        """Sum of ``n`` Bernoulli(p) draws per element (MATLAB ``binornd``)."""
        p = numpy.asarray(p_in)
        f = self.rand.rand(n, *p.shape)
        return (f < p[None]).sum(axis=0).astype(p.dtype)

    def numpy_run(self):
        self.output.map_invalidate()
        self.input.map_read()
        bs = int(self.batch_size)
        self.output.mem[...] = self.input.mem
        self.output.mem[:bs] = self.matlab_binornd(1, self.input.mem[:bs])

    def cuda_prepare(self):
        if self.rng_up_ is None:
            import torch
            from ..core.memory import ScalarUploader
            self.rng_up_ = ScalarUploader(self.device, 2, torch.int32)
        self.rng_up_.upload((self.seed & 0x7FFFFFFF, self.rng_counter & 0x7FFFFFFF))
        self.rng_counter += 1

    def cuda_run(self):
        from ..kernels import api
        api.rbm_sample(self)


class BinarizationGradH(Binarization):
    pass


class BinarizationGradV(Binarization):
    pass


class BinarizationEval(Binarization):
    pass


class IterationCounter(Unit):
    """Counts iterations of a nested loop; ``complete`` after ``max_iterations``."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.max_iterations = kwargs["max_iterations"]
        self.iteration = 0
        self.complete = Bool(False)

    def reset(self):
        self.iteration = 0
        self.complete <<= self.iteration > self.max_iterations

    def initialize(self, **kwargs):
        self.complete <<= self.iteration > self.max_iterations

    def run(self):
        self.iteration += 1
        self.complete <<= self.iteration > self.max_iterations


class BatchWeights(AcceleratedUnit):
    """<v hᵀ>, <v>, <h> over the minibatch."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.vbias_batch = Array()
        self.hbias_batch = Array()
        self.weights_batch = Array()
        self.demand("v", "h", "batch_size")

    def initialize(self, device=None, **kwargs):
        if not self.v or not self.h:
            return True
        super().initialize(device=device, **kwargs)
        vsz = self.v.size // self.v.shape[0]
        hsz = self.h.size // self.h.shape[0]
        if not self.hbias_batch:
            self.hbias_batch.reset(numpy.zeros((1, hsz), dtype=self.h.dtype))
        if not self.vbias_batch:
            self.vbias_batch.reset(numpy.zeros((1, vsz), dtype=self.h.dtype))
        if not self.weights_batch:
            self.weights_batch.reset(numpy.zeros((vsz, hsz), dtype=self.h.dtype))
        self.init_vectors(self.weights_batch, self.hbias_batch, self.vbias_batch)
        return None

    def numpy_run(self):
        self.v.map_read()
        self.h.map_read()
        bs = int(self.batch_size)
        v = self.v.matrix[:bs]
        h = self.h.matrix[:bs]
        for a in (self.weights_batch, self.hbias_batch, self.vbias_batch):
            a.map_invalidate()
        self.weights_batch.mem[...] = v.T.dot(h) / bs
        self.vbias_batch.mem[...] = v.sum(axis=0, keepdims=True) / bs
        self.hbias_batch.mem[...] = h.sum(axis=0, keepdims=True) / bs

    def cuda_run(self):
        from ..kernels import api
        api.rbm_batch_stats(self)


class BatchWeights2(BatchWeights):
    pass


class GradientsCalculator(AcceleratedUnit):
    """grad = positive-phase statistics − negative-phase statistics."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.vbias_grad = Array()
        self.hbias_grad = Array()
        self.weights_grad = Array()
        self.demand("hbias1", "vbias1", "hbias0", "vbias0", "weights0", "weights1")

    def initialize(self, device=None, **kwargs):
        if not self.hbias0 or not self.vbias0 or not self.weights0:
            return True
        super().initialize(device=device, **kwargs)
        for g, ref in ((self.hbias_grad, self.hbias0), (self.vbias_grad, self.vbias0),
                       (self.weights_grad, self.weights0)):
            if not g or g.shape != ref.shape:
                g.reset(numpy.zeros(ref.shape, dtype=ref.dtype))
        self.init_vectors(self.hbias_grad, self.vbias_grad, self.weights_grad)
        return None

    def numpy_run(self):
        for a in (self.hbias0, self.vbias0, self.weights0, self.hbias1, self.vbias1,
                  self.weights1):
            a.map_read()
        for a in (self.weights_grad, self.vbias_grad, self.hbias_grad):
            a.map_invalidate()
        self.vbias_grad.mem[...] = self.vbias0.mem - self.vbias1.mem
        self.hbias_grad.mem[...] = self.hbias0.mem - self.hbias1.mem
        self.weights_grad.mem[...] = self.weights0.mem - self.weights1.mem

    def cuda_run(self):
        from ..kernels import api
        api.rbm_gradients(self)


def _all_units(workflow):
    for u in workflow:
        yield u
        if isinstance(u, Workflow):
            yield from _all_units(u)


class WeightsUpdater(AcceleratedUnit):
    """weights += lr · gradᵀ; biases += lr · grad.

    The forward units that read ``weights`` (in mnist_rbm the hidden layer and the Gibbs chain's
    make_h) keep bf16 / fp8 copies of it on the device: each run rebuilds them."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.learning_rate = kwargs["learning_rate"]
        self.demand("hbias_grad", "vbias_grad", "weights_grad", "weights", "hbias", "vbias")

    def init_unpickled(self):
        super().init_unpickled()
        self.readers_ = []

    def initialize(self, device=None, **kwargs):
        super().initialize(device=device, **kwargs)
        if self.on_cuda:
            self.init_vectors(self.hbias_grad, self.vbias_grad, self.weights_grad, self.weights,
                              self.hbias, self.vbias)
        self.readers_ = [u for u in _all_units(self.workflow)
                         if isinstance(u, Forward) and u.weights is self.weights]
        return None

    def run(self):
        if self._backend_run_ is None:
            self.initialize()      # run without initialize(): the host update
        super().run()
        for fwd in self.readers_:
            if fwd.on_cuda:
                fwd.refresh_shadows()

    def numpy_run(self):
        for a in (self.hbias_grad, self.vbias_grad, self.weights_grad):
            a.map_read()
        for a in (self.weights, self.hbias, self.vbias):
            a.map_write()
        self.weights.mem += self.learning_rate * self.weights_grad.mem.transpose()
        self.hbias.mem += self.learning_rate * self.hbias_grad.mem.reshape(self.hbias.shape)
        self.vbias.mem += self.learning_rate * self.vbias_grad.mem.reshape(self.vbias.shape)
        for a in (self.weights, self.hbias, self.vbias):
            a.unmap()

    def cuda_run(self):
        from ..kernels import api
        api.rbm_apply(self)


class MemCpy(AcceleratedUnit):
    """output = copy(input) (device-to-device on CUDA)."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.output = Array()
        self.demand("input")

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        super().initialize(device=device, **kwargs)
        if not self.output or self.output.shape != self.input.shape:
            self.output.reset(numpy.zeros(self.input.shape, dtype=self.input.dtype))
            self.output.dev_dtype = self.input.dev_dtype
        self.init_vectors(self.input, self.output)
        return None

    def numpy_run(self):
        self.input.map_read()
        self.output.map_invalidate()
        numpy.copyto(self.output.mem, self.input.mem)

    def cuda_run(self):
        self.output.dev_out.copy_(self.input.dev)


class All2AllSigmoidH(All2AllSigmoid):
    MAPPING = set()
    hide_from_registry = True


class All2AllSigmoidV(All2AllSigmoid):
    MAPPING = set()
    hide_from_registry = True


class All2AllSigmoidWithForeignWeights(All2AllSigmoid):
    MAPPING = set()
    hide_from_registry = True


class GradientRBM(AcceleratedWorkflow):
    """CD-k Gibbs chain: h0 → (sample h → v → sample v → h) × k. Inputs: ``input`` (h0
    probabilities), ``weights`` [h, v], ``hbias``, ``vbias``, ``batch_size``; outputs
    ``v1`` (sampled visibles) and ``h1`` (hidden probabilities) after k steps."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.stddev = kwargs["stddev"]
        self.batch_size = -1
        self.mem_cpy = MemCpy(self)
        self.mem_cpy.link_from(self.start_point)
        self.repeater = Repeater(self)
        self.repeater.link_from(self.mem_cpy)
        self.decision = IterationCounter(self, max_iterations=kwargs["cd_k"])
        self.decision.link_from(self.repeater)
        self.bino_h = BinarizationGradH(self, rand=kwargs.get("rand_h", prng.get()))
        self.bino_h.link_attrs(self.mem_cpy, ("input", "output"))
        self.bino_h.link_from(self.decision)
        self.bino_h.gate_block = self.decision.complete
        self.make_v = All2AllSigmoidV(self, weights_stddev=self.stddev,
                                      weights_transposed=True,
                                      output_sample_shape=kwargs["v_size"])
        self.make_v.link_from(self.bino_h)
        self.make_v.link_attrs(self.bino_h, ("input", "output"))
        self.bino_v = BinarizationGradV(self, rand=kwargs.get("rand_v", prng.get()))
        self.bino_v.link_attrs(self.make_v, ("input", "output"))
        self.bino_v.link_from(self.make_v)
        self.make_h = All2AllSigmoidH(self, weights_stddev=self.stddev,
                                      output_sample_shape=kwargs["h_size"])
        self.make_h.link_attrs(self.bino_v, ("input", "output"))
        self.make_h.link_from(self.bino_v)
        self.h_back = MemCpy(self, name="h_to_chain")
        self.h_back.link_attrs(self.make_h, ("input", "output"))
        self.h_back.output = self.mem_cpy.output
        self.h_back.link_from(self.make_h)
        self.repeater.link_from(self.h_back)
        self.end_point.link_from(self.decision)
        self.end_point.gate_block = ~self.decision.complete
        self.mem_cpy.link_attrs(self, "input")
        self.bino_h.link_attrs(self, "batch_size")
        self.bino_v.link_attrs(self, "batch_size")
        self.make_v.link_attrs(self, "weights")
        self.make_v.link_attrs(self, ("bias", "vbias"))
        self.make_h.link_attrs(self, "weights")
        self.make_h.link_attrs(self, ("bias", "hbias"))
        self.link_attrs(self.make_h, "output")
        self.link_attrs(self.bino_v, ("v1", "output"))
        self.link_attrs(self.make_h, ("h1", "output"))
        self.demand("input", "weights", "hbias", "vbias", "batch_size")

    def run(self, iterations=None):
        self.decision.reset()
        return super().run()


class EvaluatorRBM(AcceleratedWorkflow):
    """Reconstruction error: binarise h, reconstruct v = σ(Wᵀh + vbias), MSE vs target."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.binarization = BinarizationEval(self, rand=kwargs.get("rand", prng.get()))
        self.binarization.link_from(self.start_point)
        self.rec = All2AllSigmoidWithForeignWeights(
            self, output_sample_shape=kwargs["bias_shape"], weights_transposed=True)
        self.rec.link_from(self.binarization)
        self.rec.link_attrs(self.binarization, ("input", "output"))
        self.mse = EvaluatorMSE(self, root=False, mean=False)
        self.mse.link_from(self.rec)
        self.mse.link_attrs(self.rec, "output")
        self.mse.normalizer = NoneNormalizer()
        self.end_point.link_from(self.mse)
        self.binarization.link_attrs(self, "input", "batch_size")
        self.rec.link_attrs(self, "weights")
        self.rec.link_attrs(self, ("bias", "vbias"))
        self.mse.link_attrs(self, "target", "batch_size")
        # the evaluator owns the visible bias (/root/reference/rbm_units.py:518-545); callers
        # may still link an external one over it
        self.vbias = Array(numpy.zeros(int(numpy.prod(kwargs["bias_shape"])),
                                       dtype=numpy.float32))
        self.demand("input", "weights", "target", "batch_size")

    @property
    def metrics(self):
        return self.mse.metrics

    @property
    def output(self):
        """The reconstruction of the visible layer."""
        return self.rec.output
