"""Evaluators: loss gradient + metrics for one minibatch.

Parity: /root/reference/evaluator.py (EvaluatorsRegistry :58, EvaluatorBase :73,
EvaluatorSoftmax :145-330, EvaluatorMSE :334-556).

Softmax: ``err = (y − onehot(label)) · (1/batch if mean)``; rows ≥ batch_size are
zeroed; labels < 0 are ignored; accumulates ``n_err[2]`` (errors, evaluated),
``confusion_matrix[C, C]`` (predicted, label) and ``max_err_output_sum``.
MSE: ``err = (y − t) · (1/batch if mean)``, per-sample (R)MSE on *denormalised*
values, ``metrics = [sum, max, min]``, optional nearest-``class_targets`` accuracy.

H100: both are multi-CTA kernels with warp-reduced metrics and atomics into the
small accumulators (the reference runs a single CTA and fills the confusion matrix
serially on thread 0, /root/reference/cuda/evaluator.jcu:82-88). The runtime
batch size and multiplier are read from a device scalar so the kernel can sit in
a captured CUDA graph.
"""
from __future__ import annotations

import numpy

from ..core.accelerated_units import AcceleratedUnit
from ..core.distributable import TriviallyDistributable
from ..core.memory import Array
from ..core.normalization import NoneNormalizer
from ..core.registry import make_registry
from ..loader.base import TEST

EvaluatorsRegistry = make_registry("evaluators", loss_key="LOSS")
EvaluatorsRegistry.evaluators = EvaluatorsRegistry.registry


class EvaluatorBase(AcceleratedUnit, TriviallyDistributable,
                    metaclass=EvaluatorsRegistry):
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        kwargs["view_group"] = kwargs.get("view_group", "EVALUATOR")
        super().__init__(workflow, **kwargs)
        self.mean = kwargs.get("mean", True)
        self.err_output = Array()
        self._merged_output = Array()
        self.demand("output", "batch_size")
        if self.testing:
            self.demand("class_lengths", "offset")

    def init_unpickled(self):
        super().init_unpickled()
        self.batch_dev_ = None
        self.batch_host_ = None
        self._batch_cache_ = None

    @property
    def mean(self):
        return self._mean

    @mean.setter
    def mean(self, value):
        if not isinstance(value, bool):
            raise TypeError("mean must be boolean (got %s)" % type(value))
        self._mean = value

    @property
    def merged_output(self):
        assert self.testing
        return self._merged_output.mem

    def initialize(self, device=None, **kwargs):
        super().initialize(device=device, **kwargs)
        dtype = self.output.dtype
        if self.testing:
            self._merged_output.reset(numpy.zeros(
                (self.class_lengths[TEST],) + tuple(self.output.shape[1:]), dtype))
            return None
        if not self.err_output or self.err_output.shape != self.output.shape:
            self.err_output.reset(numpy.zeros(self.output.shape, dtype))
        if self.on_cuda:
            from ..ops.nn_units import torch_act_dtype
            self.err_output.dev_dtype = torch_act_dtype()
        self.init_vectors(self.output, self.err_output)
        return None

    def sync_batch(self):
        """Upload (batch_size, multiplier) when changed; graph-safe scalar source."""
        import torch
        bs = int(self.batch_size)
        if bs == self._batch_cache_:
            return
        if self.batch_dev_ is None:
            self.batch_dev_ = torch.zeros(2, dtype=torch.float32,
                                          device=self.device.torch_device)
            # a ring of pinned staging slots: the host may run a few steps ahead of the device,
            # so the slot of an earlier (still queued) async copy must not be rewritten
            self.batch_host_ = [torch.zeros(2, dtype=torch.float32).pin_memory() for _ in range(8)]
            self.__dict__["batch_slot_"] = 0
        k = self.__dict__["batch_slot_"] = (self.__dict__.get("batch_slot_", 0) + 1) % 8
        host = self.batch_host_[k]
        host[0] = float(bs)
        host[1] = 1.0 / bs if self.mean else 1.0
        self.batch_dev_.copy_(host, non_blocking=True)
        self._batch_cache_ = bs

    def run(self):
        if self.testing:
            self.output.map_read()
            self.merge_output()
            return
        return super().run()

    def merge_output(self):
        self.merged_output[self.offset - self.batch_size:self.offset] = \
            self.output.mem[:self.batch_size]

    def get_metric_names(self):
        return {"Output"} if self.testing else set()

    def get_metric_values(self):
        return {"Output": self.merged_output} if self.testing else {}


class EvaluatorSoftmax(EvaluatorBase):
    MAPPING = "evaluator_softmax"
    LOSS = "softmax"

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.compute_confusion_matrix = kwargs.get("compute_confusion_matrix", True)
        self.confusion_matrix = Array()
        self.n_err = Array()
        self.max_err_output_sum = Array()
        self.class_keys = None
        self.demand("labels", "max_idx")
        if self.testing:
            self.demand("labels_mapping")

    def initialize(self, device=None, **kwargs):
        super().initialize(device=device, **kwargs)
        if self.testing:
            return None
        dtype = self.output.dtype
        if not self.n_err:
            self.n_err.reset(numpy.zeros(2, dtype=numpy.int32))
        out_size = self.output.sample_size
        if self.compute_confusion_matrix:
            if not self.confusion_matrix or \
                    self.confusion_matrix.size != out_size * out_size:
                self.confusion_matrix.reset(
                    numpy.zeros([out_size, out_size], numpy.int32))
        else:
            self.confusion_matrix.reset()
        if not self.max_err_output_sum:
            self.max_err_output_sum.reset(numpy.zeros(1, numpy.float32 if
                                                      dtype != numpy.float64 else dtype))
        self.init_vectors(self.confusion_matrix, self.n_err, self.max_idx,
                          self.labels, self.max_err_output_sum)
        return None

    def numpy_run(self):
        self.err_output.map_invalidate()
        for vec in self.output, self.max_idx, self.labels:
            vec.map_read()
        for vec in self.n_err, self.confusion_matrix, self.max_err_output_sum:
            if vec:
                vec.map_write()
        bs = int(self.batch_size)
        labels = self.labels.mem[:bs]
        out = self.output.matrix[:bs]
        err = self.err_output.matrix
        max_idx = self.max_idx.mem[:bs]
        mult = 1.0 / bs if self.mean else 1.0
        valid = labels >= 0
        e = out.copy()
        rows = numpy.nonzero(valid)[0]
        e[rows, labels[rows]] -= 1.0
        e *= mult
        e[~valid] = 0
        err[:bs] = e
        err[bs:] = 0
        if self.confusion_matrix:
            numpy.add.at(self.confusion_matrix.mem, (max_idx[rows], labels[rows]), 1)
        n_total = int(valid.sum())
        n_ok = int((max_idx[rows] == labels[rows]).sum())
        if rows.size:
            s = numpy.fabs(e[rows]).sum(axis=1).max()
            self.max_err_output_sum.mem[0] = max(self.max_err_output_sum.mem[0], s)
        self.n_err.mem[0] += n_total - n_ok
        self.n_err.mem[1] += n_total

    def cuda_prepare(self):
        self.sync_batch()

    def cuda_run(self):
        from ..kernels import api
        api.evaluate_softmax(self)

    def get_metric_values(self):
        if self.testing:
            output_labels = {}
            class_keys = getattr(self, "class_keys", None)
            for index, probs in enumerate(self.merged_output):
                max_index = int(numpy.argmax(probs))
                key = class_keys[TEST][index] if class_keys and class_keys[TEST] \
                    else index
                output_labels[key] = self.labels_mapping[max_index]
            return {"Output": output_labels}
        return {}


class EvaluatorMSE(EvaluatorBase):
    MAPPING = "evaluator_mse"
    LOSS = "mse"

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.metrics = Array()
        self.mse = Array()
        self.labels = None
        self.class_targets = None
        self.n_err = Array()
        self.root = kwargs.get("root", True)
        self.demand("target", "normalizer")

    @property
    def root(self):
        return self._root

    @root.setter
    def root(self, value):
        if not isinstance(value, bool):
            raise TypeError("root must be boolean (got %s)" % type(value))
        self._root = value

    def initialize(self, device=None, **kwargs):
        super().initialize(device=device, **kwargs)
        if self.testing:
            return None
        if self.target.size != self.output.size:
            raise ValueError("target.size != output.size (%s != %s)" %
                             (self.target.size, self.output.size))
        dtype = self.output.dtype
        if not self.metrics:
            self.metrics.reset(numpy.zeros(3, dtype=dtype))
            self.metrics.mem[2] = 1.0e30
        self.mse.reset(numpy.zeros(self.err_output.shape[0], dtype))
        if not self.n_err:
            self.n_err.reset(numpy.zeros(2, dtype=numpy.int32))
        self.init_vectors(self.n_err, self.target, self.metrics, self.mse)
        if self.class_targets:
            self.init_vectors(self.class_targets)
        if self.labels:
            self.init_vectors(self.labels)
        return None

    def denorm_coefficients(self):
        """(mul, add) per output element of ``raw = normalized*mul + add``."""
        norm = self.normalizer
        if norm is None or isinstance(norm, NoneNormalizer):
            return None
        co = norm.coefficients
        if co is None:
            raise ValueError("normalizer %s cannot be inverted on device" % norm)
        mul, add = co   # normalized = raw*mul + add  →  raw = (normalized-add)/mul
        mul = numpy.broadcast_to(numpy.asarray(mul, dtype=numpy.float64),
                                 self.output.shape[1:]).ravel()
        add = numpy.broadcast_to(numpy.asarray(add, dtype=numpy.float64),
                                 self.output.shape[1:]).ravel()
        safe = numpy.where(mul == 0, 1.0, mul)
        return (1.0 / safe).astype(numpy.float32), (-add / safe).astype(numpy.float32)

    def numpy_run(self):
        self.output.map_read()
        self.target.map_read()
        self.metrics.map_write()
        self.err_output.map_invalidate()
        self.mse.map_invalidate()
        bs = int(self.batch_size)
        err = self.err_output.matrix
        out = self.output.matrix[:bs]
        tgt = self.target.matrix[:bs]
        diff = out - tgt
        if self.normalizer is not None and not isinstance(self.normalizer, NoneNormalizer):
            shp = (bs,) + tuple(self.output.shape[1:])
            o = self.normalizer.denormalize(out.copy().reshape(shp)).reshape(bs, -1)
            t = self.normalizer.denormalize(tgt.copy().reshape(shp)).reshape(bs, -1)
            dd = o - t
        else:
            dd = diff
        mse = numpy.square(dd).sum(axis=1) / dd.shape[1]
        if self.root:
            mse = numpy.sqrt(mse)
        err[:bs] = diff / bs if self.mean else diff
        err[bs:] = 0
        self.mse.mem[:bs] = mse
        self.mse.mem[bs:] = 0
        self.metrics.mem[0] += mse.sum()
        self.metrics.mem[1] = max(self.metrics.mem[1], mse.max())
        self.metrics.mem[2] = min(self.metrics.mem[2], mse.min())
        if self.labels and self.class_targets:
            self.class_targets.map_read()
            self.labels.map_read()
            self.n_err.map_write()
            ct = self.class_targets.matrix
            labels = self.labels.mem[:bs]
            d = ((out[:, None, :] - ct[None, :, :]) ** 2).sum(axis=2)
            pred = d.argmin(axis=1)
            self.n_err.mem[0] += int((pred != labels).sum())
            self.n_err.mem[1] += bs

    def cuda_prepare(self):
        self.sync_batch()

    def cuda_run(self):
        from ..kernels import api
        api.evaluate_mse(self)

    def merge_output(self):
        out = self.output.mem[:self.batch_size]
        if self.normalizer is not None and not isinstance(self.normalizer, NoneNormalizer):
            out = self.normalizer.denormalize(out.copy())
        self.merged_output[self.offset - self.batch_size:self.offset] = out
