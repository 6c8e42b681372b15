"""Dropout (train-only inverted dropout).

Parity: /root/reference/dropout.py (Dropout :55, DropoutForward :84, DropoutBackward
:191, DropoutFixer :250): active only when ``minibatch_class == TRAIN`` and not in
``forward_mode``; mask ∈ {0, 1/(1−p)}; evaluation = device copy (:179-187).

H100: the mask comes from a counter-based hash of (seed, step, element) computed
in-kernel — no ``uint32[4n]`` xorshift state array (/root/reference/dropout.py:110-113);
the numpy path uses the same hash so both paths agree bit-for-bit.
"""
from __future__ import annotations

import numpy

from ..core import prng
from ..core.distributable import TriviallyDistributable
from ..core.memory import Array
from ..core.units import Unit
from .nn_units import Forward, GradientDescentBase
from .pooling import hash_u32

TRAIN = 2


class Dropout(object):
    def _init_dropout(self, kwargs):
        self.dropout_ratio = kwargs.get("dropout_ratio")

    @property
    def dropout_ratio(self):
        return self._dropout_ratio

    @dropout_ratio.setter
    def dropout_ratio(self, value):
        if value is not None and not 0.0 < value < 1.0:
            raise ValueError("dropout_ratio must be in (0, 1)")
        self._dropout_ratio = value


class DropoutForward(Forward, Dropout, TriviallyDistributable):
    __id__ = "c4117362-3c89-41bf-ba7d-a6b1bb0d8331"
    MAPPING = {"dropout"}

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._init_dropout(kwargs)
        self.mask = Array()
        self.rand = kwargs.get("rand", prng.get())
        self.seed = kwargs.get("seed")
        self.rng_counter = 0
        self.demand("minibatch_class")

    def init_unpickled(self):
        super().init_unpickled()
        self.rng_dev_ = None
        self.rng_host_ = None

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        super().initialize(device=device, **kwargs)
        if self.dropout_ratio is None:
            raise ValueError("%s: dropout_ratio is not set" % self)
        if self.seed is None:
            self.seed = int(self.rand.randint(1, 2 ** 31 - 1))
        if not self.mask or self.mask.shape != self.input.shape:
            self.mask.reset(numpy.zeros(self.input.shape, self.input.dtype))
            self.mask.dev_dtype = self.input.dev_dtype
        self.make_output(self.input.shape, self.input.dtype)
        self.output.dev_dtype = self.input.dev_dtype
        self.init_vectors(self.input, self.output, self.mask)
        return None

    @property
    def threshold(self):
        """Drop when hash < threshold (32-bit)."""
        return int(self.dropout_ratio * 4294967296.0)

    @property
    def active(self):
        return not self.forward_mode and self.minibatch_class == TRAIN

    def calc_mask(self):
        idx = numpy.arange(self.input.size, dtype=numpy.uint64)
        h = hash_u32(self.seed, self.rng_counter, idx)
        keep = h >= numpy.uint32(min(self.threshold, 0xFFFFFFFF))
        self.mask.mem.reshape(-1)[:] = keep.astype(self.mask.dtype) / \
            (1.0 - self.dropout_ratio)

    def numpy_run(self):
        self.output.map_invalidate()
        self.input.map_read()
        if self.active:
            self.mask.map_invalidate()
            self.calc_mask()
            numpy.multiply(self.input.mem, self.mask.mem, self.output.mem)
            self.rng_counter += 1
        else:
            self.output.mem[...] = self.input.mem

    def cuda_prepare(self):
        import torch
        if self.rng_dev_ is None:
            from ..core.memory import ScalarUploader
            self.rng_up_ = ScalarUploader(self.device, 2, torch.int32)
            self.rng_dev_ = self.rng_up_.dev
        if self.active:
            self.rng_up_.upload((self.seed & 0x7FFFFFFF, self.rng_counter & 0x7FFFFFFF))
            self.rng_counter += 1

    def cuda_run(self):
        from ..kernels import api
        api.dropout_forward(self)


class DropoutBackward(GradientDescentBase, Dropout, TriviallyDistributable):
    MAPPING = {"dropout"}

    def __init__(self, workflow, **kwargs):
        self.mask = None
        super().__init__(workflow, **kwargs)
        self._init_dropout(kwargs)
        self.undemand("input")
        self.demand("mask")

    def initialize(self, device=None, **kwargs):
        if not self.err_output:
            return True
        if getattr(self, "input", None) is None:
            self.input = self.err_output
        return super().initialize(device=device, **kwargs)

    def numpy_run(self):
        self.err_output.map_read()
        self.err_input.map_invalidate()
        self.mask.map_read()
        numpy.multiply(self.err_output.mem.reshape(self.mask.shape), self.mask.mem,
                       self.err_input.mem.reshape(self.mask.shape))

    def cuda_run(self):
        from ..kernels import api
        api.dropout_backward(self)


class DropoutFixer(Unit):
    """Switches every DropoutForward of the workflow into pass-through mode while
    a non-train minibatch is processed (/root/reference/dropout.py:250-266)."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)

    def init_unpickled(self):
        super().init_unpickled()
        self.drops_ = None

    def initialize(self, **kwargs):
        self.drops_ = [u for u in self.workflow if isinstance(u, DropoutForward)]

    def run(self):
        mode = self.workflow.loader.minibatch_class != TRAIN
        for u in self.drops_:
            u.forward_mode = bool(mode)
