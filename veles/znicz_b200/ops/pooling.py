"""Pooling forward units (NHWC, ceil-mode windows).

Parity: /root/reference/pooling.py (PoolingBase :67 ``out_sxy`` ceil-mode :97-106,
Pooling :122, OffsetPooling :249 ``input_offset`` int32, MaxPooling :333,
MaxAbsPooling :343, StochasticPooling :442, StochasticAbsPooling :462,
StochasticPoolingDepooling :485, StochasticAbsPoolingDepooling :508, AvgPooling :522).

* windows may be partial at the right/bottom border (ceil mode);
* max / maxabs / stochastic record the flat input offset of the chosen element;
* stochastic pooling picks an index with probability ∝ max(v, 0) (or |v|); when the
  window sum is 0 a uniformly random index is taken; randoms are 16-bit;
* avg pooling divides by the *clipped* window size.

H100: one thread handles 8 channels of one output pixel (NHWC ⇒ channels contiguous,
16-byte loads); randomness is a counter-based hash of (seed, step, element) computed
in-kernel, reproduced bit-exactly by the numpy oracle below (no state arrays, unlike
the reference's xorshift128+ buffers).
"""
from __future__ import annotations

import numpy

from ..core import prng
from ..core.distributable import TriviallyDistributable
from ..core.memory import Array
from ..core.units import Unit
from . import nn_units


def hash_u32(seed, counter, idx):
    """Counter-based 32-bit hash shared with csrc/common.cuh::hash_u32 (murmur3 fmix
    over a Weyl-mixed key). ``idx`` may be a numpy array."""
    with numpy.errstate(over="ignore"):
        x = (numpy.asarray(idx, dtype=numpy.uint64) * numpy.uint64(0x9E3779B1) +
             numpy.uint64(seed & 0xFFFFFFFF) +
             numpy.uint64(counter & 0xFFFFFFFF) * numpy.uint64(0x85EBCA77))
        x = (x & numpy.uint64(0xFFFFFFFF)).astype(numpy.uint32)
        x ^= x >> numpy.uint32(16)
        x = (x.astype(numpy.uint64) * numpy.uint64(0x85EBCA6B) &
             numpy.uint64(0xFFFFFFFF)).astype(numpy.uint32)
        x ^= x >> numpy.uint32(13)
        x = (x.astype(numpy.uint64) * numpy.uint64(0xC2B2AE35) &
             numpy.uint64(0xFFFFFFFF)).astype(numpy.uint32)
        x ^= x >> numpy.uint32(16)
    return x


class PoolingBase(Unit):
    POOL_ATTRS = ("kx", "ky", "sliding")
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._out_sxy = tuple()

    @property
    def output_shape(self):
        return self.input_batch_size, self.out_sy, self.out_sx, self.n_channels

    @property
    def output_size(self):
        return int(numpy.prod(self.output_shape))

    @property
    def input_batch_size(self):
        return self.input.shape[0]

    @property
    def sy(self):
        return self.input.shape[1]

    @property
    def sx(self):
        return self.input.shape[2]

    @property
    def out_sxy(self):
        outs = [0, 0]
        for i, last in enumerate((self.sx - self.kx, self.sy - self.ky)):
            last = max(last, 0)
            outs[i] = last // self.sliding[i] + 1
            if last % self.sliding[i] != 0:
                outs[i] += 1
        return tuple(outs)

    @property
    def out_sx(self):
        return self.out_sxy[0]

    @property
    def out_sy(self):
        return self.out_sxy[1]

    @property
    def n_channels(self):
        return self.input.size // (self.input_batch_size * self.sx * self.sy)

    @property
    def input_nhwc(self):
        return (self.input_batch_size, self.sy, self.sx, self.n_channels)

    def windows(self, x, fill):
        """[n, oy, ox, ky*kx, c] window view of NHWC ``x``; out-of-image = ``fill``.
        Also returns the flat input offset of every window element (−1 outside)."""
        n, sy, sx, c = x.shape
        ky, kx = self.ky, self.kx
        slx, sly = self.sliding
        ox, oy = self.out_sxy
        py = (oy - 1) * sly + ky
        px = (ox - 1) * slx + kx
        xp = numpy.full((n, max(py, sy), max(px, sx), c), fill, dtype=x.dtype)
        xp[:, :sy, :sx] = x
        flat = numpy.full(xp.shape, -1, dtype=numpy.int64)
        flat[:, :sy, :sx] = numpy.arange(x.size, dtype=numpy.int64).reshape(x.shape)
        win = numpy.empty((n, oy, ox, ky * kx, c), dtype=x.dtype)
        off = numpy.empty((n, oy, ox, ky * kx, c), dtype=numpy.int64)
        for i in range(ky):
            for j in range(kx):
                sl = (slice(None), slice(i, i + (oy - 1) * sly + 1, sly),
                      slice(j, j + (ox - 1) * slx + 1, slx))
                win[:, :, :, i * kx + j] = xp[sl]
                off[:, :, :, i * kx + j] = flat[sl]
        return win, off


class Pooling(PoolingBase, nn_units.Forward, TriviallyDistributable):
    MAPPING = set()
    hide_from_registry = True
    KERNEL = None

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.kx = kwargs["kx"]
        self.ky = kwargs["ky"]
        self.sliding = tuple(kwargs.get("sliding") or (self.kx, self.ky))
        self.exports.extend(self.POOL_ATTRS)
        self._no_output = False

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        super().initialize(device=device, **kwargs)
        if len(self.input.shape) != 4:
            raise ValueError("%s: input must be NHWC (got shape %s)" % (
                self, self.input.shape))
        if not self._no_output:
            self.make_output(self.output_shape, self.input.dtype)
            self.output.dev_dtype = self.input.dev_dtype
            self.init_vectors(self.output)
        self.init_vectors(self.input)
        return None

    def cuda_run(self):
        from ..kernels import api
        api.pooling_forward(self)


class OffsetPooling(Pooling):
    MAPPING = set()
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.input_offset = Array()
        self.demand("input")

    def initialize(self, device=None, **kwargs):
        r = super().initialize(device=device, **kwargs)
        if r:
            return r
        shape = self.output_shape
        if not self.input_offset or self.input_offset.shape != tuple(shape):
            self.input_offset.reset(numpy.zeros(shape, dtype=numpy.int32))
        self.init_vectors(self.input_offset)
        return None

    def choose(self, win, off):
        """Return index into the window axis, shape [n, oy, ox, c]."""
        raise NotImplementedError

    def numpy_run(self):
        self.input.map_read()
        self.output.map_invalidate()
        self.input_offset.map_invalidate()
        x = self.input.mem.reshape(self.input_nhwc)
        win, off = self.windows(x, 0)
        sel = self.choose(win, off)[:, :, :, None, :]
        self.output.mem[...] = numpy.take_along_axis(win, sel, axis=3)[:, :, :, 0, :]
        self.input_offset.mem[...] = numpy.take_along_axis(off, sel, axis=3)[:, :, :, 0, :]


class MaxPoolingBase(OffsetPooling):
    MAPPING = set()
    hide_from_registry = True
    ABS = False

    def choose(self, win, off):
        v = numpy.abs(win) if self.ABS else win
        v = numpy.where(off >= 0, v, -numpy.inf)
        return v.argmax(axis=3)


class MaxPooling(MaxPoolingBase):
    MAPPING = {"max_pooling"}
    KERNEL = "max"


class MaxAbsPooling(MaxPoolingBase):
    MAPPING = {"maxabs_pooling"}
    KERNEL = "maxabs"
    ABS = True


class StochasticPoolingBase(OffsetPooling):
    MAPPING = set()
    hide_from_registry = True
    ABS = False

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.rand = kwargs.get("rand", prng.get())
        self.seed = kwargs.get("seed")
        self.rng_counter = 0

    def init_unpickled(self):
        super().init_unpickled()
        self.rng_dev_ = None
        self.rng_host_ = None

    def initialize(self, device=None, **kwargs):
        r = super().initialize(device=device, **kwargs)
        if r:
            return r
        if self.seed is None:
            self.seed = int(self.rand.randint(1, 2 ** 31 - 1))
        return None

    def random_u16(self, n):
        """16-bit random per output element for the current step."""
        idx = numpy.arange(n, dtype=numpy.uint64)
        return (hash_u32(self.seed, self.rng_counter, idx) >> numpy.uint32(16)) \
            .astype(numpy.uint32)

    def choose(self, win, off):
        n, oy, ox, k, c = win.shape
        valid = off >= 0
        v = numpy.abs(win) if self.ABS else numpy.maximum(win, 0)
        v = numpy.where(valid, v, 0).astype(numpy.float64)
        rnd = self.random_u16(n * oy * ox * c).reshape(n, oy, ox, c).astype(numpy.float64)
        vsum = v.sum(axis=3)
        pos = rnd * vsum / 65536.0
        cs = numpy.cumsum(v, axis=3)
        # first valid index with pos <= cumsum (elements outside the image never win)
        hit = (pos[:, :, :, None, :] <= cs) & valid
        sel = hit.argmax(axis=3)
        # zero-sum windows: uniformly random valid element
        cnt = valid.sum(axis=3)
        ridx = (rnd.astype(numpy.int64) * cnt) >> 16
        order = numpy.cumsum(valid, axis=3) - 1          # rank among valid elements
        pick = ((order == ridx[:, :, :, None, :]) & valid).argmax(axis=3)
        return numpy.where(vsum == 0, pick, sel)

    def numpy_run(self):
        super().numpy_run()
        self.rng_counter += 1

    def cuda_prepare(self):
        import torch
        if self.rng_dev_ is None:
            from ..core.memory import ScalarUploader
            self.rng_up_ = ScalarUploader(self.device, 2, torch.int32)
            self.rng_dev_ = self.rng_up_.dev
        self.rng_up_.upload((self.seed & 0x7FFFFFFF, self.rng_counter & 0x7FFFFFFF))
        self.rng_counter += 1


class StochasticPooling(StochasticPoolingBase):
    MAPPING = {"stochastic_pooling"}
    KERNEL = "stochastic"


class StochasticAbsPooling(StochasticPoolingBase):
    MAPPING = {"stochastic_abs_pooling"}
    KERNEL = "stochastic_abs"
    ABS = True


class StochasticPoolingDepooling(StochasticPooling):
    """Stochastic pooling + depooling in place: the winner of every window stays,
    everything else in ``input`` becomes 0; ``output`` aliases ``input``."""
    MAPPING = {"stochastic_pool_depool"}
    KERNEL = "stochastic_depool"

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._no_output = True

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        if self.sliding != (self.kx, self.ky):
            raise ValueError("pool-depool needs non-overlapping windows")
        r = super().initialize(device=device, **kwargs)
        self.output = self.input
        return r

    def numpy_run(self):
        self.input.map_write()
        self.input_offset.map_invalidate()
        x = self.input.mem.reshape(self.input_nhwc)
        win, off = self.windows(x, 0)
        sel = self.choose(win, off)[:, :, :, None, :]
        val = numpy.take_along_axis(win, sel, axis=3)[:, :, :, 0, :]
        offs = numpy.take_along_axis(off, sel, axis=3)[:, :, :, 0, :]
        self.input_offset.mem[...] = offs
        flat = self.input.mem.reshape(-1)
        flat[:] = 0
        flat[offs.ravel()] = val.ravel()
        self.rng_counter += 1


class StochasticAbsPoolingDepooling(StochasticPoolingDepooling):
    MAPPING = {"stochastic_abs_pool_depool"}
    KERNEL = "stochastic_abs_depool"
    ABS = True


class AvgPooling(Pooling):
    MAPPING = {"avg_pooling"}
    KERNEL = "avg"

    def numpy_run(self):
        self.input.map_read()
        self.output.map_invalidate()
        x = self.input.mem.reshape(self.input_nhwc)
        win, off = self.windows(x, 0)
        valid = off >= 0
        cnt = valid.sum(axis=3)
        self.output.mem[...] = numpy.where(valid, win, 0).sum(axis=3) / cnt
