"""Seedable random generators (host) — parity with ``veles.prng``.

Used by the reference for weight filling (``rand.fill``, ``fill_normal_real``
/root/reference/all2all.py:119-127), loader shuffling and dropout/stochastic-pooling
seeds. Device-side randomness on H100 is counter-based (Philox-style hash of
(seed, step, element)) inside the kernels, so no per-element state arrays exist;
the host generator only provides the seeds.
"""
from __future__ import annotations

import numpy

_generators = {}


class RandomGenerator(object):
    def __init__(self, key=None, seed=None):
        self.key = key
        self._seed = None
        self.state = numpy.random.RandomState()
        if seed is not None:
            self.seed(seed)

    def seed(self, seed, dtype=None, count=None):
        if isinstance(seed, str):
            raw = numpy.fromfile(seed, dtype=dtype or numpy.int32,
                                 count=count if count is not None else 1024)
            seed = raw.astype(numpy.uint32)
        elif isinstance(seed, numpy.ndarray):
            seed = seed.astype(numpy.uint32).ravel()
        self._seed = seed
        self.state = numpy.random.RandomState(seed)
        return self

    @property
    def seed_value(self):
        return self._seed

    def fill(self, arr, vle_min=-1.0, vle_max=1.0):
        arr[...] = self.state.uniform(vle_min, vle_max, arr.shape).astype(arr.dtype)

    def fill_normal_real(self, arr, mean, stddev, clip_to_sigma=5.0):
        v = self.state.normal(mean, stddev, arr.shape)
        if clip_to_sigma:
            numpy.clip(v, mean - clip_to_sigma * stddev,
                       mean + clip_to_sigma * stddev, v)
        arr[...] = v.astype(arr.dtype)

    def normal(self, loc=0.0, scale=1.0, size=None):
        return self.state.normal(loc, scale, size)

    def rand(self, *shape):
        return self.state.rand(*shape)

    def randint(self, low, high=None, size=None):
        return self.state.randint(low, high, size)

    def random_sample(self, size=None):
        return self.state.random_sample(size)

    def shuffle(self, arr):
        self.state.shuffle(arr)

    def permutation(self, n):
        return self.state.permutation(n)

    def choice(self, a, size=None, replace=True, p=None):
        return self.state.choice(a, size, replace, p)

    def bytes(self, n):
        return self.state.bytes(n)

    def next_seed64(self):
        """A fresh 64-bit seed for a device-side counter-based stream."""
        return int(self.state.randint(0, 2 ** 31 - 1)) << 32 | int(
            self.state.randint(0, 2 ** 31 - 1))

    def __getstate__(self):
        return {"key": self.key, "seed": self._seed, "state": self.state.get_state()}

    def __setstate__(self, st):
        self.key = st["key"]
        self._seed = st["seed"]
        self.state = numpy.random.RandomState()
        self.state.set_state(st["state"])


def get(key=1):
    g = _generators.get(key)
    if g is None:
        g = _generators[key] = RandomGenerator(key, seed=1234 + int(key))
    return g


def seed_all(seed):
    for k in (1, 2):
        get(k).seed(seed + k)
