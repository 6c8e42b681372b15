"""Synthetic datasets of the named shapes (there is no network for real data).

Each class has a random smooth prototype; samples are prototype + noise, so the
nets actually learn (convergence tests) while shapes/dtypes match the reference
configs: MNIST 28×28×1 / 10 classes, CIFAR-10 32×32×3 / 10, ImageNet-style
227×227×3 / 1000 (the bench.py shapes).
"""
from __future__ import annotations

import numpy

from .base import TEST, VALID, TRAIN
from .fullbatch import FullBatchLoader, FullBatchLoaderMSE


def make_classification(n, shape, n_classes, seed, noise=0.5, dtype=numpy.float32,
                        prototypes=None, cover_classes=False):
    rs = numpy.random.RandomState(seed)
    if prototypes is None:
        prs = numpy.random.RandomState(seed ^ 0x5EED)
        prototypes = prs.normal(0, 1, (n_classes,) + tuple(shape)).astype(dtype)
    labels = rs.randint(0, n_classes, n).astype(numpy.int32)
    if cover_classes and n >= n_classes:
        # every class occurs: with 1000 classes and ~1000 samples plain sampling leaves ~37 % of
        # the labels unseen and the workflow sizes its softmax layer by the labels it saw
        labels[rs.permutation(n)[:n_classes]] = numpy.arange(n_classes, dtype=numpy.int32)
    data = prototypes[labels] + rs.normal(0, noise, (n,) + tuple(shape)).astype(dtype)
    return data.astype(dtype), labels, prototypes


class SyntheticImageLoader(FullBatchLoader):
    """kwargs: ``shape`` (h, w, c) or (features,), ``n_classes``, ``n_train``,
    ``n_valid``, ``n_test``, ``seed``, ``noise``."""
    MAPPING = "synthetic_image"

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.sample_shape = tuple(kwargs.get("shape", (32, 32, 3)))
        self.n_classes = kwargs.get("n_classes", 10)
        self.n_train = kwargs.get("n_train", 1000)
        self.n_valid = kwargs.get("n_valid", 200)
        self.n_test = kwargs.get("n_test", 0)
        self.seed = kwargs.get("seed", 17)
        self.noise = kwargs.get("noise", 0.5)
        self.cover_classes = kwargs.get("cover_classes", False)

    def load_data(self):
        parts_d, parts_l = [], []
        protos = None
        for i, n in ((TEST, self.n_test), (VALID, self.n_valid), (TRAIN, self.n_train)):
            self.class_lengths[i] = n
            if n:
                d, l, protos = make_classification(
                    n, self.sample_shape, self.n_classes, self.seed + 101 * i,
                    self.noise, prototypes=protos,
                    cover_classes=getattr(self, "cover_classes", False))
                parts_d.append(d)
                parts_l.append(l)
        self.original_data.reset(numpy.concatenate(parts_d).astype(self.dtype))
        self.original_labels = numpy.concatenate(parts_l).tolist()


class SyntheticMnistLoader(SyntheticImageLoader):
    MAPPING = "synthetic_mnist"

    def __init__(self, workflow, **kwargs):
        kwargs.setdefault("shape", (28, 28, 1))
        kwargs.setdefault("n_classes", 10)
        super().__init__(workflow, **kwargs)


class SyntheticCifarLoader(SyntheticImageLoader):
    MAPPING = "synthetic_cifar"

    def __init__(self, workflow, **kwargs):
        kwargs.setdefault("shape", (32, 32, 3))
        kwargs.setdefault("n_classes", 10)
        super().__init__(workflow, **kwargs)


class SyntheticImagenetLoader(SyntheticImageLoader):
    MAPPING = "synthetic_imagenet"

    def __init__(self, workflow, **kwargs):
        kwargs.setdefault("shape", (227, 227, 3))
        kwargs.setdefault("n_classes", 1000)
        kwargs.setdefault("cover_classes", True)
        super().__init__(workflow, **kwargs)


class SyntheticRegressionLoader(FullBatchLoaderMSE):
    """Inputs x ∈ R^n and smooth targets t = tanh(A x) for MSE workflows."""
    MAPPING = "synthetic_mse"

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.n_in = kwargs.get("n_in", 16)
        self.n_out = kwargs.get("n_out", 4)
        self.n_train = kwargs.get("n_train", 400)
        self.n_valid = kwargs.get("n_valid", 100)
        self.seed = kwargs.get("seed", 23)

    def load_data(self):
        rs = numpy.random.RandomState(self.seed)
        a = rs.normal(0, 1.0 / numpy.sqrt(self.n_in), (self.n_in, self.n_out))
        n = self.n_train + self.n_valid
        x = rs.normal(0, 1, (n, self.n_in)).astype(self.dtype)
        t = numpy.tanh(x.dot(a)).astype(self.dtype)
        self.class_lengths[TEST] = 0
        self.class_lengths[VALID] = self.n_valid
        self.class_lengths[TRAIN] = self.n_train
        self.original_data.reset(x)
        self.original_targets.reset(t)
        self.original_labels = []
