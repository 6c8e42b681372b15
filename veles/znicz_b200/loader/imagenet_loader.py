"""ImageNet raw-file loaders. Parity: /root/reference/loader/imagenet_loader.py:53-208
(``ImagenetLoaderBase``) and /root/reference/tests/research/AlexNet/imagenet_workflow.py:57-129
(``ImagenetLoader``: mean subtraction, random crop + mirror for TRAIN, centre crop otherwise).

Dataset files (produced by ``utils/preparation_imagenet.py``):
  ``samples_filename``          one flat uint8 file, ``sy x sx x channels`` bytes per sample,
                                ordered TEST, VALID, TRAIN
  ``original_labels_filename``  pickle: list of (text_label, int_label) per sample
  ``count_samples_filename``    json {"test": n, "val": n, "train": n}
  ``matrixes_filename``         pickle [mean (sy, sx, c) uint8/float, rdisp (sy, sx, c)]

H100 notes: the sample file is memory-mapped; a minibatch is gathered with one fancy-index
read into the pinned staging buffer (no per-sample ``seek``/``readinto`` loop), cropping and
mirroring are vectorised over the minibatch, and ``mean``/``rdisp`` are exported for the
device-side ``MeanDispNormalizer`` unit exactly like the reference.
"""
from __future__ import annotations

import json
import os
import pickle

import numpy

from ..core.accelerated_units import host_dtype
from ..core.memory import Array
from .base import Loader, LoaderError, TEST, VALID, TRAIN


class ImagenetLoaderBase(Loader):
    MAPPING = "imagenet_loader_base"

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.mean = Array()
        self.rdisp = Array()
        self.sx = kwargs.get("sx", 256)
        self.sy = kwargs.get("sy", 256)
        self.channels = kwargs.get("channels", 3)
        self.original_labels_filename = kwargs.get("original_labels_filename")
        self.count_samples_filename = kwargs.get("count_samples_filename")
        self.matrixes_filename = kwargs.get("matrixes_filename")
        self.samples_filename = kwargs.get("samples_filename")
        self.class_keys_path = kwargs.get("class_keys_path")
        self.final_sy, self.final_sx = self.sy, self.sx
        self.has_mean_file = False
        self.class_keys = None
        if self.class_keys_path is not None:
            with open(self.class_keys_path) as fin:
                self.class_keys = json.load(fin)

    def init_unpickled(self):
        super().init_unpickled()
        self._samples_ = None
        self._label_ids_ = None

    def _data_loaded(self):
        return self._samples_ is not None

    @property
    def has_labels(self):
        return True

    def _need(self, attr, hint):
        path = getattr(self, attr)
        if path is None or not os.path.exists(path):
            raise OSError("%s %s does not exist or None. %s" % (attr, path, hint))
        return path

    def load_data(self):
        hint = "Generate it with utils/preparation_imagenet.py"
        with open(self._need("original_labels_filename", hint), "rb") as fin:
            pairs = pickle.load(fin)
        self.labels_mapping = {}
        ids = numpy.empty(len(pairs), numpy.int32)
        for i, (txt, num) in enumerate(pairs):
            self.labels_mapping[txt] = int(num)
            ids[i] = int(num)
        self._label_ids_ = ids
        n_lab = max(self.labels_mapping.values()) + 1 if self.labels_mapping else 0
        self.reversed_labels_mapping = [None] * n_lab
        for k, v in self.labels_mapping.items():
            self.reversed_labels_mapping[v] = k
        with open(self._need("count_samples_filename", hint)) as fin:
            counts = json.load(fin)
        for key, cls in (("test", TEST), ("val", VALID), ("train", TRAIN)):
            self.class_lengths[cls] = int(counts.get(key, 0))
        if sum(self.class_lengths) != len(pairs):
            raise LoaderError("Number of labels mismatches the sum of class lengths")
        sample_bytes = self.sy * self.sx * self.channels
        path = self._need("samples_filename", hint)
        if os.path.getsize(path) != sample_bytes * len(pairs):
            raise LoaderError("Wrong data file size: %d bytes != %d samples x %d bytes" % (
                os.path.getsize(path), len(pairs), sample_bytes))
        self._samples_ = numpy.memmap(path, dtype=numpy.uint8, mode="r").reshape(
            len(pairs), self.sy, self.sx, self.channels)
        train_ids = ids[self.class_lengths[TEST] + self.class_lengths[VALID]:]
        self._unique_labels_count = len(numpy.unique(train_ids)) if len(train_ids) else n_lab
        if self.matrixes_filename and os.path.exists(self.matrixes_filename):
            self.load_mean()

    @property
    def unique_labels_count(self):
        return self._unique_labels_count

    def load_mean(self):
        with open(self.matrixes_filename, "rb") as fin:
            matrixes = pickle.load(fin)
        mean = numpy.asarray(matrixes[0])
        rdisp = numpy.asarray(matrixes[1]).astype(host_dtype())
        if not numpy.isfinite(rdisp).all():
            raise ValueError("rdisp matrix has NaNs or Infs")
        if mean.shape != rdisp.shape:
            raise ValueError("mean.shape != rdisp.shape")
        if mean.shape[0] != self.sy or mean.shape[1] != self.sx:
            raise ValueError("mean.shape != (%d, %d)" % (self.sy, self.sx))
        self.mean.reset(mean)
        self.rdisp.reset(rdisp)
        self.has_mean_file = True

    def create_minibatch_data(self):
        shape = (self.max_minibatch_size, self.final_sy, self.final_sx, self.channels)
        self.minibatch_data.reset(numpy.zeros(shape, dtype=host_dtype()))
        self.minibatch_labels.reset(numpy.zeros(self.max_minibatch_size, numpy.int32))
        if self.on_cuda:
            from ..ops.nn_units import torch_act_dtype
            self.minibatch_data.dev_dtype = torch_act_dtype()

    def transform_batch(self, raw):
        """uint8 [n, sy, sx, c] → what goes into ``minibatch_data`` (identity here)."""
        return raw

    def fill_minibatch(self):
        n = self.minibatch_size
        idx = numpy.sort(self.minibatch_indices.mem[:n])      # monotonic file access
        order = numpy.argsort(numpy.argsort(self.minibatch_indices.mem[:n], kind="stable"),
                              kind="stable")
        raw = self._samples_[idx][order]
        self.minibatch_data.map_invalidate()
        self.minibatch_labels.map_invalidate()
        md, ml = self.minibatch_data.mem, self.minibatch_labels.mem
        md[:n] = self.transform_batch(raw)
        md[n:] = 0
        ml[:n] = self._label_ids_[self.minibatch_indices.mem[:n]]
        ml[n:] = 0


class ImagenetLoader(ImagenetLoaderBase):
    """AlexNet-style augmentation on top of the raw loader."""
    MAPPING = "imagenet_pickle_loader"

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.crop_size_sx = kwargs.get("crop_size_sx", 224)
        self.crop_size_sy = kwargs.get("crop_size_sy", 224)
        self.mirror = kwargs.get("mirror", False)
        self.final_sy = self.crop_size_sy or self.sy
        self.final_sx = self.crop_size_sx or self.sx

    def transform_batch(self, raw):
        n = raw.shape[0]
        x = raw.astype(host_dtype())
        if self.has_mean_file:
            x -= self.mean.mem.astype(x.dtype)
        cy, cx = self.final_sy, self.final_sx
        if (cy, cx) != (self.sy, self.sx):
            if self.minibatch_class == TRAIN:
                st = self.prng.state if hasattr(self.prng, "state") else numpy.random
                hs = st.randint(0, self.sy - cy + 1, n)
                ws = st.randint(0, self.sx - cx + 1, n)
            else:
                hs = numpy.full(n, (self.sy - cy) // 2)
                ws = numpy.full(n, (self.sx - cx) // 2)
            rows = hs[:, None] + numpy.arange(cy)[None, :]
            cols = ws[:, None] + numpy.arange(cx)[None, :]
            x = x[numpy.arange(n)[:, None, None], rows[:, :, None], cols[:, None, :]]
        if self.mirror and self.minibatch_class == TRAIN:
            st = self.prng.state if hasattr(self.prng, "state") else numpy.random
            flip = st.randint(0, 2, n).astype(bool)
            x[flip] = x[flip][:, :, ::-1]
        return x
