"""ImageNet raw-file loaders. Parity: /root/reference/loader/imagenet_loader.py:53-208
(``ImagenetLoaderBase``) and /root/reference/tests/research/AlexNet/imagenet_workflow.py:57-129
(``ImagenetLoader``: mean subtraction, random crop + mirror for TRAIN, centre crop otherwise).

Dataset files (produced by ``utils/preparation_imagenet.py``):
  ``samples_filename``          one flat uint8 file, ``sy x sx x channels`` bytes per sample,
                                ordered TEST, VALID, TRAIN
  ``original_labels_filename``  pickle: list of (text_label, int_label) per sample
  ``count_samples_filename``    json {"test": n, "val": n, "train": n}
  ``matrixes_filename``         pickle [mean (sy, sx, c) uint8/float, rdisp (sy, sx, c)]

H100 notes: the sample file is memory-mapped, and ``mean``/``rdisp`` are exported for the
device-side ``MeanDispNormalizer`` unit exactly like the reference.

On ``numpy`` a minibatch is gathered with one fancy-index read, and cropping and mirroring are
vectorised over the minibatch. On ``cuda`` (device minibatch bf16 or fp32, ``fill_minibatch`` and
``transform_batch`` not overridden) only uint8 bytes cross PCIe and the augmentation runs in one
kernel (csrc/augment.cu), at the head of the captured forward graph:

* streamed (default): each step fills a pinned slot ``[header | labels | params | uint8 rows]``
  (parts 256-byte aligned; the rows gathered from the memmap by the native pool, the next
  minibatch's rows one step ahead), which reaches the device in one copy through the stream ring;
* ``on_device=True``: the sample file and the label ids live in HBM, a step uploads
  ``[header | indices | params]`` and the kernel gathers the rows and labels itself.

``augment_params`` draws the crops and flips with the same ``prng`` calls on both backends, so a
``numpy`` and a ``cuda`` loader with equal seeds serve the same minibatches.
"""
from __future__ import annotations

import json
import os
import pickle
import warnings

import numpy

from ..core.accelerated_units import host_dtype
from ..core.config import root
from ..core.memory import Array
from .base import Loader, LoaderError, TEST, VALID, TRAIN, channel_pad_target


def _align(nbytes):
    return (nbytes + 255) // 256 * 256


def _as_tensor(arr):
    """torch view of a (read-only) memmap: the native code only reads it."""
    import torch
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        return torch.from_numpy(numpy.asarray(arr))


class ImagenetLoaderBase(Loader):
    MAPPING = "imagenet_loader_base"
    # whether transform_batch subtracts the mean file (ImagenetLoader does, the raw loader does not)
    subtracts_mean = False
    SLOTS = 4           # pinned slots: one is filled while the copies out of the others run

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.on_device = kwargs.get("on_device", False)
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
        self._aug_ = None           # device augmentation state; None: the host path

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

    def augment_params(self, n):
        """int32 ``[n][3]`` of ``(y0, x0, flip)``: the crop origin and mirror flag of each sample
        of the current minibatch. The raw loader serves whole, unmirrored samples."""
        return numpy.zeros((n, 3), numpy.int32)

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

    # -- cuda: uint8 samples augmented on the device -------------------------------------------
    def _device_augment_ok(self):
        import torch
        md = self.minibatch_data
        cls = type(self)
        return cls.fill_minibatch is ImagenetLoaderBase.fill_minibatch and \
            cls.transform_batch in (ImagenetLoaderBase.transform_batch,
                                    ImagenetLoader.transform_batch) and \
            md.mem.dtype == numpy.float32 and md.devmem is not None and \
            md.devmem.dtype in (torch.float32, torch.bfloat16)

    def fill_indices(self, start, count):
        super().fill_indices(start, count)
        return self._aug_ is not None       # the minibatch is assembled in _cuda_serve

    def _cuda_setup(self):
        self.init_vectors(self.minibatch_data, self.minibatch_labels, self.minibatch_indices)
        if not self._device_augment_ok():
            return super()._cuda_setup()
        import torch
        dev = self.device.torch_device
        ext = self.device.ext
        md, ml = self.minibatch_data, self.minibatch_labels
        mb = self.max_minibatch_size
        shape = tuple(self._samples_.shape[1:])
        aug = {"mean": None, "i": 0, "pending": None, "used": [False] * self.SLOTS}
        if self.subtracts_mean and self.has_mean_file:
            aug["mean"] = torch.from_numpy(
                numpy.ascontiguousarray(self.mean.mem, dtype=numpy.float32)).to(dev)
        # part offsets: header 16 B, then [labels | params | rows] streamed or [indices | params]
        off = {"hdr": 0}
        end = 16
        for name, nbytes in ((("idx", 4 * mb), ("par", 12 * mb)) if self.on_device else
                             (("lab", 4 * mb), ("par", 12 * mb),
                              ("rows", mb * self._samples_[0].nbytes))):
            off[name] = _align(end)
            end = off[name] + nbytes
        total = _align(end)

        def views(buf):
            v = {"hdr": buf[:16].view(torch.int32),
                 "par": buf[off["par"]:off["par"] + 12 * mb].view(torch.int32).view(mb, 3)}
            if self.on_device:
                v["idx"] = buf[off["idx"]:off["idx"] + 4 * mb].view(torch.int32)
            else:
                v["lab"] = buf[off["lab"]:off["lab"] + 4 * mb].view(torch.int32)
                v["rows"] = buf[off["rows"]:off["rows"] + mb * self._samples_[0].nbytes] \
                    .view((mb,) + shape)
            return v
        aug["dev"] = torch.zeros(total, dtype=torch.uint8, device=dev)
        aug["dv"] = views(aug["dev"])
        aug["slots"] = []
        for _ in range(self.SLOTS):
            pin = torch.zeros(total, dtype=torch.uint8).pin_memory()
            v = views(pin)
            sl = {"pin": pin, "event": torch.cuda.Event(), "rows": v.get("rows")}
            sl.update({k: v[k].numpy() for k in ("hdr", "par", "idx", "lab") if k in v})
            aug["slots"].append(sl)
        self.header_dev_ = aug["dv"]["hdr"]
        if self.on_device:
            aug["src"], aug["labels"] = self._upload_dataset()
        else:
            aug["src"] = aug["dv"]["rows"]
            aug["host_src"] = _as_tensor(self._samples_)
            ml._devmem_ = aug["dv"]["lab"].view(tuple(ml.shape))
            aug["stage"] = [torch.zeros_like(aug["dev"]) for _ in range(3)]
            aug["ring"] = int(ext.stream_ring_create(len(aug["stage"]), self.SLOTS))
            aug["prefetch"] = bool(root.common.engine.get("loader_prefetch", True))
        self._aug_ = aug
        self.h2d_bytes_per_step = total

    def _upload_dataset(self):
        """The uint8 sample file and the label ids → HBM, once (``on_device=True``)."""
        import torch
        dev = self.device.torch_device
        samples, labels = self._samples_, self._label_ids_
        need = samples.nbytes + labels.nbytes
        free = torch.cuda.mem_get_info(dev)[0]
        if need > free:
            raise LoaderError(
                "on_device: the %d-byte sample file and %d bytes of labels do not fit in the %d "
                "bytes free on %s" % (samples.nbytes, labels.nbytes, free, dev))
        try:
            data = torch.empty(samples.shape, dtype=torch.uint8, device=dev)
        except torch.cuda.OutOfMemoryError as exc:
            raise LoaderError("on_device: cannot allocate %d bytes for the sample file: %s" % (
                samples.nbytes, exc)) from exc
        step = max(1, (256 << 20) // max(samples[0].nbytes, 1))
        for a in range(0, len(samples), step):
            data[a:a + step].copy_(_as_tensor(samples[a:a + step]))
        return data, torch.from_numpy(labels).to(dev)

    def _cuda_begin_step(self):
        if self._aug_ is None:
            super()._cuda_begin_step()

    def _slot_done(self, i):
        aug = self._aug_
        if self.on_device:
            return not aug["used"][i] or aug["slots"][i]["event"].query()
        return bool(self.device.ext.stream_ring_slot_done(aug["ring"], i))

    def _slot_sync(self, i):
        aug = self._aug_
        if self.on_device:
            if aug["used"][i]:
                aug["slots"][i]["event"].synchronize()
        else:
            self.device.ext.stream_ring_slot_sync(aug["ring"], i)

    def _cuda_serve(self):
        aug = self._aug_
        if aug is None:
            return super()._cuda_serve()
        ext = self.device.ext
        n = int(self.minibatch_size)
        idx = self.minibatch_indices.mem
        i = aug["i"]
        sl = aug["slots"][i]
        pend, aug["pending"] = aug["pending"], None
        hit = False
        if pend is not None:
            ext.host_prefetch_wait(pend["ticket"])
            hit = pend["slot"] == i and pend["n"] == n and numpy.array_equal(pend["idx"], idx[:n])
        if not hit:
            self._slot_sync(i)          # the copy out of this slot must be done
        aug["hits"] = aug.get("hits", 0) + int(hit)
        sl["hdr"][:3] = (n, self.minibatch_class, self.epoch_number)
        sl["par"][:n] = self.augment_params(n)
        sl["par"][n:] = 0
        if self.on_device:
            sl["idx"][:] = idx
            ext.pull_from_host(sl["pin"], aug["dev"])
            sl["event"].record()
        else:
            if not hit:
                import torch
                ext.host_gather_rows(aug["host_src"], torch.from_numpy(idx), sl["rows"], n)
            numpy.take(self._label_ids_, idx[:n], out=sl["lab"][:n], mode="clip")
            sl["lab"][n:] = 0
            ext.stream_ring_step(aug["ring"], sl["pin"], i, aug["stage"], aug["dev"],
                                 self.device.copy_stream.cuda_stream)
            self.minibatch_labels.dev_written()
        aug["used"][i] = True
        aug["i"] = (i + 1) % self.SLOTS
        if not self.__dict__.get("augment_in_graph_"):
            self._device_augment()
        if not self.on_device and aug["prefetch"]:
            self._prefetch_next()

    def _prefetch_next(self):
        """Gather the rows of the following minibatch (same epoch only: its indices are fixed in
        ``shuffled_indices``) into the next pinned slot on the native worker pool. Its crops and
        flips are drawn when it is served, so the ``prng`` order does not change."""
        aug = self._aug_
        peek = self.peek_next_indices()
        if peek is None:
            return
        start, n = peek
        i = aug["i"]
        if not self._slot_done(i):
            self._slot_sync(i)
        idx = numpy.ascontiguousarray(self.shuffled_indices.mem[start:start + n], numpy.int32)
        import torch
        ticket = self.device.ext.host_prefetch_submit(aug["host_src"], torch.from_numpy(idx),
                                                      aug["slots"][i]["rows"], n)
        aug["pending"] = {"ticket": ticket, "slot": i, "n": n, "idx": idx}

    def graph_prelude(self):
        """Hands the augmentation launch to the workflow's forward graph segment: it only reads
        device buffers at fixed addresses that ``_cuda_serve`` refills each step."""
        if self._aug_ is None:
            return None
        self.__dict__["augment_in_graph_"] = True
        return self._device_augment

    def _device_augment(self):
        aug = self._aug_
        md, ml = self.minibatch_data, self.minibatch_labels
        dv = aug["dv"]
        self.device.ext.augment_minibatch(
            aug["src"], dv["hdr"], dv.get("idx"), dv["par"], aug["mean"], md.devmem,
            aug.get("labels"), ml.devmem if self.on_device else None, channel_pad_target(md))
        md.dev_written()
        ml.dev_written()

    def stop(self):
        """Do not leave a prefetch job writing into a pinned slot behind."""
        aug = self._aug_
        if aug is not None and aug["pending"] is not None:
            pend, aug["pending"] = aug["pending"], None
            self.device.ext.host_prefetch_wait(pend["ticket"])
        parent = super()
        if hasattr(parent, "stop"):
            parent.stop()


class ImagenetLoader(ImagenetLoaderBase):
    """AlexNet-style augmentation on top of the raw loader."""
    MAPPING = "imagenet_pickle_loader"
    subtracts_mean = True

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.crop_size_sx = kwargs.get("crop_size_sx", 224)
        self.crop_size_sy = kwargs.get("crop_size_sy", 224)
        self.mirror = kwargs.get("mirror", False)
        self.final_sy = self.crop_size_sy or self.sy
        self.final_sx = self.crop_size_sx or self.sx

    def augment_params(self, n):
        """Random crops (TRAIN) or centre crops, then random flips (TRAIN with ``mirror``)."""
        p = numpy.zeros((n, 3), numpy.int32)
        cy, cx = self.final_sy, self.final_sx
        st = self.prng.state if hasattr(self.prng, "state") else numpy.random
        if (cy, cx) != (self.sy, self.sx):
            if self.minibatch_class == TRAIN:
                p[:, 0] = st.randint(0, self.sy - cy + 1, n)
                p[:, 1] = st.randint(0, self.sx - cx + 1, n)
            else:
                p[:, 0] = (self.sy - cy) // 2
                p[:, 1] = (self.sx - cx) // 2
        if self.mirror and self.minibatch_class == TRAIN:
            p[:, 2] = st.randint(0, 2, n)
        return p

    def transform_batch(self, raw):
        n = raw.shape[0]
        p = self.augment_params(n)
        x = raw.astype(host_dtype())
        if self.has_mean_file:
            x -= self.mean.mem.astype(x.dtype)
        cy, cx = self.final_sy, self.final_sx
        if (cy, cx) != (self.sy, self.sx):
            rows = p[:, 0, None] + numpy.arange(cy)[None, :]
            cols = p[:, 1, None] + numpy.arange(cx)[None, :]
            x = x[numpy.arange(n)[:, None, None], rows[:, :, None], cols[:, None, :]]
        flip = p[:, 2].astype(bool)
        if flip.any():
            x[flip] = x[flip][:, :, ::-1]
        return x
