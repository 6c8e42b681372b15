"""Full-batch loaders: the whole dataset lives in memory.

Fresh design for ``veles.loader.fullbatch`` (FullBatchLoader, FullBatchLoaderMSE)
as consumed by the reference's loaders (/root/reference/loader/loader_wine.py:48-66,
/root/reference/loader/loader_mnist.py:53-186, /root/reference/samples/CIFAR10/cifar.py:47-66).

Data layout: ``original_data[total, ...]`` ordered TEST, VALID, TRAIN;
``original_labels`` a python list / int32 array of raw labels mapped to
0..n-1 via ``labels_mapping``.

H100: with ``on_device=True`` (default when the dataset fits comfortably in the
80 GB of HBM3) the dataset is uploaded once and every
minibatch is produced by a device gather kernel (``gather_rows``), so no host
traffic happens in the training loop; with ``on_device=False`` minibatches are
staged through pinned memory each step (streaming mode, the path ``bench.py``
times end-to-end).
"""
from __future__ import annotations

import numpy

from ..core.config import root

from ..core.accelerated_units import host_dtype
from ..core.memory import Array
from .base import (Loader, LoaderMSEMixin, LoaderWithValidationRatio, TEST, VALID,
                   TRAIN, LoaderError, channel_pad_target)


def _pull_ok(ext):
    """Per-step uploads go through a kernel that reads the pinned buffer (ext.pull_from_host)
    rather than cudaMemcpyAsync; ``root.common.engine.loader_pull = False`` restores the copies."""
    return ext is not None and hasattr(ext, "pull_from_host") and \
        bool(root.common.engine.get("loader_pull", True))


class FullBatchLoader(Loader, LoaderWithValidationRatio):
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.original_data = Array()
        self.original_labels = []
        self.on_device = kwargs.get("on_device", False)
        self.validation_ratio = kwargs.get("validation_ratio", None)
        self.validation_seed = kwargs.get("validation_seed", 0x5EED)
        self._mapped_original_labels = Array()
        self._normalized = False

    def init_unpickled(self):
        super().init_unpickled()
        self._labels_dev_ = None

    def _data_loaded(self):
        return bool(self.original_data)

    def on_data_loaded(self):
        """``validation_ratio``: shuffle VALID+TRAIN with a fixed seed (the dataset is
        usually sorted by label) and move the class boundary."""
        if not self.validation_ratio:
            return
        start = self.class_lengths[TEST]
        n = self.class_lengths[VALID] + self.class_lengths[TRAIN]
        before = self.class_lengths[VALID]
        self.resize_validation()
        if self.class_lengths[VALID] == before:
            return
        perm = numpy.random.RandomState(self.validation_seed).permutation(n) + start
        for arr in (self.original_data, getattr(self, "original_targets", None)):
            if arr is not None and arr:
                arr.mem[start:start + n] = arr.mem[perm]
        if len(self.original_labels):
            labels = list(self.original_labels)
            labels[start:start + n] = [labels[i] for i in perm]
            self.original_labels = labels

    @property
    def dtype(self):
        return host_dtype()

    def create_minibatch_data(self):
        shape = (self.max_minibatch_size,) + tuple(self.original_data.shape[1:])
        if not self.minibatch_data or self.minibatch_data.shape != shape:
            self.minibatch_data.reset(numpy.zeros(shape, dtype=self.dtype))
        if self.on_cuda:
            from ..ops.nn_units import torch_act_dtype
            self.minibatch_data.dev_dtype = torch_act_dtype()
        if self.has_labels and (
                not self.minibatch_labels or
                self.minibatch_labels.shape[0] != self.max_minibatch_size):
            self.minibatch_labels.reset(
                numpy.zeros(self.max_minibatch_size, dtype=numpy.int32))

    @property
    def has_labels(self):
        return len(self.original_labels) > 0

    def analyze_dataset(self):
        """Map raw labels, carve validation, normalise in place (once)."""
        if self.has_labels and not self.labels_mapping:
            uniq = sorted(set(self.original_labels[self.class_end_offsets[VALID]:]) or
                          set(self.original_labels))
            # labels that only exist outside train are appended after
            extra = sorted(set(self.original_labels) - set(uniq))
            self.labels_mapping = {l: i for i, l in enumerate(uniq + extra)}
            self.reversed_labels_mapping = uniq + extra
        if self.has_labels:
            mapped = numpy.fromiter(
                (self.labels_mapping[l] for l in self.original_labels),
                dtype=numpy.int32, count=len(self.original_labels))
            self._mapped_original_labels.reset(mapped)
        if not self._normalized:
            self._normalize_dataset()
            self._normalized = True

    def _normalize_dataset(self):
        data = self.original_data.mem
        if self.normalization_type == "none":
            if data.dtype != self.dtype:
                self.original_data.reset(data.astype(self.dtype))
            return
        if data.dtype != self.dtype:
            data = data.astype(self.dtype)
        norm = self.normalizer
        train = data[self.class_end_offsets[VALID]:] if self.class_lengths[TRAIN] \
            else data
        if not norm.is_initialized:
            norm.analyze(train)
        data = norm.normalize(data)
        self.original_data.reset(data)

    def fill_minibatch(self):
        if self.__dict__.get("_packed_") is not None:
            return self._fill_packed()
        n = self.minibatch_size
        idx = self.minibatch_indices.mem[:n]
        self.minibatch_data.map_invalidate()
        md = self.minibatch_data.mem
        numpy.take(self.original_data.mem, idx, axis=0, out=md[:n], mode="clip")
        if n < md.shape[0]:
            md[n:] = 0
        if self.has_labels:
            self.minibatch_labels.map_invalidate()
            ml = self.minibatch_labels.mem
            numpy.take(self._mapped_original_labels.mem, idx, out=ml[:n], mode="clip")
            ml[n:] = -1

    # -- device-resident dataset ---------------------------------------------------------
    def fill_indices(self, start, count):
        super().fill_indices(start, count)
        # dataset in HBM: only the indices travel, the rows are gathered on the device
        return bool(self.on_device and self.on_cuda)

    def _cuda_setup(self):
        super()._cuda_setup()
        if self.on_device:
            import torch
            # only header + indices are staged per step; data/labels stay in HBM
            self._pinned_["bufs"] = {}
            self.original_data.initialize(self.device)
            if self.has_labels:
                self._mapped_original_labels.initialize(self.device)
            n = 4 + self.max_minibatch_size
            self._hdr_idx_dev_ = torch.zeros(n, dtype=torch.int32,
                                             device=self.device.torch_device)
            self.header_dev_ = self._hdr_idx_dev_[:4]
            pins = [torch.zeros(n, dtype=torch.int32).pin_memory() for _ in range(2)]
            self._pinned_["hdr_idx"] = pins
            self._pinned_["hdr_idx_np"] = [p.numpy() for p in pins]
            self.h2d_bytes_per_step = n * 4
            row = self.original_data.size // self.original_data.shape[0]
            self._fused_gather_ = (row % 8 == 0)
        else:
            self._setup_packed()

    # -- streaming from host memory: one packed pinned buffer, one H2D copy per step ----------
    def _setup_packed(self):
        """Header, labels and the minibatch share ONE device buffer fed by ONE asynchronous copy
        from a pinned slot; the slot is filled by the native gather (rows by index on the
        intra-op thread pool, converted to the device dtype on the fly), so a bf16 model moves
        half the bytes and needs no cast kernel. The Arrays' device tensors become views."""
        import torch
        self.__dict__["_packed_"] = None
        ext = getattr(self.device, "ext", None)
        md, ml = self.minibatch_data, self.minibatch_labels
        od = self.original_data.mem
        if ext is None or not hasattr(ext, "host_gather_rows") or type(self).fill_minibatch \
                is not FullBatchLoader.fill_minibatch or od.dtype != numpy.float32 or \
                not od.flags["C_CONTIGUOUS"] or md.devmem is None or \
                md.devmem.dtype not in (torch.float32, torch.bfloat16) or \
                self.minibatch_indices.mem.dtype != numpy.int32:
            return
        labels = bool(self.has_labels and ml and ml.devmem is not None and
                      ml.devmem.dtype == torch.int32)
        if self.has_labels and not labels:
            return
        mb = self.max_minibatch_size
        dt = md.devmem.dtype
        esz = 2 if dt == torch.bfloat16 else 4
        off_data = (16 + (4 * mb if labels else 0) + 255) // 256 * 256
        total = off_data + md.size * esz
        devp = torch.zeros(total, dtype=torch.uint8, device=self.device.torch_device)
        depth = 4       # pinned slots: the prefetcher fills slot i+1 while the copy out of slot i
        pins = [torch.zeros(total, dtype=torch.uint8).pin_memory() for _ in range(depth)]

        def views(buf):
            hdr = buf[:16].view(torch.int32)
            lab = buf[16:16 + 4 * mb].view(torch.int32) if labels else None
            data = buf[off_data:].view(dt).view(tuple(md.shape))
            return hdr, lab, data
        hdr_d, lab_d, data_d = views(devp)
        md._devmem_ = data_d
        if labels:
            ml._devmem_ = lab_d.view(tuple(ml.shape))
        self.header_dev_ = hdr_d
        slots = []
        for p in pins:
            hdr, lab, data = views(p)
            slots.append({"pin": p, "hdr": hdr.numpy(), "lab": lab.numpy() if labels else None,
                          "data": data, "event": torch.cuda.Event(), "used": False})
        self._pinned_["bufs"] = {}
        self.__dict__["_packed_"] = {
            "dev": devp, "slots": slots, "labels": labels, "i": 0, "pending": None,
            "src": torch.from_numpy(od),
            "idx": torch.from_numpy(self.minibatch_indices.mem),
            "prefetch": hasattr(ext, "host_prefetch_submit") and
            root.common.engine.get("loader_prefetch", True),
            "pull": _pull_ok(ext)}
        self.h2d_bytes_per_step = total
        # Early pull: the host runs 1-3 steps ahead of the device, so the PCIe pull of the next
        # minibatch is issued on the copy stream into a small ring of device staging buffers and
        # executes while earlier steps still compute; the step's own stream only carries a
        # device-to-device copy (615 KB: 2-3 us instead of the 18 us PCIe-bound pull).
        pk = self._packed_
        pk["early"] = bool(pk["pull"] and hasattr(ext, "device_copy") and
                           getattr(self.device, "copy_stream", None) is not None and
                           root.common.engine.get("loader_early_pull", True))
        pk["ring"] = None
        if pk["early"]:
            import os
            if hasattr(ext, "stream_ring_step") and os.environ.get("ZNICZ_STREAM_RING", "1") != "0":
                # the whole per-step copy sequence in one native call (events owned by the ring)
                pk["ring"] = int(ext.stream_ring_create(3, depth))
            pk["stage"] = [torch.zeros_like(devp) for _ in range(3)]
            pk["stage_evt"] = [torch.cuda.Event() for _ in range(3)]
            pk["stage_used"] = [False] * 3
            pk["pull_evt"] = [torch.cuda.Event() for _ in range(3)]
            pk["s"] = 0

    def _fill_packed(self):
        """Minibatch → pinned slot: already there when the prefetcher guessed this minibatch
        (same index list), otherwise gathered now."""
        pk = self._packed_
        ext = self.device.ext
        n = int(self.minibatch_size)
        idx = self.minibatch_indices.mem
        pend, pk["pending"] = pk["pending"], None
        hit = False
        if pend is not None:
            ext.host_prefetch_wait(pend["ticket"])
            hit = pend["slot"] == pk["i"] and pend["n"] == n and \
                numpy.array_equal(pend["idx"], idx[:n])
        sl = pk["slots"][pk["i"]]
        if not hit:
            if sl["used"]:
                self._slot_sync(pk["i"])       # the copy out of this slot must be done
            ext.host_gather_rows(pk["src"], pk["idx"], sl["data"], n)
        pk["hits"] = pk.get("hits", 0) + int(hit)
        if pk["labels"]:
            lab = sl["lab"]
            numpy.take(self._mapped_original_labels.mem, idx[:n], out=lab[:n], mode="clip")
            lab[n:] = -1

    def _serve_packed(self):
        pk = self._packed_
        sl = pk["slots"][pk["i"]]
        hn = sl["hdr"]
        hn[0] = self.minibatch_size
        hn[1] = self.minibatch_class
        hn[2] = self.epoch_number
        if pk.get("ring") is not None:
            self.device.ext.stream_ring_step(pk["ring"], sl["pin"], pk["i"], pk["stage"], pk["dev"],
                                             self.device.copy_stream.cuda_stream)
        elif pk.get("early"):
            import torch
            ext = self.device.ext
            k = pk["s"]
            pk["s"] = (k + 1) % len(pk["stage"])
            side = self.device.copy_stream      # (not the wgrad side stream: that one is captured)
            if pk["stage_used"][k]:
                side.wait_event(pk["stage_evt"][k])      # its previous contents were copied out
            with torch.cuda.stream(side):
                ext.pull_from_host(sl["pin"], pk["stage"][k])
                pk["pull_evt"][k].record()
                sl["event"].record()                      # pinned slot free once the pull is done
            main = torch.cuda.current_stream()
            main.wait_event(pk["pull_evt"][k])
            ext.device_copy(pk["stage"][k], pk["dev"])
            pk["stage_evt"][k].record()
            pk["stage_used"][k] = True
        elif pk["pull"]:
            self.device.ext.pull_from_host(sl["pin"], pk["dev"])    # SMs read the pinned slot
            sl["event"].record()
        else:
            pk["dev"].copy_(sl["pin"], non_blocking=True)
            sl["event"].record()
        sl["used"] = True
        self.minibatch_data.dev_written()
        if pk["labels"]:
            self.minibatch_labels.dev_written()
        pk["i"] = (pk["i"] + 1) % len(pk["slots"])
        if pk["prefetch"]:
            self._prefetch_next()

    def _slot_done(self, i):
        pk = self._packed_
        if pk.get("ring") is not None:
            return bool(self.device.ext.stream_ring_slot_done(pk["ring"], i))
        return pk["slots"][i]["event"].query()

    def _slot_sync(self, i):
        pk = self._packed_
        if pk.get("ring") is not None:
            self.device.ext.stream_ring_slot_sync(pk["ring"], i)
        else:
            pk["slots"][i]["event"].synchronize()

    def _prefetch_next(self):
        """Start assembling the following minibatch (same epoch only: its indices are already
        fixed in ``shuffled_indices``) into the next pinned slot on the native worker pool."""
        pk = self._packed_
        peek = self.peek_next_indices()
        if peek is None:
            return                              # epoch wrap: the train part is reshuffled first
        start, n = peek
        sl = pk["slots"][pk["i"]]
        if sl["used"] and not self._slot_done(pk["i"]):
            # the copy out of this slot (issued depth - 1 steps ago) has not finished: the device
            # is that far behind, so the host has time to spare - wait for it rather than give
            # up the prefetch (bounds the run-ahead to depth - 1 steps)
            self._slot_sync(pk["i"])
        idx = numpy.ascontiguousarray(self.shuffled_indices.mem[start:start + n], numpy.int32)
        import torch
        ticket = self.device.ext.host_prefetch_submit(pk["src"], torch.from_numpy(idx),
                                                      sl["data"], n)
        pk["pending"] = {"ticket": ticket, "slot": pk["i"], "n": n, "idx": idx}

    def stop(self):
        """Do not leave a prefetch job writing into a pinned slot behind."""
        pk = self.__dict__.get("_packed_")
        if pk and pk.get("pending") is not None:
            pend, pk["pending"] = pk["pending"], None
            self.device.ext.host_prefetch_wait(pend["ticket"])
        parent = super()
        if hasattr(parent, "stop"):
            parent.stop()

    def _cuda_serve(self):
        if not self.on_device:
            if self.__dict__.get("_packed_") is not None:
                return self._serve_packed()
            return super()._cuda_serve()
        pd = self._pinned_
        slot = pd["slot"]
        n = int(self.minibatch_size)
        hn = pd["hdr_idx_np"][slot]
        hn[0] = n
        hn[1] = self.minibatch_class
        hn[2] = self.epoch_number
        hn[4:4 + self.max_minibatch_size] = self.minibatch_indices.mem
        if _pull_ok(self.device.ext):
            # no copy-engine operation in the step's stream
            self.device.ext.pull_from_host(pd["hdr_idx"][slot], self._hdr_idx_dev_)
        else:
            self._hdr_idx_dev_.copy_(pd["hdr_idx"][slot], non_blocking=True)
        pd["events"][slot].record()
        if self.__dict__.get("gather_in_graph_"):
            return          # the forward graph segment starts with the gather (graph_prelude)
        self._device_gather()

    def graph_prelude(self):
        """Called by the workflow when it builds its forward CUDA-graph segment: hands the
        device-side minibatch gather over to the segment (it only reads the header + index
        buffer this loader uploads each step, so it can be captured)."""
        if not (self.on_cuda and self.on_device and self.__dict__.get("_fused_gather_")):
            return None
        self.__dict__["gather_in_graph_"] = True
        return self._device_gather

    def _device_gather(self):
        ext = self.device.ext
        labels = self.has_labels
        n = int(self.minibatch_size)
        if self._fused_gather_:
            # a first conv layer with C % 8 != 0 asks for a channel-padded copy
            # (``pad_request_`` on the Array, kernels/api.py::conv_forward): produce it here
            md = self.minibatch_data
            pad = channel_pad_target(md)
            c = int(md.devmem.shape[3]) if pad is not None else 0
            ext.gather_minibatch(
                self.original_data.devmem,
                self._mapped_original_labels.devmem if labels else None,
                self._hdr_idx_dev_, md.devmem,
                self.minibatch_labels.devmem if labels else None, pad, c)
        else:
            idx = self._hdr_idx_dev_[4:]
            ext.gather_rows(self.original_data.devmem, idx, self.minibatch_data.devmem, n)
            if labels:
                ext.gather_labels(self._mapped_original_labels.devmem, idx,
                                  self.minibatch_labels.devmem, n)
        self.minibatch_data.dev_written()
        if labels:
            self.minibatch_labels.dev_written()


class FullBatchLoaderMSE(FullBatchLoader, LoaderMSEMixin):
    """Adds ``original_targets`` → ``minibatch_targets`` for MSE workflows."""
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._init_mse(kwargs)
        self.original_targets = Array()
        self._targets_normalized = False

    def create_minibatch_data(self):
        super().create_minibatch_data()
        shape = (self.max_minibatch_size,) + tuple(self.original_targets.shape[1:])
        if not self.minibatch_targets or self.minibatch_targets.shape != shape:
            self.minibatch_targets.reset(numpy.zeros(shape, dtype=self.dtype))
        if self.on_cuda:
            from ..ops.nn_units import torch_act_dtype
            self.minibatch_targets.dev_dtype = torch_act_dtype()
        self.targets_shape = tuple(self.original_targets.shape[1:])

    def analyze_dataset(self):
        super().analyze_dataset()
        if not self._targets_normalized and self.target_normalization_type != "none":
            t = self.original_targets.mem.astype(self.dtype)
            norm = self.target_normalizer
            train = t[self.class_end_offsets[VALID]:] if self.class_lengths[TRAIN] else t
            if not norm.is_initialized:
                norm.analyze(train)
            self.original_targets.reset(norm.normalize(t))
            if self.class_targets:
                ct = self.class_targets.mem.astype(self.dtype)
                self.class_targets.reset(norm.normalize(ct))
            self._targets_normalized = True

    def fill_minibatch(self):
        super().fill_minibatch()
        n = self.minibatch_size
        idx = self.minibatch_indices.mem[:n]
        self.minibatch_targets.map_invalidate()
        mt = self.minibatch_targets.mem
        numpy.take(self.original_targets.mem, idx, axis=0, out=mt[:n], mode="clip")
        mt[n:] = 0

    def _staged_arrays(self):
        return super()._staged_arrays() + [self.minibatch_targets]

    def _cuda_setup(self):
        self.init_vectors(self.minibatch_targets)
        super()._cuda_setup()

    def _cuda_serve(self):
        if self.on_device:
            raise LoaderError("on_device mode is not implemented for MSE loaders")
        return super()._cuda_serve()
