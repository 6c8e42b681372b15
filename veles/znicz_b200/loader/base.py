"""Loader base classes (fresh design for the absent ``veles.loader``).

Contract = SURVEY §8 "Loader attributes consumed by Znicz"
(/root/reference/standard_workflow.py:429-447,469-489,554-565;
/root/reference/evaluator.py:85-87; /root/reference/decision.py:165-166).

Serving order inside one epoch is TEST(0) → VALID(1) → TRAIN(2) over a global
sample index space laid out in that order; ``last_minibatch`` marks the last
minibatch of a class, ``epoch_ended`` fires on the last VALID minibatch (or TRAIN
when there is no validation set) and ``epoch_number`` advances when TRAIN wraps.
The last minibatch of a class may be short: buffers are max-sized, the tail is
zero-filled (labels -1) and ``minibatch_size`` carries the real count.

H100 path: the minibatch is staged in pinned host memory and copied H2D on a
dedicated copy stream into one of two device buffers (double buffering, the
``Avatar`` equivalent), together with a small device-side header
``[minibatch_size, minibatch_class]`` so captured CUDA graphs read the runtime
batch size from HBM instead of being re-captured.
"""
from __future__ import annotations

import numpy

from ..core import prng
from ..core.accelerated_units import AcceleratedUnit, host_dtype
from ..core.config import root
from ..core.distributable import IDistributable
from ..core.memory import Array
from ..core.mutable import Bool
from ..core.normalization import make_normalizer, NoneNormalizer
from ..core.registry import make_registry
from ..core.units import Unit

TEST, VALID, TRAIN = 0, 1, 2
CLASS_NAME = ["test", "validation", "train"]
TARGET, LABEL = "target", "label"

UserLoaderRegistry = make_registry("loaders")
UserLoaderRegistry.loaders = UserLoaderRegistry.registry


class LoaderFactory(object):
    """Picklable ``callable(workflow, **extra) -> Loader`` bound to a registry name."""

    def __init__(self, name, kwargs):
        if name not in UserLoaderRegistry.registry:
            raise ValueError("Unknown loader %r (known: %s)" % (
                name, sorted(UserLoaderRegistry.registry)))
        self.name = name
        self.kwargs = dict(kwargs)

    def __call__(self, workflow, **extra):
        kw = dict(self.kwargs)
        kw.update(extra)
        return UserLoaderRegistry.registry[self.name](workflow, **kw)


def _get_factory(name, **kwargs):
    return LoaderFactory(name, kwargs)


UserLoaderRegistry.get_factory = staticmethod(_get_factory)


class LoaderError(Exception):
    pass


def channel_pad_target(md):
    """The channel-padded copy ``[n][h][w][8]`` of the minibatch that a first conv layer with
    C < 8 asks for (``pad_request_`` on the Array, kernels/api.py::conv_forward), allocated on
    first use, so the loader's device kernel writes it with the minibatch; None when nobody asked."""
    cp = md.__dict__.get("pad_request_")
    if not cp or md.devmem.dim() != 4 or md.devmem.shape[3] >= 8:
        return None
    pad = md.__dict__.get("padded_dev_")
    shape = tuple(md.devmem.shape[:3]) + (8,)
    if pad is None or tuple(pad.shape) != shape or pad.dtype != md.devmem.dtype:
        import torch
        pad = torch.zeros(shape, dtype=md.devmem.dtype, device=md.devmem.device)
        md.__dict__["padded_dev_"] = pad
    return pad


class Loader(AcceleratedUnit, metaclass=UserLoaderRegistry):
    """Serves minibatches. Subclasses implement ``load_data`` (set class_lengths),
    ``create_minibatch_data`` and ``fill_minibatch``."""
    hide_from_registry = True
    exports = ("minibatch_data", "minibatch_labels", "minibatch_indices",
               "minibatch_size", "minibatch_class", "minibatch_offset",
               "last_minibatch", "epoch_ended", "epoch_number", "train_ended",
               "class_lengths", "total_samples", "max_minibatch_size")

    def __init__(self, workflow, **kwargs):
        kwargs.setdefault("view_group", "LOADER")
        self.last_minibatch = Bool(False)
        self.epoch_ended = Bool(False)
        self.train_ended = Bool(False)
        self.complete = Bool(False)
        super().__init__(workflow, **kwargs)
        self.max_minibatch_size = int(kwargs.get("minibatch_size", 100))
        if self.max_minibatch_size < 1:
            raise ValueError("minibatch_size must be >= 1")
        self.class_lengths = [0, 0, 0]
        self.class_end_offsets = [0, 0, 0]
        self.total_samples = 0
        self.epoch_number = 0
        self.minibatch_class = TRAIN
        self.minibatch_size = 0
        self.minibatch_offset = 0
        self.global_offset = 0
        self.samples_served = 0
        self.minibatch_data = Array(shallow_pickle=True)
        self.minibatch_indices = Array(shallow_pickle=True)
        self.minibatch_labels = Array(shallow_pickle=True)
        self.shuffled_indices = Array()
        self.shuffle_limit = kwargs.get("shuffle_limit", numpy.iinfo(numpy.uint32).max)
        self.prng = kwargs.get("prng", prng.get(2))
        self.normalization_type = kwargs.get("normalization_type", "none")
        self.normalization_parameters = kwargs.get("normalization_parameters", {})
        self.train_ratio = kwargs.get("train_ratio", 1.0)
        self.validation_ratio = kwargs.get("validation_ratio", None)
        self.testing_mode = False
        self.labels_mapping = {}
        self.reversed_labels_mapping = []
        self.on_initialized = None
        self.has_labels_override = None
        self._normalizer = None
        self.class_keys = [[], [], []]
        self.epoch_limit = kwargs.get("epoch_limit")

    def init_unpickled(self):
        super().init_unpickled()
        self._dev_bufs_ = None
        self._dev_buf_idx_ = 0
        self._pinned_ = None
        self.header_dev_ = None
        self._copy_events_ = None

    # -- derived properties ---------------------------------------------------------
    @property
    def has_labels(self):
        if self.has_labels_override is not None:
            return self.has_labels_override
        return bool(self.labels_mapping) or bool(self.minibatch_labels)

    @property
    def unique_labels_count(self):
        return len(self.labels_mapping)

    @property
    def normalizer(self):
        if self._normalizer is None:
            self._normalizer = make_normalizer(
                self.normalization_type, **dict(self.normalization_parameters))
        return self._normalizer

    @property
    def class_ended(self):
        off = self.global_offset
        return any(off == e for e in self.class_end_offsets if e)

    @property
    def effective_class_end_offsets(self):
        return self.class_end_offsets

    @property
    def pending_minibatches_count(self):
        return 0

    def derive_from(self, loader):
        """Copy dataset-independent settings (normalizer state, label maps)."""
        self.normalization_type = loader.normalization_type
        self.normalization_parameters = loader.normalization_parameters
        self._normalizer = loader._normalizer
        self.labels_mapping = dict(loader.labels_mapping)
        self.reversed_labels_mapping = list(loader.reversed_labels_mapping)
        self.max_minibatch_size = loader.max_minibatch_size

    # -- to be implemented by subclasses ----------------------------------------------
    def load_data(self):
        raise NotImplementedError

    def create_minibatch_data(self):
        raise NotImplementedError

    def fill_minibatch(self):
        raise NotImplementedError

    def fill_indices(self, start, count):
        """Default: indices come from ``shuffled_indices``. Returns True if the
        subclass already filled the minibatch data itself."""
        self.minibatch_indices.map_invalidate()
        idx = self.minibatch_indices.mem
        idx[:count] = self.shuffled_indices.mem[start:start + count]
        idx[count:] = -1
        return False

    def map_minibatch_labels(self):
        pass

    # -- life cycle -------------------------------------------------------------------
    def initialize(self, device=None, **kwargs):
        super().initialize(device=device, **kwargs)
        snapshot = kwargs.get("snapshot", False)
        self.testing_mode = bool(self.testing)
        if not snapshot or not self.total_samples:
            self.load_data()
            self.on_data_loaded()
            self._update_total_samples()
            if self.testing_mode:
                self.shuffle_limit = 0
            self.global_offset = 0
            self.epoch_number = 0
            self.epoch_ended <<= False
            self.train_ended <<= False
            self.last_minibatch <<= False
            self.complete <<= False
        else:
            if not self._data_loaded():
                self.load_data()
                self.on_data_loaded()
            self._update_total_samples()
        self.max_minibatch_size = min(
            self.max_minibatch_size, max(self.class_lengths) or self.max_minibatch_size)
        self.info("Samples: test %d, validation %d, train %d; minibatch %d",
                  *(list(self.class_lengths) + [self.max_minibatch_size]))
        self.create_minibatch_data()
        if not self.minibatch_indices or \
                self.minibatch_indices.shape[0] != self.max_minibatch_size:
            self.minibatch_indices.reset(
                numpy.zeros(self.max_minibatch_size, dtype=numpy.int32))
        if not self.shuffled_indices or self.shuffled_indices.size != self.total_samples:
            self.shuffled_indices.reset(
                numpy.arange(self.total_samples, dtype=numpy.int32))
        self.analyze_dataset()
        if self.on_cuda:
            self._cuda_setup()
        if self.on_initialized is not None:
            cb = self.on_initialized
            cb()
        return None

    def _data_loaded(self):
        return True

    def on_data_loaded(self):
        """Hook between ``load_data`` and the offsets computation (validation carving)."""
        pass

    def analyze_dataset(self):
        pass

    def _update_total_samples(self):
        self.total_samples = int(sum(self.class_lengths))
        if self.total_samples == 0:
            raise LoaderError("There is no data to serve")
        acc = 0
        for i, n in enumerate(self.class_lengths):
            acc += n
            self.class_end_offsets[i] = acc
        if self.class_lengths[TRAIN] < 1 and not self.testing_mode and \
                not self.class_lengths[VALID] and not self.class_lengths[TEST]:
            raise LoaderError("class_length for TRAIN dataset is invalid")

    def shard(self, rank, world):
        """Data-parallel sharding: rank r keeps every world-th sample of each class
        (equal shard sizes, remainder dropped) — the synchronous equivalent of the master
        handing different minibatches to different slaves."""
        # Idempotent and re-shardable: the unsharded index set is kept (and pickled with the
        # snapshot), every call derives the shard from it. A snapshot taken on 8 ranks resumes
        # on 8, 4 or 1 rank(s) over the whole dataset instead of 1/N^2 (or 1/N) of it.
        cur = (getattr(self, "dp_rank", 0), getattr(self, "dp_world", 1))
        if cur == (rank, max(world, 1)) and (world <= 1 or
                                             getattr(self, "unsharded_indices", None) is not None):
            return
        if getattr(self, "unsharded_indices", None) is None:
            if world <= 1:
                return
            self.shuffled_indices.map_read()
            self.unsharded_indices = numpy.array(self.shuffled_indices.mem, copy=True)
            self.unsharded_class_lengths = list(self.class_lengths)
        full = self.unsharded_indices
        world = max(world, 1)
        parts, start = [], 0
        for i in range(3):
            n = self.unsharded_class_lengths[i]
            keep = (n // world)
            parts.append(full[start:start + keep * world][rank::world][:keep])
            start += n
            self.class_lengths[i] = keep
        self.shuffled_indices.reset(numpy.concatenate(parts).astype(numpy.int32))
        self._update_total_samples()
        # Same world size, other rank (rank 0's snapshot restored on rank r): the class layout of
        # every shard is identical, so the position inside the epoch is kept - rank 0 keeps its
        # own, and the replicas must stay in lock step. A different world size moves every class
        # boundary: all ranks restart the epoch (all of them take this branch).
        if cur[1] != world:
            self.global_offset = 0
        self.dp_rank, self.dp_world = rank, world
        self.prng = prng.RandomGenerator(seed=977 + rank)

    # -- serving --------------------------------------------------------------------
    def shuffle(self):
        if self.shuffle_limit <= 0 or self.class_lengths[TRAIN] == 0:
            return
        self.shuffle_limit -= 1
        self.shuffled_indices.map_write()
        self.prng.shuffle(self.shuffled_indices.mem[self.class_end_offsets[VALID]:])

    def class_index_by_offset(self, offset):
        for i, e in enumerate(self.class_end_offsets):
            if offset < e:
                return i
        raise LoaderError("offset %d is out of range" % offset)

    def _advance(self):
        """Pick the next minibatch: (class, start, count)."""
        if self.global_offset >= self.total_samples:
            self.global_offset = 0
        off = self.global_offset
        cls = self.class_index_by_offset(off)
        count = min(self.max_minibatch_size, self.class_end_offsets[cls] - off)
        return cls, off, count

    def run(self):
        if self.global_offset == 0 or self.global_offset >= self.total_samples:
            self.shuffle()  # epoch start: reshuffle the train part
        prof = self.__dict__.get("prof_")      # ZNICZ_BENCH_STATS: where the host time goes
        if prof is not None:
            import time
            t0 = time.perf_counter()
        if self.on_cuda:
            self._cuda_begin_step()
        if prof is not None:
            t1 = time.perf_counter()
        cls, start, count = self._advance()
        self.minibatch_class = cls
        self.minibatch_size = count
        self.global_offset = start + count
        self.minibatch_offset = self.global_offset
        self.samples_served += count
        if not self.fill_indices(start, count):
            self.fill_minibatch()
        self.map_minibatch_labels()
        self._update_flags()
        if prof is not None:
            t2 = time.perf_counter()
        if self.on_cuda:
            self._cuda_serve()
        if prof is not None:
            t3 = time.perf_counter()
            prof[0] += t1 - t0     # wait for the pinned slot (= how far the device lags)
            prof[1] += t2 - t1     # bookkeeping + minibatch assembly on the host
            prof[2] += t3 - t2     # H2D enqueue (+ gather launch)
            prof[3] += 1

    def peek_next_indices(self):
        """(start, count) of the slice of ``shuffled_indices`` the *next* ``run()`` will serve, or
        None when that run starts a new epoch (the train part is reshuffled first, so its indices
        are not known yet). Pure function of the loader state after a ``run()``."""
        start = self.global_offset
        if start <= 0 or start >= self.total_samples:
            return None
        cls = self.class_index_by_offset(start)
        n = int(min(self.max_minibatch_size, self.class_end_offsets[cls] - start))
        return (start, n) if n > 0 else None

    def _update_flags(self):
        last_mb = self.global_offset == self.class_end_offsets[self.minibatch_class]
        self.last_minibatch <<= last_mb
        cls = self.minibatch_class
        no_valid = self.class_lengths[VALID] == 0
        self.epoch_ended <<= last_mb and (
            cls == VALID or (cls == TRAIN and no_valid) or
            (cls == TEST and no_valid and self.class_lengths[TRAIN] == 0))
        self.train_ended <<= last_mb and cls == TRAIN
        if last_mb and self.global_offset >= self.total_samples:
            self.epoch_number += 1
            if self.testing_mode or (
                    self.epoch_limit is not None and
                    self.epoch_number >= self.epoch_limit):
                self.complete <<= True

    # -- H100 staging -----------------------------------------------------------------
    def _staged_arrays(self):
        """Arrays copied H2D every step."""
        arrs = [self.minibatch_data]
        if self.minibatch_labels:
            arrs.append(self.minibatch_labels)
        return arrs

    def _cuda_setup(self):
        import torch
        dev = self.device
        self.init_vectors(self.minibatch_data, self.minibatch_labels,
                          self.minibatch_indices)
        # device header: [minibatch_size, minibatch_class, epoch_number, reserved]
        self.header_dev_ = torch.zeros(4, dtype=torch.int32, device=dev.torch_device)
        hdr = torch.zeros(4, dtype=torch.int32).pin_memory()
        self._pinned_ = {"header": hdr, "header_np": hdr.numpy(), "slot": 0,
                         "events": [torch.cuda.Event(), torch.cuda.Event()], "bufs": {}}
        # double-buffered pinned staging: the Arrays' host memory *is* the pinned buffer, so
        # fill_minibatch gathers straight into DMA-able memory (no extra host copy)
        for a in self._staged_arrays():
            t = torch.from_numpy(a.mem)
            pair = [torch.zeros_like(t).pin_memory(), torch.zeros_like(t).pin_memory()]
            self._pinned_["bufs"][id(a)] = (a, pair, [p.numpy() for p in pair])
        self.h2d_bytes_per_step = sum(
            a.mem.nbytes for a in self._staged_arrays()) + 16

    def _cuda_begin_step(self):
        """Flip to the other pinned staging slot (waiting for its previous H2D copy)."""
        pd = self._pinned_
        slot = pd["slot"] ^ 1
        pd["slot"] = slot
        pd["events"][slot].synchronize()
        for a, pair, views in pd["bufs"].values():
            a._mem = views[slot]

    def _cuda_serve(self):
        """Copy this step's minibatch host→device from pinned memory (async on the
        compute stream so the captured step graph that follows sees the data)."""
        import torch
        pd = self._pinned_
        slot = pd["slot"]
        for a, pair, views in pd["bufs"].values():
            pin = pair[slot]
            dst = a.devmem
            if dst.dtype != pin.dtype:
                # fp32 payload -> device staging -> one cast kernel produces the bf16 minibatch.
                # (A side-stream variant that overlapped this copy with the previous step was
                # measured *slower* end to end, 267 K vs 307 K images/s: the extra stream/event
                # calls cost more host time than the 25 us copy they hid.)
                key = "_stage_%d_" % id(a)
                tmp = self.__dict__.get(key)
                if tmp is None:
                    tmp = torch.empty(pin.shape, dtype=pin.dtype, device=dst.device)
                    self.__dict__[key] = tmp
                tmp.copy_(pin, non_blocking=True)
                self.device.ext.cast_copy(tmp, dst)
            else:
                dst.copy_(pin, non_blocking=True)
            a.dev_written()
        hn = pd["header_np"]
        hn[0] = self.minibatch_size
        hn[1] = self.minibatch_class
        hn[2] = self.epoch_number
        self.header_dev_.copy_(pd["header"], non_blocking=True)
        # the pinned slot may be refilled once every copy out of it has been issued and finished:
        # the compute stream already waits for the side-stream copy, so one event covers both
        pd["events"][slot].record()

    # -- IDistributable: the master serves indices, the slaves read the data --------------
    def generate_data_for_slave(self, slave=None):
        self.run()
        self.minibatch_indices.map_read()
        return {"indices": self.minibatch_indices.mem[:self.minibatch_size].copy(),
                "minibatch_class": self.minibatch_class,
                "minibatch_size": self.minibatch_size,
                "minibatch_offset": self.minibatch_offset,
                "epoch_number": self.epoch_number,
                "last_minibatch": bool(self.last_minibatch),
                "epoch_ended": bool(self.epoch_ended)}

    def apply_data_from_master(self, data):
        n = data["minibatch_size"]
        self.minibatch_class = data["minibatch_class"]
        self.minibatch_size = n
        self.minibatch_offset = data["minibatch_offset"]
        self.epoch_number = data["epoch_number"]
        self.last_minibatch <<= data["last_minibatch"]
        self.epoch_ended <<= data["epoch_ended"]
        self.minibatch_indices.map_invalidate()
        self.minibatch_indices.mem[:n] = data["indices"]
        self.minibatch_indices.mem[n:] = -1
        self.fill_minibatch()

    def generate_data_for_master(self):
        return True

    def apply_data_from_slave(self, data, slave=None):
        pass

    def drop_slave(self, slave=None):
        pass


class LoaderMSEMixin(object):
    """Adds regression targets (``minibatch_targets``, ``class_targets``,
    ``target_normalizer``) — consumed by EvaluatorMSE
    (/root/reference/standard_workflow.py:443-447)."""

    def _init_mse(self, kwargs):
        self.minibatch_targets = Array(shallow_pickle=True)
        self.class_targets = Array()
        self.target_normalization_type = kwargs.get(
            "target_normalization_type", kwargs.get("normalization_type", "none"))
        self.target_normalization_parameters = kwargs.get(
            "target_normalization_parameters",
            kwargs.get("normalization_parameters", {}))
        self._target_normalizer = None
        self.targets_shape = kwargs.get("targets_shape", ())

    @property
    def target_normalizer(self):
        if self._target_normalizer is None:
            self._target_normalizer = make_normalizer(
                self.target_normalization_type,
                **dict(self.target_normalization_parameters))
        return self._target_normalizer


class LoaderWithValidationRatio(object):
    """Mixin: carve a validation set out of the train set (``validation_ratio``)."""

    def resize_validation(self, rand=None):
        ratio = self.validation_ratio
        if ratio is None or ratio <= 0:
            return
        if not 0 < ratio < 1:
            raise ValueError("validation_ratio must be in (0, 1)")
        n_train = self.class_lengths[TRAIN]
        n_valid = int(numpy.round(ratio * (n_train + self.class_lengths[VALID])))
        delta = n_valid - self.class_lengths[VALID]
        if delta <= 0:
            return
        self.class_lengths[VALID] += delta
        self.class_lengths[TRAIN] -= delta
        return delta
