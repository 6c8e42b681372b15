"""The localisation workflow (/root/reference/tests/research/ImagenetAE/imagenet_forward/
imagenet_forward.py:237-388, imagenet_forward_config.py:40-86, distribute_forward.py:40-85).

    Repeater -> ForwardLoaderBbox -> [MeanDispNormalizer] -> trained forward units
             -> MergeBboxes -> (loop until the loader ends) -> ResultWriter -> End

``run_pipeline`` runs it twice: the MERGE stage over the raw candidate stream (few angles, boxes
merged per class) and the FINAL stage over the merge stage's own JSON (finer angles, one label per
box, thresholds). The reference restarts itself from ``on_workflow_finished``; here the two stages
are two explicit ``run()`` calls.
"""
from __future__ import annotations

import os
import pickle
import shutil

import numpy

from ...core.accelerated_units import AcceleratedWorkflow
from ...core.config import root
from ...core.workflow import Repeater
from .loader import ForwardLoaderBbox
from .merge import MergeBboxes
from .writer import ResultWriter

root.imagenet_forward.update({
    "loader": {"path_to_bboxes": "", "min_index": 0, "max_index": 0, "minibatch_size": 32,
               "only_this_file": "",
               "angle_step_merge": 1.0, "min_angle_merge": 0.0, "max_angle_merge": 0.0,
               "angle_step_final": numpy.pi / 12, "min_angle_final": -numpy.pi / 12,
               "max_angle_final": numpy.pi / 12,
               "raw_bboxes_min_area": 256, "raw_bboxes_min_size": 8,
               "raw_bboxes_min_area_ratio": 0.005, "raw_bboxes_min_size_ratio": 0.05},
    "trained_workflow": "",
    "result_path": "",
    "labels_txt": "",
    "mergebboxes": {"raw_path": "", "ignore_negative": False, "max_per_class": 6,
                    "probability_threshold": 0.45, "last_chance_probability_threshold": 0.39,
                    "mode": "", "labels_compatibility": "", "use_compatibility": True},
})


class ImagenetForward(AcceleratedWorkflow):
    """``forwards``: the trained forward units in order (taken over by this workflow), or
    ``trained_workflow``: a snapshot to import them from (every other unit of it is dropped).
    ``normalizer``: an optional MeanDispNormalizer of the trained workflow; ``mean``: the mean
    image shown outside the boxes (defaults to the normaliser's mean)."""
    hide_from_registry = True

    def __init__(self, workflow, forwards=None, normalizer=None, mean=None, **kwargs):
        super().__init__(workflow, **kwargs)
        cfg = root.imagenet_forward
        lcfg = dict(cfg.loader.__content__) if hasattr(cfg.loader, "__content__") else {}
        lcfg.update(kwargs.get("loader_config", {}))
        mcfg = dict(cfg.mergebboxes.__content__) if hasattr(cfg.mergebboxes, "__content__") else {}
        mcfg.update(kwargs.get("merge_config", {}))
        self.loader_config, self.merge_config = lcfg, mcfg
        self.result_path = kwargs.get("result_path") or cfg.get("result_path", "")
        if forwards is None:
            forwards, normalizer = self._import_trained(
                kwargs.get("trained_workflow") or cfg.get("trained_workflow", ""), normalizer)
        self.forwards = list(forwards)
        self.meandispnorm = normalizer
        if mean is None and normalizer is not None:
            mean = normalizer.mean

        self.repeater = Repeater(self)
        self.repeater.link_from(self.start_point)
        self.loader = ForwardLoaderBbox(
            self, bboxes_file_name=lcfg.get("path_to_bboxes") or None,
            bboxes=kwargs.get("bboxes", {}), image_reader=kwargs.get("image_reader"),
            angle_step=lcfg.get("angle_step_merge", 1.0),
            min_angle=lcfg.get("min_angle_merge", 0.0), max_angle=lcfg.get("max_angle_merge", 0.0),
            **{k: lcfg[k] for k in ("min_index", "max_index", "only_this_file", "minibatch_size",
                                    "raw_bboxes_min_area", "raw_bboxes_min_size",
                                    "raw_bboxes_min_area_ratio", "raw_bboxes_min_size_ratio",
                                    "add_relative_bboxes", "path_to_empty_images") if k in lcfg})
        if self.loader.image_reader is None:
            from .loader import default_image_reader
            self.loader.image_reader = default_image_reader
        self.loader.link_from(self.repeater)
        self.loader.gate_block = self.loader.ended
        for f in self.forwards:
            f.workflow = self
        shape = list(self.forwards[0].input.shape) if self.forwards[0].input else \
            list(kwargs["entry_shape"])
        shape[0] = self.loader.max_minibatch_size
        self.loader.entry_shape = shape
        self.loader.mean = mean
        # a bf16 first layer takes its input in bf16 (the wgmma path); the normaliser computes
        # in fp32, so in front of it the minibatch stays fp32
        self.loader.feeds_first_layer = normalizer is None
        first = self.forwards[0]
        if normalizer is not None:
            normalizer.workflow = self
            normalizer.unlink_all()
            normalizer.link_from(self.loader)
            normalizer.link_attrs(self.loader, ("input", "minibatch_data"))
            first.unlink_all()
            first.link_from(normalizer)
            first.link_attrs(normalizer, ("input", "output"))
        else:
            first.unlink_all()
            first.link_from(self.loader)
            first.link_attrs(self.loader, ("input", "minibatch_data"))
        for prev, cur in zip(self.forwards, self.forwards[1:]):
            cur.unlink_all()
            cur.link_from(prev)
            cur.link_attrs(prev, ("input", "output"))

        self.mergebboxes = MergeBboxes(
            self, labels_compatibility=mcfg.get("labels_compatibility") or None,
            save_raw_file_name=mcfg.get("raw_path", ""),
            **{k: mcfg[k] for k in ("ignore_negative", "max_per_class", "probability_threshold",
                                    "last_chance_probability_threshold", "use_compatibility")
               if k in mcfg})
        self.mergebboxes.link_attrs(self.forwards[-1], ("probabilities", "output"))
        self.mergebboxes.link_attrs(self.loader, "ended", "minibatch_bboxes", "minibatch_size",
                                    "minibatch_images")
        self.json_writer = ResultWriter(
            self, kwargs.get("labels_txt") or cfg.get("labels_txt") or None, self.result_path,
            ignore_negative=self.mergebboxes.ignore_negative,
            labels_mapping=kwargs.get("labels_mapping", {}),
            image_size_fn=lambda p: tuple(reversed(self.loader.image_size(p)))
            if p in self.loader.bboxes else (-1, -1))
        self.mergebboxes.labels_mapping = self.json_writer.labels_mapping
        if mcfg.get("mode"):
            self.mergebboxes.mode = self.json_writer.mode = mcfg["mode"]
        else:
            self.mergebboxes.link_attrs(self.loader, "mode")
            self.json_writer.link_attrs(self.loader, "mode")
        self.mergebboxes.link_from(self.forwards[-1])
        self.repeater.link_from(self.mergebboxes)
        self.json_writer.link_attrs(self.mergebboxes, "winners")
        self.json_writer.link_from(self.mergebboxes)
        self.json_writer.gate_block = ~self.loader.ended
        self.end_point.link_from(self.json_writer)

    @staticmethod
    def _import_trained(path, normalizer):
        from ...core.snapshotter import SnapshotterToFile
        from ...ops.nn_units import ForwardBase
        from ...utils.mean_disp_normalizer import MeanDispNormalizer
        train = SnapshotterToFile.import_file(path)
        forwards = list(getattr(train, "forwards", None) or
                        [u for u in train.units_in_dependency_order if isinstance(u, ForwardBase)])
        if normalizer is None:
            found = [u for u in train if isinstance(u, MeanDispNormalizer)]
            normalizer = found[0] if found else None
        for u in list(train):
            if u not in forwards and u is not normalizer:
                u.unlink_all()
                train.del_ref(u)
        return forwards, normalizer

    # -- the two stages -----------------------------------------------------------------------
    def run_stage(self):
        self.loader.ended <<= False
        self.run()
        return self.json_writer.results

    def run_pipeline(self):
        """merge stage -> final stage; returns the final {picture: detections} dictionary."""
        results = self.run_stage()
        if self.loader.mode != "merge" or not self.result_path:
            return results
        lcfg = self.loader_config
        shutil.copy(self.result_path, self.result_path + ".raw")
        self.loader.angle_step = lcfg.get("angle_step_final", numpy.pi / 12)
        self.loader.min_angle = lcfg.get("min_angle_final", -numpy.pi / 12)
        self.loader.max_angle = lcfg.get("max_angle_final", numpy.pi / 12)
        self.loader.bboxes_file_name = self.result_path
        self.loader.reset()
        if self.loader.total == 0:
            return results
        self.mergebboxes.reset()
        self.json_writer.results = {}
        return self.run_stage()


def shard_range(stream_path, rank, world):
    """[min_index, max_index) of the pickled candidate stream for ``rank`` of ``world``: ranges
    with (nearly) equal numbers of candidate boxes, not pictures (distribute_forward.py:40-85
    printed one command line per slave; under torchrun each rank calls this with its RANK /
    WORLD_SIZE and the per-rank JSON files are combined with ``writer.merge_json``)."""
    counts = []
    with open(stream_path, "rb") as fin:
        while True:
            try:
                counts.append(len(pickle.load(fin)[1]["bbxs"]))
            except EOFError:
                break
    total = sum(counts)
    bounds, acc, target = [0], 0, total / float(max(world, 1))
    for i, c in enumerate(counts):
        acc += c
        if len(bounds) < world and acc >= target * len(bounds):
            bounds.append(i + 1)
    while len(bounds) < world:
        bounds.append(len(counts))
    bounds.append(len(counts))
    return bounds[rank], bounds[rank + 1]


def run_from_config(device="auto"):
    """Entry point driven by ``root.imagenet_forward`` (imagenet_forward.py:365-388); under
    torchrun every rank takes its ``shard_range`` and writes ``<result>.rank<k>.json``."""
    cfg = root.imagenet_forward
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    lcfg = {}
    result_path = cfg.result_path
    if world > 1 and cfg.loader.path_to_bboxes:
        lo, hi = shard_range(cfg.loader.path_to_bboxes, rank, world)
        lcfg.update(min_index=lo, max_index=hi)
        base, ext = os.path.splitext(result_path)
        result_path = "%s.rank%d%s" % (base, rank, ext)        # keeps the .json the final stage reads
    from ...core.workflow import DummyLauncher
    wf = ImagenetForward(DummyLauncher(testing=True), loader_config=lcfg, result_path=result_path)
    wf.initialize(device=device)
    return wf, wf.run_pipeline()
