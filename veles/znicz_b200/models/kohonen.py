"""DemoKohonen sample: 8x8 self-organising map on 1000 2-D points.

Parity: /root/reference/samples/DemoKohonen/kohonen.py:50-154, kohonen_config.py:40-60
(KohonenTrainer + KohonenDecision, 200 epochs, decay lambdas in the config, three SOM
plotters and a Shell unit in the loop). The reference forces the OpenCL backend
(kohonen_config.py:40); here the trainer runs on the H100 kernels (``csrc/som.cu``) or numpy.
"""
from __future__ import annotations

import os

import numpy

from ..core.config import root
from ..loader.base import TEST, VALID, TRAIN, LoaderError
from ..loader.fullbatch import FullBatchLoader
from ..ops import kohonen
from ..ops.nn_units import NNWorkflow
from ..utils import nn_plotting_units
from ..utils.downloader import Downloader
from ..utils.interaction import Shell


def _gradient_decay(t):
    return 0.05 / (1.0 + t * 0.005)


def _radius_decay(t):
    return 1.0 / (1.0 + t * 0.005)


root.kohonen.update({
    "forward": {"shape": (8, 8), "weights_stddev": 0.05, "weights_filling": "uniform"},
    "downloader": {"url": None, "directory": root.common.dirs.datasets,
                   "files": ["kohonen"]},
    "decision": {"snapshot_prefix": "kohonen", "epochs": 200},
    "loader": {"minibatch_size": 10,
               "dataset_file": os.path.join(str(root.common.dirs.datasets), "kohonen",
                                            "kohonen.txt.gz"),
               "force_numpy": False},
    "train": {"gradient_decay": _gradient_decay, "radius_decay": _radius_decay}})


def generate_dataset(path, n=1000, clusters=4, seed=5):
    """2 x n text table (the reference file layout): points around ``clusters`` centres."""
    rs = numpy.random.RandomState(seed)
    centres = rs.uniform(-1, 1, (clusters, 2))
    pts = centres[rs.randint(0, clusters, n)] + rs.randn(n, 2) * 0.08
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    numpy.savetxt(path, pts.T)
    return path


class KohonenLoader(FullBatchLoader):
    MAPPING = "kohonen_demo_loader"

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.dataset_file = kwargs.get("dataset_file")

    def load_data(self):
        file_name = self.dataset_file or root.kohonen.loader.dataset_file
        try:
            data = numpy.loadtxt(file_name)
        except Exception as e:
            raise LoaderError("Could not load data from %s: %s" % (file_name, e))
        if data.ndim != 2 or data.shape[0] != 2:
            raise LoaderError("Data in %s has the invalid shape %s" % (file_name, data.shape))
        self.original_data.reset(numpy.ascontiguousarray(data.T, dtype=self.dtype))
        self.class_lengths[TEST] = self.class_lengths[VALID] = 0
        self.class_lengths[TRAIN] = data.shape[1]


class KohonenWorkflow(NNWorkflow):
    def __init__(self, workflow, **kwargs):
        kwargs.setdefault("name", "Kohonen")
        super().__init__(workflow, **kwargs)
        cfg = root.kohonen
        self.downloader = Downloader(self, url=cfg.downloader.url,
                                     directory=cfg.downloader.directory, files=[])
        self.downloader.link_from(self.start_point)
        self.repeater.link_from(self.downloader)
        self.loader = KohonenLoader(
            self, name="Kohonen fullbatch loader",
            minibatch_size=cfg.loader.minibatch_size,
            dataset_file=kwargs.get("dataset_file", cfg.loader.dataset_file),
            force_numpy=cfg.loader.force_numpy)
        self.loader.link_from(self.repeater)
        self.trainer = kohonen.KohonenTrainer(
            self, shape=cfg.forward.shape, weights_filling=cfg.forward.weights_filling,
            weights_stddev=cfg.forward.weights_stddev,
            gradient_decay=cfg.train.gradient_decay, radius_decay=cfg.train.radius_decay)
        self.trainer.link_from(self.loader)
        self.trainer.link_attrs(self.loader, ("input", "minibatch_data"))
        self.decision = kohonen.KohonenDecision(
            self, max_epochs=kwargs.get("epochs", cfg.decision.epochs))
        self.decision.link_from(self.trainer)
        self.decision.link_attrs(self.loader, "minibatch_class", "last_minibatch",
                                 "class_lengths", "epoch_ended", "epoch_number")
        self.decision.link_attrs(self.trainer, "weights", "winners")
        self.ipython = Shell(self, enabled=kwargs.get("shell", False))
        self.ipython.link_from(self.decision)
        self.ipython.gate_skip = ~self.decision.epoch_ended
        self.repeater.link_from(self.ipython)
        self.ipython.gate_block = self.decision.complete
        self.end_point.link_from(self.decision)
        self.end_point.gate_block = ~self.decision.complete
        self.loader.gate_block = self.decision.complete
        self.plotters = [nn_plotting_units.KohonenHits(self),
                         nn_plotting_units.KohonenInputMaps(self),
                         nn_plotting_units.KohonenNeighborMap(self)]
        for p, src in zip(self.plotters, ("winners_mem", "weights_mem", "weights_mem")):
            p.link_attrs(self.trainer, "shape").link_from(self.ipython)
            p.link_attrs(self.decision, ("input", src))
            p.gate_block = ~self.decision.epoch_ended


def build(launcher=None, **kwargs):
    from ..core.workflow import DummyLauncher
    return KohonenWorkflow(launcher or DummyLauncher(), **kwargs)


def run(load, main):
    load(KohonenWorkflow)
    main()
