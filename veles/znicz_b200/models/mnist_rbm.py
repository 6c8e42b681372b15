"""MnistRBM: CD-1 restricted Boltzmann machine (196 visible, 1000 hidden).
Parity: /root/reference/tests/research/MnistRBM/mnist_rbm.py:60-186, config :43-51.
The reference loads 240 14x14 patches from a .mat file; offline the loader falls back to
down-sampled synthetic digits when ``data_path`` does not exist. Unlike the reference the loader
is not forced onto the host: on CUDA it gathers the minibatch on the device in the compute
type's dtype, which the Binarization output and the reconstruction evaluator then share."""
from __future__ import annotations

import os

import numpy

from ..core.config import root
from ..core.workflow import FireStarter
from ..loader.base import TEST, VALID, TRAIN
from ..loader.fullbatch import FullBatchLoader
from ..ops import rbm_units
from ..ops.nn_units import NNWorkflow
from ..utils.interaction import Shell
from ..workflow.decision import TrivialDecision

root.mnist_rbm.update({
    "all2all": {"weights_stddev": 0.05, "output_sample_shape": 1000},
    "decision": {"max_epochs": 100},
    "snapshotter": {"prefix": "mnist_rbm"},
    "learning_rate": 0.001,
    "cd_k": 1,
    "loader": {"minibatch_size": 128, "force_numpy": False,
               "data_path": os.path.join(str(root.common.dirs.datasets), "rbm_data",
                                         "test_rbm_functional.mat")}})


class MnistRBMLoader(FullBatchLoader):
    MAPPING = "mnist_rbm_loader"

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.data_path = kwargs.get("data_path")
        self.n_samples = kwargs.get("n_samples", 240)

    def load_data(self):
        if self.data_path and os.path.exists(self.data_path):
            import scipy.io
            patches = numpy.asarray(scipy.io.loadmat(self.data_path)["patches"])
        else:
            from ..loader.synthetic import make_classification
            d, _l, _p = make_classification(self.n_samples, (14, 14, 1), 10, 99, 0.2)
            patches = (d.reshape(self.n_samples, -1) > d.mean()).astype(numpy.float32)
        self.original_data.reset(patches.reshape(patches.shape[0], -1).astype(self.dtype))
        self.class_lengths[TEST] = self.class_lengths[VALID] = 0
        self.class_lengths[TRAIN] = patches.shape[0]


class MnistRBMWorkflow(NNWorkflow):
    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        cfg = root.mnist_rbm
        self.repeater.link_from(self.start_point)
        self.loader = MnistRBMLoader(
            self, name="Mnist RBM fullbatch loader",
            minibatch_size=kwargs.get("minibatch_size", cfg.loader.minibatch_size),
            force_numpy=cfg.loader.force_numpy, data_path=cfg.loader.data_path,
            n_samples=kwargs.get("n_samples", 240), normalization_type="none")
        self.loader.link_from(self.repeater)
        self.fire_starter = FireStarter(self)
        self.fire_starter.link_from(self.loader)
        v_size = kwargs.get("v_size", 196)
        h_size = kwargs.get("h_size", cfg.all2all.output_sample_shape)

        b1 = rbm_units.Binarization(self)
        del self.forwards[:]
        self.forwards.append(b1)
        b1.link_from(self.fire_starter)
        b1.link_attrs(self.loader, ("input", "minibatch_data"),
                      ("batch_size", "minibatch_size"))
        a2a = rbm_units.All2AllSigmoid(self, output_sample_shape=h_size,
                                       weights_stddev=cfg.all2all.weights_stddev)
        self.forwards.append(a2a)
        a2a.link_from(b1)
        a2a.link_attrs(b1, ("input", "output"))
        self.evaluator = rbm_units.EvaluatorRBM(self, bias_shape=v_size)
        self.fire_starter.units.add(self.evaluator)
        self.evaluator.link_from(a2a)
        self.evaluator.link_attrs(a2a, "weights", ("input", "output"))
        self.evaluator.link_attrs(b1, ("target", "output"))
        self.evaluator.link_attrs(self.loader, ("batch_size", "minibatch_size"))

        self.decision = TrivialDecision(
            self, max_epochs=kwargs.get("max_epochs", cfg.decision.max_epochs))
        self.decision.link_from(self.evaluator)
        self.decision.link_attrs(self.loader, "minibatch_class", "minibatch_size",
                                 "last_minibatch", "class_lengths", "epoch_ended",
                                 "epoch_number")
        self.ipython = Shell(self, enabled=kwargs.get("shell", False))
        self.ipython.link_from(self.decision)
        self.ipython.gate_skip = ~self.decision.epoch_ended

        del self.gds[:]
        grad = rbm_units.GradientRBM(self, stddev=0.05, v_size=v_size, h_size=h_size,
                                     cd_k=cfg.cd_k)
        self.fire_starter.units.add(grad)
        self.gds.append(grad)
        grad.link_from(self.ipython)
        grad.link_attrs(a2a, ("input", "output"), ("hbias", "bias"), "weights")
        grad.link_attrs(self.loader, ("batch_size", "minibatch_size"))
        grad.link_attrs(self.evaluator, "vbias")
        bw0 = rbm_units.BatchWeights(self, name="BatchWeights #1")
        self.gds.append(bw0)
        bw0.link_from(grad)
        bw0.link_attrs(b1, ("v", "output"))
        bw0.link_attrs(a2a, ("h", "output"))
        bw0.link_attrs(self.loader, ("batch_size", "minibatch_size"))
        bw1 = rbm_units.BatchWeights2(self, name="BatchWeights #2")
        self.gds.append(bw1)
        bw1.link_from(bw0)
        bw1.link_attrs(grad, ("v", "v1"), ("h", "h1"))
        bw1.link_attrs(self.loader, ("batch_size", "minibatch_size"))
        gc = rbm_units.GradientsCalculator(self)
        self.gds.append(gc)
        gc.link_from(bw1)
        gc.link_attrs(bw0, ("hbias0", "hbias_batch"), ("vbias0", "vbias_batch"),
                      ("weights0", "weights_batch"))
        gc.link_attrs(bw1, ("hbias1", "hbias_batch"), ("vbias1", "vbias_batch"),
                      ("weights1", "weights_batch"))
        upd = rbm_units.WeightsUpdater(
            self, learning_rate=kwargs.get("learning_rate", cfg.learning_rate))
        self.gds.append(upd)
        upd.link_from(gc)
        upd.link_attrs(gc, "hbias_grad", "vbias_grad", "weights_grad")
        upd.link_attrs(a2a, "weights", ("hbias", "bias"))
        upd.link_attrs(self.evaluator, "vbias")
        self.repeater.link_from(upd)
        self.end_point.link_from(upd)
        self.end_point.gate_block = ~self.decision.complete
        self.repeater.gate_block = self.decision.complete


def build(launcher=None, **kwargs):
    from ..core.workflow import DummyLauncher
    return MnistRBMWorkflow(launcher or DummyLauncher(), **kwargs)


def run(load, main):
    load(MnistRBMWorkflow)
    main()
