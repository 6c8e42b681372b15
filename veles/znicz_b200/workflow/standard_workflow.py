"""StandardWorkflow: the self-constructing training loop.

Parity: /root/reference/standard_workflow.py (StandardWorkflow :81, ``create_workflow``
:173, ``extract_forward_workflow`` :210, ``link_gds`` :289, ``link_avatar`` :386,
``link_evaluator`` :413, ``link_decision`` :451, ``link_snapshotter`` :493,
``link_end_point`` :518, ``link_image_saver`` :533, ``link_lr_adjuster`` :573,
``link_rollback`` :594, ``link_meandispnorm`` :603, ``link_gd_diff_stats`` :626,
``link_ipython`` :648, ``link_publisher`` :663, plotters :672-1101,
``link_result_unit`` :1103, ``link_data_saver`` :1121, ForwardWorkflowExtractor :1175).

The loop is ``Repeater → Loader → forwards → Evaluator → Decision → Snapshotter →
GDs → Repeater`` with ``EndPoint`` gated on ``~decision.complete``.

H100 additions: after ``initialize`` on a CUDA device the forward chain (+evaluator)
and the GD chain are wrapped into two :class:`GraphSegment` s — the python unit graph
still decides *what* runs each minibatch, a captured CUDA graph removes the per-unit
launch overhead — and, when launched under ``torchrun``, a
:class:`~veles.znicz_b200.parallel.DataParallel` context turns every GD unit's
update into the fused cross-GPU reduce+update kernel.
"""
from __future__ import annotations

import os

from collections import namedtuple

from ..core.avatar import Avatar
from ..core.config import root
from ..core.distributable import TriviallyDistributable
from ..core.snapshotter import SnapshotterRegistry
from ..core.units import Unit
from ..ops import nn_units  # noqa: F401
from ..ops.all2all import All2AllSoftmax
from ..ops.conv import ConvolutionalBase
from ..ops.gd_pooling import GDPooling
from ..ops.nn_units import NNSnapshotterToFile  # noqa: F401 (registers "nnfile")
from . import lr_adjust
from .decision import DecisionsRegistry
from .evaluator import EvaluatorsRegistry
from .nn_rollback import NNRollback
from .standard_workflow_base import StandardWorkflowBase, BaseWorkflowConfig

StandardWorkflowConfig = namedtuple(
    "StandardWorkflowConfig",
    ("decision", "snapshotter", "image_saver", "evaluator", "data_saver",
     "result_loader", "weights_plotter", "similar_weights_plotter",
     "lr_adjuster", "downloader", "publisher", "rollback")
    + BaseWorkflowConfig._fields)


class StandardWorkflow(StandardWorkflowBase):
    """
    Arguments:
        loss_function: "softmax" or "mse" (selects evaluator/decision)
        decision_name / evaluator_name / snapshotter_name / result_loader_name
        <unit>_config: kwargs for the unit
    """
    WorkflowConfig = StandardWorkflowConfig
    CONFIGURABLE_UNIT_NAMES = ("result_loader", "decision", "evaluator", "snapshotter")

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.result_unit_factory = kwargs.get("result_unit_factory")
        self._loss_function = None
        self.loss_function = kwargs.get("loss_function", None)
        self._decision_name = self._evaluator_name = None
        self.result_loader_name = kwargs.get("result_loader_name")
        self.snapshotter_name = kwargs.get("snapshotter_name")
        self.decision_name = kwargs.get("decision_name")
        self.evaluator_name = kwargs.get("evaluator_name")
        self.use_graphs = kwargs.get("use_graphs", root.common.engine.get("graphs", True))
        self.create_workflow()

    def init_unpickled(self):
        super().init_unpickled()
        self.segments_ = []
        self.dp_ = None
        self.fused_step_ = None

    # -- names ---------------------------------------------------------------------------------
    @property
    def loss_function(self):
        return self._loss_function

    @loss_function.setter
    def loss_function(self, value):
        if value not in ("softmax", "mse", None):
            raise ValueError("Unknown loss function type %s" % value)
        self._loss_function = value

    def _set_name_of_unit(self, value, name, mapping):
        if value is None and self.loss_function is None and not self.preprocessing:
            raise ValueError("%s name or loss function must be defined" % name)
        if value is None and self.loss_function is not None:
            value = mapping[self.loss_function]
        elif value is not None and self.loss_function is not None:
            self.debug("Both loss function and %s name are defined; the name wins", name)
        setattr(self, "_%s_name" % name, value)

    decision_name = property(
        lambda self: self._decision_name,
        lambda self, v: self._set_name_of_unit(v, "decision",
                                               DecisionsRegistry.loss_mapping))
    evaluator_name = property(
        lambda self: self._evaluator_name,
        lambda self, v: self._set_name_of_unit(v, "evaluator",
                                               EvaluatorsRegistry.loss_mapping))

    # -- construction -----------------------------------------------------------------------------
    def link_forwards(self, init_attrs, *parents):
        last_fwd = super().link_forwards(init_attrs, *parents)
        if self.loss_function == "mse" and isinstance(last_fwd, All2AllSoftmax):
            raise NotImplementedError(
                "Softmax last layer does not currently support MSE.")
        return last_fwd

    def create_workflow(self):
        self.link_repeater(self.start_point)
        self.link_loader(self.repeater)
        self.link_forwards(("input", "minibatch_data"), self.loader)
        self.link_evaluator(self.forwards[-1])
        self.link_decision(self.evaluator)
        self.link_snapshotter(self.decision)
        last_gd = self.link_gds(self.snapshotter)
        if self.loss_function == "mse":
            last_err = self.link_min_max_plotter(False, self.link_min_max_plotter(
                True, self.link_mse_plotter(last_gd)))
        elif self.loss_function == "softmax":
            last_err = self.link_error_plotter(last_gd)
        else:
            last_err = last_gd
        self.link_loop(last_err)
        self.link_end_point(last_gd)

    def extract_forward_workflow(self, loader_unit_factory=None, loader_name=None,
                                 loader_config=None, result_unit_factory=None,
                                 result_unit_config=None, cyclic=True):
        """Build a forward-only workflow carrying the trained weights
        (/root/reference/standard_workflow.py:210-286)."""
        if loader_unit_factory is not None:
            assert loader_name is None and loader_config is None
            wf = StandardWorkflowBase(self.workflow, name="Forwards@%s" % self.name,
                                      loader_factory=loader_unit_factory,
                                      layers=self.layers)
        else:
            wf = StandardWorkflowBase(self.workflow, name="Forwards@%s" % self.name,
                                      loader_name=loader_name,
                                      loader_config=loader_config, layers=self.layers)
        start_unit = wf.link_repeater(wf.start_point) if cyclic else wf.start_point
        wf.link_loader(start_unit)
        wf.loader.derive_from(self.real_loader)
        if cyclic:
            wf.end_point.link_from(wf.loader).gate_block = ~wf.loader.complete
        wf.link_forwards(("input", "minibatch_data"), wf.loader)
        if cyclic:
            wf.forwards[0].gate_block = wf.loader.complete
        result_unit_config = self.config2kwargs(result_unit_config)
        if result_unit_factory is not None:
            wf.result_unit = result_unit_factory(wf, **result_unit_config) \
                .link_from(wf.forwards[-1])
            wf.result_unit.link_attrs(wf.forwards[-1], ("input", "output"))
            wf.result_unit.link_attrs(
                wf.loader, ("labels_mapping", "reversed_labels_mapping"))
            if self.loss_function == "mse":
                wf.result_unit.link_attrs(wf.loader, "target_normalizer")
            last_unit = wf.result_unit
        else:
            last_unit = wf.forwards[-1]
        if cyclic:
            wf.repeater.link_from(last_unit)
        else:
            wf.link_end_point(last_unit)
        for fwd_exp, fwd_imp in zip(self.forwards, wf.forwards):
            gen = getattr(fwd_exp, "generate_data_for_slave", None)
            app = getattr(fwd_imp, "apply_data_from_master", None)
            if gen is not None and app is not None:
                app(gen(None))
            fwd_imp.forward_mode = True
        return wf

    @StandardWorkflowBase.check_forward_units
    def link_gds(self, *parents):
        """Create GD units in reverse order, chain ``err_output ← err_input`` and
        share input/weights/bias/output/input_offset/mask with the forward units."""
        if not isinstance(self.layers, (tuple, list)):
            raise ValueError("layers should be a list of dicts")
        self.gds[:] = (None,) * len(self.layers)
        first_gd = None
        units_to_delete = []
        for i, layer in reversed(list(enumerate(self.layers))):
            tpe, _, kwargs = self._get_layer_type_kwargs(layer)
            if not isinstance(self.forwards[i], self.layer_map[tpe].forward):
                raise ValueError(
                    "Forward layer %s at position %d is not an instance of %s" %
                    (self.forwards[i], i, self.layer_map[tpe].forward))
            if "name" in kwargs:
                kwargs["name"] = "gd_" + kwargs["name"]
            try:
                unit = next(self.layer_map[tpe].backwards)(self, **kwargs)
            except StopIteration:
                units_to_delete.append(i)
                continue
            self.gds[i] = unit
            if first_gd is not None:
                unit.link_from(first_gd).link_attrs(first_gd, ("err_output", "err_input"))
            else:
                unit.link_from(*parents).link_attrs(self.evaluator, "err_output")
            first_gd = unit
            try_link_attrs = {"input", "weights", "bias", "input_offset", "mask", "output"}
            if isinstance(unit, ConvolutionalBase):
                try_link_attrs.update(ConvolutionalBase.CONV_ATTRS)
            if isinstance(unit, GDPooling):
                try_link_attrs.update(GDPooling.POOL_ATTRS)
            try_link_attrs.update(getattr(self.forwards[i], "GD_LINK_ATTRS", ()))
            attrs = [a for a in sorted(try_link_attrs) if hasattr(self.forwards[i], a)]
            unit.link_attrs(self.forwards[i], *attrs)
            unit.forward_unit = self.forwards[i]
            unit.gate_skip = self.decision.gd_skip
        for i in sorted(units_to_delete, reverse=True):
            del self.gds[i]
        self.gds[0].need_err_input = False
        return first_gd

    def link_loop(self, parent):
        self.repeater.link_from(parent)

    def link_avatar(self, *extra_attrs):
        """Replace the loader with its avatar (loader runs ahead of the contour)."""
        self.loader.ignores_gate <<= True
        self.avatar = Avatar(self)
        self.avatar.reals[self.loader] = tuple(self.loader.exports) + extra_attrs
        self.avatar.clone()
        self.avatar.link_from(self.loader)
        self.loader.link_from(self.avatar)
        self.avatar.link_from(self.repeater).gate_block = self.loader.gate_block
        self._loader = self.avatar
        return self.avatar

    def link_downloader(self, *parents):
        from ..utils.downloader import Downloader
        self.downloader = Downloader(self, **self.config.downloader).link_from(*parents)
        return self.downloader

    @StandardWorkflowBase.reset_unit
    @StandardWorkflowBase.check_forward_units
    def link_evaluator(self, *parents):
        cls = EvaluatorsRegistry.registry[self.evaluator_name]
        self.evaluator = cls(self, **self.config.evaluator) \
            .link_from(*parents) \
            .link_attrs(self.forwards[-1], "output") \
            .link_attrs(self.loader, ("batch_size", "minibatch_size"),
                        ("labels", "minibatch_labels"),
                        ("max_samples_per_epoch", "total_samples"),
                        "class_lengths", ("offset", "minibatch_offset"))
        if hasattr(self.loader, "reversed_labels_mapping"):
            self.evaluator.link_attrs(
                self.loader, ("labels_mapping", "reversed_labels_mapping"))
        if hasattr(self.loader, "class_keys"):
            self.evaluator.link_attrs(self.loader, "class_keys")
        if self.evaluator_name == "evaluator_softmax":
            self.evaluator.link_attrs(self.forwards[-1], "max_idx")
        elif self.evaluator_name == "evaluator_mse":
            self.evaluator.link_attrs(
                self.loader, ("target", "minibatch_targets"), "class_targets",
                ("normalizer", "target_normalizer"))
        return self.evaluator

    @StandardWorkflowBase.reset_unit
    def link_decision(self, *parents):
        cls = DecisionsRegistry.registry[self.decision_name]
        self.decision = cls(self, **self.config.decision) \
            .link_from(*parents) \
            .link_attrs(self.loader, "minibatch_class", "last_minibatch",
                        "minibatch_size", "class_lengths", "epoch_ended",
                        "epoch_number")
        if self.decision_name == "decision_mse":
            self.decision.link_attrs(self.loader, "minibatch_offset")
        self.decision.link_attrs(self.evaluator, ("minibatch_n_err", "n_err"))
        if self.decision_name == "decision_gd":
            self.decision.link_attrs(
                self.evaluator, ("minibatch_confusion_matrix", "confusion_matrix"),
                ("minibatch_max_err_y_sum", "max_err_output_sum"))
        elif self.decision_name == "decision_mse":
            self.decision.link_attrs(
                self.evaluator, ("minibatch_metrics", "metrics"),
                ("minibatch_mse", "mse"))
        self.repeater.gate_block = self.decision.complete
        self.real_loader.gate_block = self.decision.complete
        return self.decision

    @StandardWorkflowBase.reset_unit
    def link_snapshotter(self, *parents):
        name = self.snapshotter_name or "nnfile"
        cls = SnapshotterRegistry.registry[name]
        self.snapshotter = cls(self, **self.config.snapshotter) \
            .link_from(*parents) \
            .link_attrs(self.decision, ("suffix", "snapshot_suffix"))
        self.snapshotter.gate_skip = ~self.decision.epoch_ended
        self.snapshotter.skip = ~self.decision.improved
        return self.snapshotter

    def link_end_point(self, *parents):
        self.end_point.link_from(*parents)
        self.end_point.gate_block = ~self.decision.complete
        return self.end_point

    @StandardWorkflowBase.reset_unit
    @StandardWorkflowBase.check_forward_units
    def link_image_saver(self, *parents):
        from ..utils.image_saver import ImageSaver
        self.image_saver = ImageSaver(self, **self.config.image_saver).link_from(*parents)
        if self.evaluator_name == "evaluator_softmax":
            self.image_saver.link_attrs(self.forwards[-1], "max_idx")
        self.image_saver.link_attrs(self.forwards[-1], "output")
        if hasattr(self.loader, "color_space"):
            self.image_saver.link_attrs(self.loader, "color_space")
        if hasattr(self.loader, "reversed_labels_mapping"):
            self.image_saver.link_attrs(self.loader, "reversed_labels_mapping")
        self.image_saver.link_attrs(
            self.loader, ("input", "minibatch_data"), ("indices", "minibatch_indices"),
            ("labels", "minibatch_labels"), "minibatch_class", "minibatch_size")
        if self.evaluator_name == "evaluator_mse":
            self.image_saver.link_attrs(self.loader, ("target", "minibatch_targets"))
        self.image_saver.link_attrs(self.snapshotter, ("this_save_time", "time")) \
            .gate_skip = ~self.decision.improved
        return self.image_saver

    @StandardWorkflowBase.reset_unit
    @StandardWorkflowBase.check_backward_units
    def link_lr_adjuster(self, *parents):
        self.lr_adjuster = lr_adjust.LearningRateAdjust(
            self, **self.dictify(self.config.lr_adjuster))
        for gd_elm in self.gds:
            self.lr_adjuster.add_gd_unit(gd_elm)
        self.lr_adjuster.link_from(*parents)
        return self.lr_adjuster

    @StandardWorkflowBase.reset_unit
    def link_rollback(self, *parents):
        self.rollback = NNRollback(self, **self.config.rollback)
        self.rollback.link_from(*parents)
        self.rollback.improved = self.decision.train_improved
        self.rollback.gate_skip = ~self.loader.epoch_ended | self.decision.complete
        for gd_elm in self.gds:
            self.rollback.add_gd(gd_elm)
        return self.rollback

    @StandardWorkflowBase.reset_unit
    def link_meandispnorm(self, *parents):
        from ..utils.mean_disp_normalizer import MeanDispNormalizer
        self.meandispnorm = MeanDispNormalizer(self) \
            .link_attrs(self.loader, ("input", "minibatch_data"), "mean", "rdisp") \
            .link_from(*parents)
        return self.meandispnorm

    @StandardWorkflowBase.check_backward_units
    def link_gd_diff_stats(self, *parents, **kwargs):
        from ..utils.diff_stats import DiffStats
        self.diff_stats = DiffStats(
            self, arrays={u: ("weights", "bias") for u in self.gds if u is not None},
            file_name=kwargs.get("file_name", "diff_stats.pickle"))
        self.diff_stats.link_from(*parents)
        self.diff_stats.gate_skip = self.decision.gd_skip
        return self.diff_stats

    @StandardWorkflowBase.reset_unit
    def link_ipython(self, *parents):
        from ..utils.interaction import Shell
        self.ipython = Shell(self).link_from(*parents)
        self.ipython.gate_skip = ~self.decision.epoch_ended
        return self.ipython

    @StandardWorkflowBase.reset_unit
    def link_publisher(self, *parents):
        from ..utils.publishing import Publisher
        self.publisher = Publisher(self, **self.config.publisher).link_from(*parents)
        self.publisher.result_providers.add(self.decision)
        self.publisher.loader_unit = self.real_loader
        self.publisher.gate_skip = ~self.decision.complete
        return self.publisher

    # -- plotters (recording units; rendering only when plotting is enabled) -------------------
    def link_error_plotter(self, *parents):
        from ..utils import plotting_units as pu
        self.error_plotter = []
        prev = parents
        styles = ["r-", "b-", "k-"]
        for i in (1, 2):
            p = pu.AccumulatingPlotter(self, name="Errors", plot_style=styles[i])
            p.link_attrs(self.decision, ("input", "epoch_n_err_pt"))
            p.input_field = i
            p.link_from(*prev)
            p.gate_skip = ~self.decision.epoch_ended
            self.error_plotter.append(p)
            prev = (p,)
        return self.error_plotter[-1]

    def link_conf_matrix_plotter(self, *parents):
        from ..utils import plotting_units as pu
        self.conf_matrix_plotter = []
        prev = parents
        for i in (1, 2):
            p = pu.MatrixPlotter(self, name="Confusion matrix %d" % i)
            p.link_attrs(self.decision, ("input", "confusion_matrixes"))
            p.input_field = i
            p.link_from(*prev)
            p.gate_skip = ~self.decision.epoch_ended
            self.conf_matrix_plotter.append(p)
            prev = (p,)
        return self.conf_matrix_plotter[-1]

    def link_err_y_plotter(self, *parents):
        from ..utils import plotting_units as pu
        self.err_y_plotter = []
        prev = parents
        for i in (1, 2):
            p = pu.AccumulatingPlotter(self, name="Last layer max gradient sum")
            p.link_attrs(self.decision, ("input", "max_err_y_sums"))
            p.input_field = i
            p.link_from(*prev)
            p.gate_skip = ~self.decision.epoch_ended
            self.err_y_plotter.append(p)
            prev = (p,)
        return self.err_y_plotter[-1]

    def _has_weights(self, i):
        """Only conv and fully connected layers are plotted
        (/root/reference/standard_workflow.py:899-903)."""
        from ..ops.all2all import All2All
        from ..ops.conv import Conv
        return isinstance(self.forwards[i], (Conv, All2All))

    def link_multi_hist_plotter(self, weights_input, *parents):
        from ..utils import plotting_units as pu
        self.multi_hist_plotter = []
        prev = parents
        for i, (unit, layer) in enumerate(
                zip(self._get_weights_source_units(weights_input), self.layers)):
            if unit is None or not self._has_weights(i):
                continue
            p = pu.MultiHistogram(self, name="Histogram %s %d" % (weights_input, i + 1))
            p.link_attrs(unit, ("input", weights_input))
            p.link_from(*prev)
            p.gate_skip = ~self.decision.epoch_ended
            self.multi_hist_plotter.append(p)
            prev = (p,)
        return prev[0]

    def link_weights_plotter(self, weights_input, *parents):
        from ..utils.nn_plotting_units import Weights2D
        self.weights_plotter = []
        prev = parents
        for i, unit in enumerate(self._get_weights_source_units(weights_input)):
            if unit is None or not self._has_weights(i):
                continue
            p = Weights2D(self, name="%s %d" % (weights_input, i + 1),
                          **self.dictify(self.config.weights_plotter))
            p.link_attrs(unit, ("input", weights_input))
            if hasattr(self.forwards[i], "kx"):
                p.get_shape_from = [self.forwards[i].kx, self.forwards[i].ky,
                                    self.forwards[i].input]
            p.link_from(*prev)
            p.gate_skip = ~self.decision.epoch_ended
            self.weights_plotter.append(p)
            prev = (p,)
        return prev[0]

    def link_similar_weights_plotter(self, weights_input, *parents):
        from ..utils.diversity import SimilarWeights2D
        self.similar_weights_plotter = []
        prev = parents
        for i, unit in enumerate(self._get_weights_source_units(weights_input)):
            if unit is None or not self._has_weights(i):
                continue
            p = SimilarWeights2D(self, name="similar %s %d" % (weights_input, i + 1),
                                 **self.dictify(self.config.similar_weights_plotter))
            p.link_attrs(unit, ("input", weights_input))
            p.link_from(*prev)
            p.gate_skip = ~self.decision.epoch_ended
            self.similar_weights_plotter.append(p)
            prev = (p,)
        return prev[0]

    def link_table_plotter(self, *parents):
        from ..utils import plotting_units as pu
        self.table_plotter = pu.TableMaxMin(self, name="Max, Min")
        for unit in self.forwards:
            for attr in ("weights", "output"):
                if getattr(unit, attr, None) is not None:
                    self.table_plotter.add(unit, attr)
        for unit in self.gds:
            for attr in ("gradient_weights", "err_input"):
                if unit is not None and getattr(unit, attr, None) is not None:
                    self.table_plotter.add(unit, attr)
        self.table_plotter.link_from(*parents)
        self.table_plotter.gate_skip = ~self.decision.epoch_ended
        return self.table_plotter

    def link_mse_plotter(self, *parents):
        from ..utils import plotting_units as pu
        self.mse_plotter = []
        prev = parents
        for i in (1, 2):
            p = pu.AccumulatingPlotter(self, name="mse")
            p.link_attrs(self.decision, ("input", "epoch_metrics"))
            p.input_field = i
            p.input_offset = 0
            p.link_from(*prev)
            p.gate_skip = ~self.decision.epoch_ended
            self.mse_plotter.append(p)
            prev = (p,)
        return self.mse_plotter[-1]

    def link_min_max_plotter(self, is_min, *parents):
        from ..utils import plotting_units as pu
        plotters = []
        prev = parents
        for i in (1, 2):
            p = pu.AccumulatingPlotter(self, name="mse %s" % ("min" if is_min else "max"))
            p.link_attrs(self.decision, ("input", "epoch_metrics"))
            p.input_field = i
            p.input_offset = 2 if is_min else 1
            p.link_from(*prev)
            p.gate_skip = ~self.decision.epoch_ended
            plotters.append(p)
            prev = (p,)
        setattr(self, "min_plotter" if is_min else "max_plotter", plotters)
        return plotters[-1]

    def link_image_plotter(self, *parents):
        from ..utils import plotting_units as pu
        self.image_plotter = pu.ImagePlotter(self, name="output sample")
        self.image_plotter.inputs.append(self.forwards[-1].output)
        self.image_plotter.input_fields.append(0)
        self.image_plotter.link_from(*parents)
        self.image_plotter.gate_skip = ~self.decision.epoch_ended
        return self.image_plotter

    def link_immediate_plotter(self, *parents):
        from ..utils import plotting_units as pu
        self.immediate_plotter = pu.ImmediatePlotter(self, name="ImmediatePlotter")
        self.immediate_plotter.link_from(*parents)
        self.immediate_plotter.gate_skip = ~self.decision.epoch_ended
        return self.immediate_plotter

    def link_result_unit(self):
        self.result_unit = ForwardWorkflowExtractor(
            self, loader_name=self.result_loader_name,
            loader_config=self.config.result_loader,
            result_unit_factory=self.result_unit_factory)
        self.decision.link_from(self.result_unit)
        self.result_unit.gate_block = ~self.decision.complete
        return self.result_unit

    @StandardWorkflowBase.reset_unit
    def link_data_saver(self, *parents):
        from ..loader.saver import MinibatchesSaver
        if self.loss_function not in ("softmax", None):
            raise NotImplementedError("MinibatchSaverMSE's not been written yet")
        self.data_saver = MinibatchesSaver(self, **self.config.data_saver) \
            .link_from(*parents)
        self.data_saver.link_attrs(
            self.loader, "shuffle_limit", "minibatch_class", "minibatch_data",
            "minibatch_labels", "class_lengths", "max_minibatch_size", "has_labels",
            "labels_mapping", "minibatch_size")
        return self.data_saver

    def _get_weights_source_units(self, weights_input):
        if weights_input == "weights":
            self._check_forwards()
            return self.forwards
        if weights_input == "gradient_weights":
            self._check_gds()
            return self.gds
        raise ValueError("weights_input should be 'weights' or 'gradient_weights'")

    # -- H100: CUDA-graph segments + data parallel -------------------------------------------------
    def initialize(self, device=None, **kwargs):
        if device is None or isinstance(device, str):
            from ..core.backends import get_device
            device = get_device(device)
        from . import fusion
        self.fused_activations_ = fusion.fuse_activations(self, device)
        self.fused_derivatives_ = fusion.fuse_backward_derivatives(self, device)
        self.fused_evaluator_ = fusion.fuse_evaluator(self, device)
        res = super().initialize(device=device, **kwargs)
        dev = self.device
        if int(os.environ.get("WORLD_SIZE", "1")) <= 1:
            # a data-parallel snapshot resumed in a single process: back to the whole dataset
            ld = getattr(self, "real_loader", None) or self.loader
            if getattr(ld, "dp_world", 1) > 1:
                ld.shard(0, 1)
        if dev is not None and not dev.is_cuda:
            # CPU multi-process runs (gloo): same sharding / metric reduction, gradients are
            # all-reduced on the host inside the numpy GD step
            from ..parallel import DataParallel
            self.dp_ = DataParallel.from_env(dev)
            if self.dp_ is not None:
                self.dp_.attach(self)
        if dev is not None and dev.is_cuda:
            from ..parallel import DataParallel
            self.dp_ = DataParallel.from_env(dev)
            if self.dp_ is not None:
                self.dp_.attach(self)
            self.fused_step_ = None
            if root.common.engine.get("fused_step", True):
                from ..ops.fused_step import FusedStep
                self.fused_step_ = FusedStep.attach(self, self.dp_)
            if self.use_graphs:
                self._build_segments()
        return res

    def _build_segments(self):
        from ..core.graphs import GraphSegment
        self.segments_ = []
        fwd_units = [u for u in self.forwards] + [self.evaluator]
        if all(getattr(u, "on_cuda", False) for u in fwd_units):
            ld = getattr(self, "real_loader", None) or self.loader
            hook = getattr(ld, "graph_prelude", None)
            pre = hook() if callable(hook) else None
            self.segments_.append(GraphSegment(
                "forward", fwd_units, key_fn=self._segment_key, prelude=[pre] if pre else None))
        gd_units = [u for u in reversed(self.gds) if u is not None]
        if gd_units and all(getattr(u, "on_cuda", False) for u in gd_units):
            self.segments_.append(GraphSegment("backward", gd_units,
                                               key_fn=self._segment_key))
            if len(self.segments_) == 2 and root.common.engine.get("fuse_train_step", True):
                self.segments_[0].fuse_with(self.segments_[1], self._train_step_fusable)

    def _train_step_fusable(self):
        """Forward and backward may run as ONE graph on a steady-state TRAIN minibatch: nothing
        that executes on the host between them (decision, snapshotter, rollback, plotters) acts
        before the last minibatch of the epoch, and the GD gates are open."""
        ld, dec = self.loader, self.decision
        if ld.minibatch_class != 2 or bool(ld.last_minibatch) or bool(dec.complete) or \
                bool(getattr(dec, "gd_skip", False)):
            return False
        g0 = self.segments_[1].units[0]
        return not bool(g0.gate_skip) and not bool(g0.gate_block)

    def _segment_key(self):
        return int(self.loader.minibatch_class == 2)


class ForwardWorkflowExtractor(Unit, TriviallyDistributable):
    """Extracts the forward core of the network when training completes."""

    def __init__(self, workflow, **kwargs):
        assert isinstance(workflow, StandardWorkflow)
        super().__init__(workflow, **kwargs)
        self.loader_name = kwargs["loader_name"]
        self.loader_config = kwargs["loader_config"]
        self.result_unit_factory = kwargs["result_unit_factory"]
        self.result_unit_config = kwargs.get("result_unit_config")
        self.cyclic = kwargs.get("cyclic", False)
        self.forward_workflow = False

    def initialize(self, **kwargs):
        pass

    def run(self):
        self.forward_workflow = self.workflow.extract_forward_workflow(
            loader_name=self.loader_name, loader_config=self.loader_config,
            result_unit_factory=self.result_unit_factory,
            result_unit_config=self.result_unit_config, cyclic=self.cyclic)

    def apply_data_from_slave(self, data, slave=None):
        if not bool(self.gate_block):
            self.run()
