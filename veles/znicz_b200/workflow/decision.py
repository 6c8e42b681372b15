"""Decision units: epoch bookkeeping, best-so-far tracking, early stop, gd_skip.

Parity: /root/reference/decision.py (IDecision :83, DecisionBase :131-291,
TrivialDecision :295, DecisionGD :334-584, DecisionMSE :587-768). Reference quirks
listed in SURVEY §9 are implemented as intended (statistics really reset, the
``[[None]*3]*3`` aliasing removed, no pdb drop at epoch 0).

Data-parallel H100: per-rank metric accumulators are summed / max-ed / min-ed across
ranks right before the epoch logic runs (``dp.reduce_metrics``), the equivalent of the
reference's slave→master metric messages (:511-541,716-738).
"""
from __future__ import annotations

import time

import numpy

from ..core.config import root
from ..core.distributable import IDistributable
from ..core.mutable import Bool
from ..core.registry import make_registry
from ..core.units import Unit
from ..core.workflow import NoMoreJobs
from ..loader.base import CLASS_NAME, TRAIN, VALID, TEST

DecisionsRegistry = make_registry("decisions", loss_key="LOSS")
DecisionsRegistry.decisions = DecisionsRegistry.registry


def nvl(x, none_vle):
    return none_vle if x is None else x


def nmax(x, y, none_vle=None):
    return none_vle if x is None and y is None else max(nvl(x, y), nvl(y, x))


def pt_str(x, percent_sign=True):
    return "None" if x is None else ("%.2f%%" if percent_sign else "%.2f") % x


def rpt_str(x):
    return "None" if x is None else "%.2f%%" % (100.0 - x)


def _default_eval_transform(valid_fitness, train_fitness):
    return valid_fitness


class IDecision(object):
    __required__ = ("on_run", "on_last_minibatch", "improve_condition",
                    "on_training_finished", "fill_statistics",
                    "fill_snapshot_suffixes", "stop_condition")


class DecisionBase(Unit, metaclass=DecisionsRegistry):
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        kwargs["view_group"] = kwargs.get("view_group", "TRAINER")
        self.complete = Bool(False)
        super().__init__(workflow, **kwargs)
        self.verify_interface(IDecision)
        self.max_epochs = kwargs.get("max_epochs", None)
        self.improved = Bool(False)
        self.improved_epoch_number = None
        self.train_improved = Bool(False)
        self.snapshot_suffix = ""
        self.demand("last_minibatch", "minibatch_class", "class_lengths",
                    "epoch_number", "epoch_ended")

    def init_unpickled(self):
        super().init_unpickled()
        self.epoch_timestamp_ = False
        self.dp_ = None   # parallel.DataParallel context (set by the workflow)

    @property
    def max_epochs(self):
        return self._max_epochs

    @max_epochs.setter
    def max_epochs(self, value):
        ok_type = value is None or (isinstance(value, int) and not isinstance(value, bool))
        if not ok_type:
            raise TypeError("max_epochs: int >= 1 or None expected, got %r" % (value,))
        if value is not None and value < 1:
            raise ValueError("max_epochs: int >= 1 or None expected, got %r" % (value,))
        self._max_epochs = value

    def initialize(self, **kwargs):
        if self.max_epochs is not None:
            self.info("Will allow max %d epochs", self.max_epochs)
        if self.testing:
            self.improved <<= False
            self.train_improved <<= False
            self.complete <<= False

    def run(self):
        if self.epoch_timestamp_ is False:
            self.epoch_timestamp_ = time.time()
        self.on_run()
        if self.is_slave:
            self.complete <<= True
            self.on_last_minibatch()
            self._print_statistics()
        elif bool(self.last_minibatch):
            self._on_last_minibatch()

    # -- IDistributable ---------------------------------------------------------------
    def generate_data_for_master(self):
        data = {}
        self.on_generate_data_for_master(data)
        return data

    def generate_data_for_slave(self, slave=None):
        if bool(self.complete):
            raise NoMoreJobs()
        data = {}
        self.on_generate_data_for_slave(data)
        return data

    def apply_data_from_master(self, data):
        self.complete <<= False
        self.on_apply_data_from_master(data)

    def apply_data_from_slave(self, data, slave=None):
        if slave is None and data is None:
            return
        self.on_apply_data_from_slave(data, slave)
        if bool(self.last_minibatch):
            self._on_last_minibatch()

    def drop_slave(self, slave=None):
        pass

    def on_generate_data_for_master(self, data):
        pass

    def on_generate_data_for_slave(self, data):
        pass

    def on_apply_data_from_master(self, data):
        pass

    def on_apply_data_from_slave(self, data, slave):
        pass

    # -- epoch logic --------------------------------------------------------------------
    def _on_last_minibatch(self):
        """End of one sample class. At the end of an epoch the hooks decide, in this order:
        did train improve, did the tracked (minimax) error improve, what is the snapshot called,
        are we done."""
        self.on_last_minibatch()
        if self.epoch_ended:
            self._close_epoch()
        if self.minibatch_class == TRAIN:
            self.on_training_finished()
        self._print_statistics()

    def _close_epoch(self):
        train_better = bool(self.train_improve_condition())
        better = bool(self.improve_condition())
        self.train_improved <<= train_better
        self.improved <<= better
        if better:
            self.improved_epoch_number = self.epoch_number
        parts = []
        self.fill_snapshot_suffixes(parts)
        self.snapshot_suffix = "_".join(parts)
        self.complete <<= self._stop_condition()

    def _stop_condition(self):
        if self.testing:
            return True
        return self.stop_condition() or (
            self.max_epochs is not None and self.epoch_number >= self.max_epochs)

    def _print_statistics(self):
        stats = []
        self.fill_statistics(stats)
        timestamp = time.time()
        t0 = self.epoch_timestamp_ or timestamp
        self.info("Epoch %d class %s %s in %.2f sec", self.epoch_number,
                  CLASS_NAME[self.minibatch_class], " ".join(stats), timestamp - t0)
        self.epoch_timestamp_ = timestamp

    # defaults
    def on_run(self):
        pass

    def on_last_minibatch(self):
        pass

    def improve_condition(self):
        return False

    def train_improve_condition(self):
        return False

    def on_training_finished(self):
        pass

    def fill_statistics(self, stats):
        pass

    def fill_snapshot_suffixes(self, suffixes):
        pass

    def stop_condition(self):
        return False


class TrivialDecision(DecisionBase):
    pass


class DecisionGD(DecisionBase):
    """Rules the gradient-descent learning process (softmax / classification)."""
    MAPPING = "decision_gd"
    LOSS = "softmax"
    BIGNUM = 1.0e30

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.fail_iterations = kwargs.get("fail_iterations", 100)
        self.gd_skip = Bool()
        self.epoch_n_err = [None] * 3
        self.epoch_n_evaluated_samples = [0] * 3
        self.epoch_n_err_pt = [None] * 3
        self.best_n_err_pt = [None] * 3
        self.best_n_err_pt_epoch_number = [None] * 3
        self.best_n_err_pt_others = [[None] * 3 for _ in range(3)]
        self._store_best_n_err_pt_others = [False] * 3
        self.best_minimax_n_err_pt = [None] * 3
        self.best_minimax_n_err_pt_epoch_number = -1
        self.minibatch_n_err = None
        self.minibatch_confusion_matrix = None
        self.minibatch_max_err_y_sum = None
        self.confusion_matrixes = [None] * 3
        self.max_err_y_sums = [0] * 3
        self.autoencoder = False
        self.demand("minibatch_size")

    def initialize(self, **kwargs):
        super().initialize(**kwargs)
        if not kwargs.get("snapshot", False):
            self.epoch_n_err[:] = [None] * 3
            self.epoch_n_evaluated_samples[:] = [0] * 3
            self.epoch_n_err_pt[:] = [None] * 3
            for i in range(3):
                self.reset_statistics(i)
        cm = self.minibatch_confusion_matrix
        if cm is not None and cm:
            for i in range(3):
                if self.confusion_matrixes[i] is None or \
                        self.confusion_matrixes[i].size != cm.size:
                    self.confusion_matrixes[i] = numpy.zeros_like(cm.mem)

    def get_metric_names(self):
        if not self.testing:
            return {"Min errors", "Accuracy", "EvaluationFitness", "Best epoch"}
        return set()

    def get_metric_values(self):
        if self.testing:
            return {}
        tstr = CLASS_NAME[TRAIN]
        vstr = CLASS_NAME[VALID]
        cstr = "minimax(%s, %s)" % (tstr, vstr)
        evalfun = root.common.get("evaluation_transform") or _default_eval_transform
        mm = nmax(self.best_minimax_n_err_pt[VALID], self.best_minimax_n_err_pt[TRAIN])
        return {
            "Min errors": {tstr: pt_str(self.best_n_err_pt[TRAIN]),
                           vstr: pt_str(self.best_n_err_pt[VALID]),
                           cstr: pt_str(mm)},
            "Accuracy": {tstr: rpt_str(self.best_n_err_pt[TRAIN]),
                         vstr: rpt_str(self.best_n_err_pt[VALID]),
                         cstr: rpt_str(mm)},
            "EvaluationFitness": evalfun(
                1 - nvl(self.best_n_err_pt[VALID], 100) / 100,
                1 - nvl(self.best_n_err_pt[TRAIN], 100) / 100),
            "Best epoch": {
                tstr: nvl(self.best_n_err_pt_epoch_number[TRAIN], "None"),
                vstr: nvl(self.best_n_err_pt_epoch_number[VALID], "None"),
                cstr: nvl(self.best_minimax_n_err_pt_epoch_number, "None")}}

    def on_run(self):
        self.gd_skip <<= (self.minibatch_class != TRAIN)

    def _reduce_across_ranks(self):
        dp = self.dp_
        if dp is None or dp.world_size == 1:
            return
        if dp.symm is None:
            # host-side collectives follow: find a dead rank here, with its number in the error,
            # rather than as a hang inside the reduction (the on-device flag barriers of the
            # fused path trap on their own after ZN_PEER_TIMEOUT_NS)
            dp.check_ranks()
        dp.reduce_metrics(n_err=self.minibatch_n_err,
                          confusion=self.minibatch_confusion_matrix,
                          max_err=self.minibatch_max_err_y_sum,
                          mse_metrics=getattr(self, "minibatch_metrics", None))

    def on_last_minibatch(self):
        self._reduce_across_ranks()
        mc = self.minibatch_class
        cm = self.minibatch_confusion_matrix
        if cm is not None and cm:
            cm.map_read()
            if self.confusion_matrixes[mc] is None:
                self.confusion_matrixes[mc] = numpy.zeros_like(cm.mem)
            self.confusion_matrixes[mc][:] = cm.mem
        ne = self.minibatch_n_err
        if ne is not None and ne:
            ne.map_read()
            self.epoch_n_err[mc] = int(ne.mem[0])
            self.epoch_n_evaluated_samples[mc] = int(ne.mem[1])
            if self.class_lengths[mc] and self.epoch_n_evaluated_samples[mc]:
                self.epoch_n_err_pt[mc] = (100.0 * self.epoch_n_err[mc] /
                                           self.epoch_n_evaluated_samples[mc])
                if self.epoch_n_err_pt[mc] < nvl(self.best_n_err_pt[mc], self.BIGNUM):
                    self.best_n_err_pt[mc] = self.epoch_n_err_pt[mc]
                    self.best_n_err_pt_epoch_number[mc] = self.epoch_number
                    self._store_best_n_err_pt_others[mc] = True
        me = self.minibatch_max_err_y_sum
        if me is not None and me:
            me.map_read()
            self.max_err_y_sums[mc] = float(me.mem[0])

    def improve_condition(self):
        """Called at the end of an epoch; ``minibatch_class`` is VALID when a
        validation set exists, else TRAIN. Minimax rule over (valid, train)."""
        for i, store in enumerate(self._store_best_n_err_pt_others):
            if store:
                self.best_n_err_pt_others[i][:] = self.epoch_n_err_pt
                self._store_best_n_err_pt_others[i] = False
        # minimax: the worse of (this class, TRAIN) must beat the best such pair seen so far
        cls = self.minibatch_class
        now, best = self.epoch_n_err_pt, self.best_minimax_n_err_pt
        if not nmax(now[cls], now[TRAIN], self.BIGNUM) < nmax(best[cls], best[TRAIN], self.BIGNUM):
            return False
        best[cls], best[TRAIN], best[TEST] = now[cls], now[TRAIN], now[TEST]
        self.best_minimax_n_err_pt_epoch_number = self.epoch_number
        return True

    def train_improve_condition(self):
        now = nvl(self.epoch_n_err_pt[TRAIN], self.BIGNUM)
        if not now < nvl(self.best_n_err_pt[TRAIN], self.BIGNUM):
            return False
        self.best_n_err_pt[TRAIN] = self.epoch_n_err_pt[TRAIN]
        self.best_n_err_pt_epoch_number[TRAIN] = self.epoch_number
        self._store_best_n_err_pt_others[TRAIN] = True
        return True

    _SLAVE_PAYLOAD = ("minibatch_n_err", "minibatch_max_err_y_sum", "minibatch_confusion_matrix")

    def on_generate_data_for_master(self, data):
        for name in self._SLAVE_PAYLOAD:
            arr = getattr(self, name)
            if arr:
                arr.map_read()
                data[name] = numpy.array(arr.mem, copy=True)

    def on_generate_data_for_slave(self, data):
        data["improved"] = bool(self.improved)

    def on_apply_data_from_master(self, data):
        self.improved <<= data["improved"]
        self.reset_statistics(self.minibatch_class)
        self.best_minimax_n_err_pt[VALID] = 0
        self.best_minimax_n_err_pt[TRAIN] = 0

    def on_apply_data_from_slave(self, data, slave):
        # counts and the confusion matrix add up, the gradient-norm watermark is a maximum
        merge = {"minibatch_n_err": numpy.add, "minibatch_confusion_matrix": numpy.add,
                 "minibatch_max_err_y_sum": numpy.maximum}
        for name, op in merge.items():
            arr = getattr(self, name)
            if arr and name in data:
                arr.map_write()
                op(arr.mem, data[name], out=arr.mem)

    def stop_condition(self):
        if all(nvl(self.best_minimax_n_err_pt[i], 0) <= 0 for i in (VALID, TRAIN)):
            return True
        if self.improved_epoch_number is not None and (
                self.epoch_number - self.improved_epoch_number > self.fail_iterations):
            return True
        return False

    def fill_statistics(self, ss):
        mc = self.minibatch_class
        if self.minibatch_n_err is not None and self.minibatch_n_err and \
                not self.autoencoder and self.epoch_n_err[mc] is not None:
            ss.append("n_err %d of %d (%.2f%%)" % (
                self.epoch_n_err[mc], self.epoch_n_evaluated_samples[mc],
                nvl(self.epoch_n_err_pt[mc], 0.0)))
        if not self.is_slave:
            self.reset_statistics(mc)

    def fill_snapshot_suffixes(self, ss):
        if self.minibatch_n_err is not None and self.minibatch_n_err:
            for set_samples in (TEST, VALID, TRAIN):
                if self.epoch_n_err_pt[set_samples] is not None:
                    ss.append("%s_%s" % (CLASS_NAME[set_samples],
                                         pt_str(self.epoch_n_err_pt[set_samples], False)))

    def reset_statistics(self, minibatch_class):
        for vec in (self.minibatch_n_err, self.minibatch_max_err_y_sum,
                    self.minibatch_confusion_matrix):
            if vec is None or not vec:
                continue
            vec.map_invalidate()
            vec.mem[:] = 0
            vec.unmap()


class DecisionMSE(DecisionGD):
    """Rules the MSE learning process (regression / autoencoders)."""
    MAPPING = "decision_mse"
    LOSS = "mse"

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.epoch_mse = [None] * 3
        self.best_mse = [None] * 3
        self.best_mse_epoch_number = [None] * 3
        self.best_mse_others = [[None] * 3 for _ in range(3)]
        self._store_best_mse_others = [False] * 3
        self.best_minimax_mse = [None] * 3
        self.best_minimax_mse_epoch_number = -1
        self.epoch_metrics = [None] * 3
        self.root = kwargs.get("root", True)
        self.minibatch_mse = None
        self.demand("minibatch_metrics", "minibatch_class", "class_lengths")

    def initialize(self, **kwargs):
        super().initialize(**kwargs)
        mm = self.minibatch_metrics
        for i in range(3):
            if self.epoch_metrics[i] is None or (
                    mm and self.epoch_metrics[i].size != mm.size):
                self.epoch_metrics[i] = numpy.zeros(3, dtype=numpy.float64)

    def get_metric_names(self):
        if self.testing:
            return set()
        names = set(super().get_metric_names())
        mstr = "RMSE" if self.root else "MSE"
        tstr, vstr = CLASS_NAME[TRAIN], CLASS_NAME[VALID]
        names.update({mstr, "Min %s epochs number" % mstr,
                      "%s %s on min %s %s" % (tstr, mstr, vstr, mstr),
                      "EvaluationFitness"})
        return names

    def get_metric_values(self):
        if self.testing:
            return {}
        values = super().get_metric_values()
        mstr = "RMSE" if self.root else "MSE"
        tstr, vstr = CLASS_NAME[TRAIN], CLASS_NAME[VALID]
        cstr = "minimax(%s, %s)" % (tstr, vstr)
        evalfun = root.common.get("evaluation_transform") or _default_eval_transform

        def fmt(x):
            return "None" if x is None else "%.12f" % x
        values.update({
            mstr: {tstr: fmt(self.best_mse[TRAIN]), vstr: fmt(self.best_mse[VALID]),
                   cstr: fmt(nmax(self.best_minimax_mse[VALID],
                                  self.best_minimax_mse[TRAIN]))},
            "EvaluationFitness": evalfun(-nvl(self.best_minimax_mse[VALID], self.BIGNUM),
                                         -nvl(self.best_minimax_mse[TRAIN], self.BIGNUM)),
            "Min %s epochs number" % mstr: {
                tstr: self.best_mse_epoch_number[TRAIN],
                vstr: self.best_mse_epoch_number[VALID],
                cstr: self.best_minimax_mse_epoch_number},
            "%s %s on min %s %s" % (tstr, mstr, vstr, mstr):
                self.best_mse_others[VALID][TRAIN]})
        return values

    def on_last_minibatch(self):
        super().on_last_minibatch()
        mc = self.minibatch_class
        self.minibatch_metrics.map_read()
        self.epoch_metrics[mc][:] = self.minibatch_metrics.mem
        if self.class_lengths[mc]:
            self.epoch_metrics[mc][0] /= self.class_lengths[mc]
        if self.epoch_number == 0 and mc == VALID:
            self.epoch_metrics[TRAIN][:] = self.epoch_metrics[VALID]

    def improve_condition(self):
        if (nvl(self.epoch_metrics[VALID][0], self.BIGNUM) <
                nvl(self.best_mse[VALID], self.BIGNUM)) and self.class_lengths[VALID]:
            self.best_mse[VALID] = float(self.epoch_metrics[VALID][0])
            self.best_mse_epoch_number[VALID] = self.epoch_number
            self._store_best_mse_others[VALID] = True
        for i, store in enumerate(self._store_best_mse_others):
            if store:
                self.best_mse_others[i][:] = [float(x[0]) for x in self.epoch_metrics]
                self._store_best_mse_others[i] = False
        mc = self.minibatch_class
        if (nmax(self.epoch_metrics[mc][0], self.epoch_metrics[TRAIN][0], self.BIGNUM) <
                nmax(self.best_minimax_mse[mc], self.best_minimax_mse[TRAIN],
                     self.BIGNUM)):
            for i in (mc, TRAIN, TEST):
                self.best_minimax_mse[i] = float(self.epoch_metrics[i][0])
            self.best_minimax_mse_epoch_number = self.epoch_number
            return True
        return super().improve_condition()

    def train_improve_condition(self):
        if (nvl(self.epoch_metrics[TRAIN][0], self.BIGNUM) <
                nvl(self.best_mse[TRAIN], self.BIGNUM)):
            self.best_mse[TRAIN] = float(self.epoch_metrics[TRAIN][0])
            self.best_mse_epoch_number[TRAIN] = self.epoch_number
            self._store_best_mse_others[TRAIN] = True
            return True
        return super().train_improve_condition()

    def on_generate_data_for_master(self, data):
        super().on_generate_data_for_master(data)
        mm = self.minibatch_metrics
        if mm is not None and mm:
            mm.map_read()
            data["minibatch_metrics"] = mm.mem.copy()

    def on_apply_data_from_master(self, data):
        super().on_apply_data_from_master(data)
        self.best_minimax_mse[TRAIN] = 0
        self.best_minimax_mse[VALID] = 0

    def on_apply_data_from_slave(self, data, slave):
        super().on_apply_data_from_slave(data, slave)
        mm = self.minibatch_metrics
        if mm is not None and mm and "minibatch_metrics" in data:
            mm.map_write()
            d = data["minibatch_metrics"]
            mm.mem[0] += d[0]
            mm.mem[1] = max(mm.mem[1], d[1])
            mm.mem[2] = min(mm.mem[2], d[2])

    def fill_snapshot_suffixes(self, ss):
        if self.minibatch_metrics is not None:
            for mc in (VALID, TRAIN):
                if self.epoch_metrics[mc] is not None:
                    ss.append("%.4f" % self.epoch_metrics[mc][0])
        super().fill_snapshot_suffixes(ss)

    def fill_statistics(self, ss):
        mc = self.minibatch_class
        if self.epoch_metrics[mc] is not None:
            ss.append("%s %.6f (max %.6f; min %.3e)" % (
                ("RMSE" if self.root else "MSE",) + tuple(self.epoch_metrics[mc])))
        super().fill_statistics(ss)

    def reset_statistics(self, minibatch_class):
        super().reset_statistics(minibatch_class)
        mm = getattr(self, "minibatch_metrics", None)
        if mm is not None and mm:
            mm.map_invalidate()
            mm.mem[0] = 0
            mm.mem[1] = 0
            mm.mem[2] = 1.0e30
            mm.unmap()

    def stop_condition(self):
        if all(nvl(self.best_minimax_mse[i], 0) <= 0 for i in (VALID, TRAIN)):
            return True
        if self.improved_epoch_number is not None and (
                self.epoch_number - self.improved_epoch_number > self.fail_iterations):
            return True
        return False
