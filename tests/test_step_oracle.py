"""The benchmarked training step, tensor by tensor, against a float64 oracle.

``bench.build_workflow`` builds the system under test exactly as ``bench.py`` times it: on the GPU
that is the HBM-resident loader gather, activations folded into producer epilogues and derivatives
into the consumer's backward kernel (workflow/fusion.py), the softmax evaluator inside the
few-output FC launch, the halo / LSTM persistent kernels, ``multi_update_k`` and the whole step
replayed as one CUDA graph. A hook on the loader's ``run`` checks every training step after it ran:
the same model built on ``device="numpy"`` in float64 is anchored to the device's pre-step state
(fp32 master weights, momentum, the minibatch the device consumed) and its units are driven by hand
through the same step, so each step is an independent check and no drift builds up.

What each device tensor means is derived from the fusion marks: a producer with ``fused_act_``
holds f(y); a GD unit with ``in_deriv_act_`` writes err * f'(y) of the layer below; an activation
unit folded away has no tensor of its own.

Discrete decisions that rounding noise may flip (a max-pool window whose top two values are within
the noise bound, a ReLU gate with |x| inside it, a near-tied softmax row) adopt the device's choice
after checking that the choice is legitimate; the adoptions are counted and must stay rare. A wrong
choice outside the noise band still fails.

The CPU tier runs the same harness with the numpy float32 workflow as the system under test.
"""
import os
import sys
import time

import numpy
import pytest

from veles.znicz_b200.core.config import root
from veles.znicz_b200.core.memory import Array

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

TRAIN = 2
FP32_TOL = 2e-4          # the fp32 bar of tests/test_gpu_units.py
# bf16: the bar is this many times the distance between the exact oracle and a second oracle pass
# that rounds to bf16 wherever the device stores bf16. One rounded pass captures the storage
# rounding but neither the device's other bf16 roundings (LSTM gates, the dgrad / wgrad operand
# shadows) nor its accumulation order; those are of the same order, so 3x covers them while a
# real defect (a wrong row, border or channel: an error of the tensor's own magnitude) still
# exceeds it by far.
BF16_FACTOR = 3.0
BF16_FLOOR = FP32_TOL
# n_train per model: the last minibatch of each epoch is ragged and every class occurs
N_TRAIN = {"cifar_caffe": 250, "mnist_conv": 16, "lstm": 300}
N_CLASSES = {"cifar_caffe": 10, "mnist_conv": 9, "lstm": 10}
EPOCHS = 3


# ------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------
def _host(a):
    if a is None or not isinstance(a, Array) or not a:
        return None
    a.map_read()
    return numpy.array(a.mem, copy=True)


def bf16_round(x):
    """Round to the nearest bf16 (ties to even), returned in float64."""
    f = numpy.ascontiguousarray(x, dtype=numpy.float32)
    u = f.view(numpy.uint32).astype(numpy.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(numpy.uint32).view(numpy.float32).astype(numpy.float64).reshape(f.shape)


def deriv_from_output(code, y):
    """f'(x) expressed through y = f(x) for the fusable activations (workflow/fusion.py)."""
    if code == 1:
        return 1.14381894 - 0.388484177 * y * y
    if code == 2:
        return 1.0 - numpy.exp(-y)
    if code == 3:
        return (y > 0).astype(y.dtype)
    if code == 4:
        return y * (1.0 - y)
    raise ValueError(code)


def errors(a, r, slack=None):
    """(max-abs over max|ref|, relative L2) of ``a`` against ``r``; ``slack`` is an elementwise
    quantum the difference may have without counting (the fp32 resolution of a weight update)."""
    a = numpy.asarray(a, numpy.float64).ravel()
    r = numpy.asarray(r, numpy.float64).ravel()
    scale = max(float(numpy.abs(r).max()) if r.size else 0.0, 1e-30)
    d = a - r
    if slack is not None:
        d = numpy.sign(d) * numpy.maximum(numpy.abs(d) - slack.ravel(), 0.0)
    return (float(numpy.abs(d).max()) / scale if d.size else 0.0,
            float(numpy.linalg.norm(d)) / max(float(numpy.linalg.norm(r)), 1e-30))


def within(a, r, tol, slack=None):
    if not numpy.isfinite(numpy.asarray(a, numpy.float64)).all():
        return False
    e_max, e_l2 = errors(a, r, slack)
    return e_max <= tol and e_l2 <= tol


def perturbed(a, r, tol, index):
    """A copy of ``a`` whose element ``index`` moved by twice the max-abs tolerance, away from
    the reference."""
    b = numpy.array(a, numpy.float64, copy=True)
    scale = float(numpy.abs(r).max())
    d = float(b[index] - r[index])
    b[index] += (1.0 if d >= 0 else -1.0) * 2.0 * tol * scale
    return b


def _gd_of(wf):
    return {id(g.forward_unit): g for g in wf.gds
            if g is not None and getattr(g, "forward_unit", None) is not None}


# ------------------------------------------------------------------------------------------------
# the float64 oracle
# ------------------------------------------------------------------------------------------------
HYPER = ("learning_rate", "learning_rate_bias", "weights_decay", "weights_decay_bias",
         "l1_vs_l2", "l1_vs_l2_bias", "gradient_moment", "gradient_moment_bias", "factor_ortho")


def build(model, compute, device):
    import bench
    wf = bench.build_workflow(False, compute, True, N_TRAIN[model], model)
    wf.initialize(device=device)
    return wf


class Oracle(object):
    """The model on device="numpy" in float64, its units driven by hand (the scheduler never
    runs)."""

    def __init__(self, model):
        root.common.engine.precision_type = "double"
        try:
            self.wf = build(model, "fp32", "numpy")
        finally:
            root.common.engine.precision_type = "float"
        assert self.wf.forwards[-1].output.dtype == numpy.float64

    def step(self, pre, post, sut, noise):
        """One training step from the device's pre-step state; returns {key: array}.
        ``noise`` rounds every tensor the device stores in bf16 to bf16. Decisions within
        ``sut.bound`` adopt the device's choice."""
        wf = self.wf
        rnd = bf16_round if noise else (lambda x: x)
        ld = wf.loader
        ld.minibatch_data.map_write()
        ld.minibatch_data.mem[...] = rnd(post["data"].reshape(ld.minibatch_data.shape))
        ld.minibatch_labels.map_write()
        ld.minibatch_labels.mem[...] = post["labels"]
        ld.minibatch_size = post["batch"]
        ev = wf.evaluator
        for k, v in pre["eval"].items():
            a = getattr(ev, k)
            a.map_write()
            a.mem[...] = v
        gd_of = _gd_of(wf)
        for i, f in enumerate(wf.forwards):
            for part in ("weights", "bias"):
                w = getattr(f, part, None)
                if isinstance(w, Array) and w and (i, part) in pre["w"]:
                    w.map_write()
                    w.mem[...] = pre["w"][(i, part)]
                    g = gd_of.get(id(f))
                    m = getattr(g, "gradient_%s_with_moment" % part, None)
                    if isinstance(m, Array) and m and (i, part) in pre["m"]:
                        m.map_write()
                        m.mem[...] = pre["m"][(i, part)]
            g = gd_of.get(id(f))
            if g is not None:
                for h in HYPER:
                    if h in pre["hyper"].get(i, {}):
                        setattr(g, h, pre["hyper"][i][h])
        out, adopted = {}, {}
        for i, f in enumerate(wf.forwards):
            saved = None
            if noise and isinstance(getattr(f, "weights", None), Array) and f.weights:
                saved = f.weights.mem.copy()          # the bf16 weight shadow the kernels read
                f.weights.mem[...] = rnd(saved)
            f.run()
            if saved is not None:
                f.weights.mem[...] = saved
            adopted.update(sut.align(i, f, post))
            if noise and type(f).__name__ != "All2AllSoftmax":
                f.output.mem[...] = rnd(f.output.mem)
            out[("fwd", i, "output")] = f.output.mem.copy()
            if hasattr(f, "max_idx") and isinstance(f.max_idx, Array) and f.max_idx:
                out[("fwd", i, "max_idx")] = f.max_idx.mem.copy()
        ev.run()
        if noise:
            ev.err_output.mem[...] = rnd(ev.err_output.mem)
        for k in ("err_output", "n_err", "confusion_matrix", "max_err_output_sum"):
            a = getattr(ev, k)
            if isinstance(a, Array) and a:
                out[("eval", k)] = a.mem.copy()
        fwd_index = {id(f): i for i, f in enumerate(wf.forwards)}
        for g in reversed([g for g in wf.gds if g is not None]):
            i = fwd_index[id(g.forward_unit)]
            f = g.forward_unit
            w0 = {p: getattr(f, p).mem.copy() for p in ("weights", "bias")
                  if isinstance(getattr(f, p, None), Array) and getattr(f, p)}
            g.run()
            if noise and isinstance(g.err_input, Array) and g.err_input:
                g.err_input.mem[...] = rnd(g.err_input.mem)
            for p, w in w0.items():
                out[("upd", i, p)] = getattr(f, p).mem - w
        # read after the whole backward pass, as on the device: a GD unit with an activation
        # scales its err_output (the err_input of the unit above) by f'(y) in place
        for g in wf.gds:
            if g is None:
                continue
            i = fwd_index[id(g.forward_unit)]
            for k in ("err_input", "gradient_weights", "gradient_bias"):
                a = getattr(g, k, None)
                if isinstance(a, Array) and a:
                    out[("gd", i, k)] = a.mem.copy()
        return out, adopted


# ------------------------------------------------------------------------------------------------
# the system under test
# ------------------------------------------------------------------------------------------------
class StepOracleChecker(object):
    """Wraps the loader's run: before each minibatch the previous TRAIN step is checked."""

    def __init__(self, wf, oracle, bf16, on_gpu):
        self.wf, self.oracle, self.bf16, self.on_gpu = wf, oracle, bf16, on_gpu
        self.ld = wf.loader
        self.pre = None
        self.steps = []              # per checked step: {key: (ratio, e_max, e_l2, tol)}
        self.adoptions = {}
        self.kept = None             # (sut, ref, tol) of the last ragged step, for the self-check
        self.ragged = self.ragged_replays = 0
        self.runs = 0
        inner = self.ld.run

        def run():
            self.check()
            r = inner()
            self.runs += 1
            self.pre = self.record_pre() if self.ld.minibatch_class == TRAIN else None
            if self.pre is not None:
                self.pre["graphs"] = self.graph_state()
            return r
        self.ld.run = run

    def graph_state(self):
        segs = getattr(self.wf, "segments_", None) or []
        if not self.on_gpu or not segs:
            return None
        return sum(sg.replays for sg in segs), sum(len(sg._graphs) for sg in segs)

    # -- recording ------------------------------------------------------------------------------
    def record_pre(self):
        wf = self.wf
        gd_of = _gd_of(wf)
        rec = {"w": {}, "m": {}, "hyper": {}, "eval": {}}
        for i, f in enumerate(wf.forwards):
            g = gd_of.get(id(f))
            for part in ("weights", "bias"):
                w = getattr(f, part, None)
                if isinstance(w, Array) and w:
                    rec["w"][(i, part)] = _host(w)
                    m = _host(getattr(g, "gradient_%s_with_moment" % part, None))
                    if m is not None:
                        rec["m"][(i, part)] = m
        for k in ("n_err", "confusion_matrix", "max_err_output_sum"):
            v = _host(getattr(wf.evaluator, k, None))
            if v is not None:
                rec["eval"][k] = v
        return rec

    def record_post(self):
        wf, ld = self.wf, self.ld
        post = {"batch": int(ld.minibatch_size), "data": _host(ld.minibatch_data),
                "labels": _host(ld.minibatch_labels), "fwd": {}, "gd": {}, "eval": {},
                "last": bool(ld.last_minibatch)}
        for i, f in enumerate(wf.forwards):
            post["fwd"][i] = {k: _host(getattr(f, k, None))
                              for k in ("output", "max_idx", "input_offset", "weights", "bias")}
        gd_of = _gd_of(wf)
        hyper = {}
        for i, f in enumerate(wf.forwards):
            g = gd_of.get(id(f))
            if g is None:
                continue
            hyper[i] = {h: getattr(g, h) for h in HYPER if hasattr(g, h)}
            post["gd"][i] = {k: _host(getattr(g, k, None))
                             for k in ("err_input", "gradient_weights", "gradient_bias")}
        self.pre["hyper"] = hyper
        ev = wf.evaluator
        post["eval"]["err_output"] = _host(ev.err_output)
        if post["last"]:
            # the decision read the epoch's metrics and reset the evaluator's accumulators
            dec = wf.decision
            post["eval"]["n_err"] = numpy.array(
                [dec.epoch_n_err[TRAIN], dec.epoch_n_evaluated_samples[TRAIN]], numpy.int64)
            if dec.confusion_matrixes[TRAIN] is not None:
                post["eval"]["confusion_matrix"] = numpy.array(dec.confusion_matrixes[TRAIN])
            post["eval"]["max_err_output_sum"] = numpy.array([dec.max_err_y_sums[TRAIN]])
        else:
            for k in ("n_err", "confusion_matrix", "max_err_output_sum"):
                v = _host(getattr(ev, k, None))
                if v is not None:
                    post["eval"][k] = v
        if self.on_gpu:
            pad = ld.minibatch_data.__dict__.get("padded_dev_")
            if pad is not None:
                c = post["data"].shape[-1]
                assert float(pad[..., c:].abs().max()) == 0.0, "channel padding is not zero"
                post["pad_checked"] = True
        return post

    # -- decision alignment ------------------------------------------------------------------------
    def noise_bound(self, x):
        rel = 2.0 ** -7 if self.bf16 else FP32_TOL / 4
        return rel * max(float(numpy.abs(x).max()), 1e-30)

    def align(self, i, f, post):
        """Adopt the device's choice where the oracle's decision is within the noise bound."""
        name = type(f).__name__
        gpu = post["fwd"][i]
        key = (i, name)
        if name == "MaxPooling":
            x = f.input.mem.reshape(f.input_nhwc)
            win, off = f.windows(x, -numpy.inf)
            top2 = numpy.sort(win, axis=3)[:, :, :, -2:, :]
            b = self.noise_bound(x)
            amb = (top2[:, :, :, 1, :] - top2[:, :, :, 0, :]) <= b
            goff = gpu["input_offset"].reshape(f.input_offset.shape).astype(numpy.int64)
            mine = f.input_offset.mem
            amb &= goff != mine
            if amb.any():
                flat = x.ravel()
                chosen = flat[goff[amb]]
                assert (chosen >= top2[:, :, :, 1, :][amb] - b).all(), \
                    "%s: the device picked a value outside the noise band of the window max" % f
                inside = (off == goff[:, :, :, None, :]).any(axis=3)
                assert inside[amb].all(), "%s: the device's offset lies outside its window" % f
                f.input_offset.mem[amb] = goff[amb]
                f.output.mem[amb] = chosen
            return {key: int(amb.sum())}
        if name == "ForwardStrictRELU" or (name in ("Conv", "All2All") and f.ACT == 3):
            pre = f.input.mem if name == "ForwardStrictRELU" else None
            if pre is None:
                return {}
            g = self._gpu_value(i, post)
            if g is None:
                return {}
            b = self.noise_bound(pre)
            amb = (numpy.abs(pre) <= b) & ((g.reshape(pre.shape) > 0) != (f.output.mem > 0))
            bs = post["batch"]
            amb[bs:] = False
            if amb.any():
                f.output.mem[amb] = numpy.maximum(g.reshape(pre.shape)[amb], 0.0)
            return {key: int(amb.sum())}
        if name == "All2AllSoftmax":
            mi = gpu["max_idx"]
            y = f.output.mem
            bs = post["batch"]
            rows = numpy.arange(bs)
            mine = f.max_idx.mem[:bs]
            theirs = mi[:bs].astype(numpy.int64)
            b = self.noise_bound(y[:bs])
            amb = (theirs != mine)
            if amb.any():
                assert (y[rows[amb], theirs[amb]] >= y[rows[amb], mine[amb]] - b).all(), \
                    "%s: the device's arg-max is not within the noise band of the row max" % f
                f.max_idx.mem[:bs][amb] = theirs[amb]
            return {key: int(amb.sum())}
        return {}

    def _gpu_value(self, i, post):
        """The device tensor holding forward unit i's output (an activation folded into its
        producer lives in the producer's output)."""
        f = self.wf.forwards[i]
        p = getattr(f, "fused_into_", None)
        if p is not None:
            return post["fwd"][self.wf.forwards.index(p)]["output"]
        return post["fwd"][i]["output"]

    # -- comparison -----------------------------------------------------------------------------
    def pairs(self, post, ref):
        """(name, sut, ref) for every tensor the device materialises, in the oracle's meaning."""
        wf = self.wf
        fw = wf.forwards
        bs = post["batch"]
        gd_of = _gd_of(wf)
        out = []
        self.update_keys = {"%s.%s_update" % (f.name, p): (i, p)
                            for i, f in enumerate(fw) for p in ("weights", "bias")}
        for i, f in enumerate(fw):
            if getattr(f, "fused_into_", None) is not None:
                continue                         # aliased: no tensor of its own
            act = int(f.__dict__.get("fused_act_", 0) or 0)
            # a folded activation: the producer's tensor holds f(y), the activation unit's output
            j = i + 1 if act else i
            r = ref[("fwd", j, "output")]
            out.append(("%s.output" % f.name, post["fwd"][i]["output"][:bs], r[:bs]))
            if post["fwd"][i]["max_idx"] is not None and ("fwd", i, "max_idx") in ref:
                out.append(("%s.max_idx" % f.name, post["fwd"][i]["max_idx"][:bs],
                            ref[("fwd", i, "max_idx")][:bs]))
        for k in ("err_output", "n_err", "confusion_matrix", "max_err_output_sum"):
            if ("eval", k) in ref and k in post["eval"]:
                r = ref[("eval", k)]
                out.append(("evaluator.%s" % k, post["eval"][k].reshape(r.shape), r))
        for i, f in enumerate(fw):
            g = gd_of.get(id(f))
            if g is None or getattr(g, "fused_into_", None) is not None:
                continue
            for k in ("err_input", "gradient_weights", "gradient_bias"):
                a = post["gd"][i][k]
                if a is None or ("gd", i, k) not in ref:
                    continue
                r = ref[("gd", i, k)]
                if k == "err_input":
                    code = int(g.__dict__.get("in_deriv_act_", 0) or 0)
                    if code and getattr(fw[i - 1], "fused_into_", None) is not None:
                        # the consumer's kernel applied the derivative of the activation folded
                        # into the conv below: the error with respect to the conv's output
                        # before its activation (a conv with an activation of its own scales
                        # this tensor in place in the oracle as well)
                        y = ref[("fwd", i - 1, "output")]
                        r = r * deriv_from_output(code, y)
                    a, r = a[:bs], r[:bs]
                out.append(("%s.%s" % (g.name, k), a.reshape(r.shape), r))
            for p in ("weights", "bias"):
                if ("upd", i, p) in ref and (i, p) in self.pre["w"]:
                    w0 = self.pre["w"][(i, p)].astype(numpy.float64)
                    upd = post["fwd"][i][p] - w0
                    # the master weights are fp32: the update the device can store is the
                    # rounded sum minus the old weight, exact to one ulp of the weight
                    r = (w0 + ref[("upd", i, p)]).astype(numpy.float32) - w0
                    out.append(("%s.%s_update" % (f.name, p), upd, r))
        return out

    def check(self):
        if self.pre is None:
            return
        post = self.record_post()
        ref, adopted = self.oracle.step(self.pre, post, self, False)
        if self.bf16:
            noisy, _ = self.oracle.step(self.pre, post, self, True)
        for k, v in adopted.items():
            self.adoptions[k] = self.adoptions.get(k, 0) + v
        results, kept, slack_of = {}, {}, {}
        for name, a, r in self.pairs(post, ref):
            if a.dtype.kind in "iu" or name.endswith(("n_err", "confusion_matrix")) or \
                    name.endswith("max_idx"):
                assert numpy.array_equal(numpy.asarray(a, numpy.int64),
                                         numpy.asarray(r, numpy.int64)), \
                    "step %d: %s differs: %s vs %s" % (len(self.steps), name, a, r)
                continue
            tol = FP32_TOL
            if self.bf16:
                nn = dict((n, rr) for n, _, rr in self.pairs(post, noisy))[name]
            else:
                nn = None
            slack = None
            if name.endswith("_update"):
                w = numpy.abs(self.pre["w"][self.update_keys[name]]).astype(numpy.float32)
                slack = numpy.spacing(w).astype(numpy.float64)
            if self.bf16:
                # an update inherits the bf16 noise of the gradient it applies
                tol = max(BF16_FACTOR * max(errors(nn, r, slack)), BF16_FLOOR)
            e_max, e_l2 = errors(a, r, slack)
            assert within(a, r, tol, slack), "step %d (batch %d): %s: max-abs %.3g, L2 %.3g > tol %.3g" % (
                len(self.steps), post["batch"], name, e_max, e_l2, tol)
            results[name] = (max(e_max, e_l2) / tol, e_max, e_l2, tol)
            kept[name] = (numpy.asarray(a, numpy.float64), numpy.asarray(r, numpy.float64), tol)
            if slack is not None:
                slack_of[name] = slack
        # every tensor of the step is above
        if post["batch"] < self.ld.max_minibatch_size:
            self.ragged += 1
            g0, g1 = self.pre["graphs"], self.graph_state()
            if g0 is not None and g1[0] > g0[0] and g1[1] == g0[1]:
                self.ragged_replays += 1      # step graphs replayed, nothing was captured
            self.kept = kept
            self.kept_batch = post["batch"]
        self.steps.append(results)
        self.pre = None

    # -- the sensitivity self-check -------------------------------------------------------------
    def self_check(self):
        """One element of a real result moved by twice its tolerance must fail the comparison: a
        border pixel of a conv err_input, one gradient row, one padding row of err_output."""
        assert self.kept, "no ragged step was checked"
        probes = []
        for name, (a, r, tol) in sorted(self.kept.items()):
            if name.endswith("err_input") and a.ndim == 4:
                probes.append((name, (a.shape[0] - 1, 0, a.shape[2] - 1, a.shape[3] - 1)))
            elif name.endswith("gradient_weights"):
                probes.append((name, (a.shape[0] - 1,) + (0,) * (a.ndim - 1)))
            elif name == "evaluator.err_output":
                probes.append((name, (self.kept_batch,) + (a.shape[1] - 1,)))
        kinds = {n.rsplit(".", 1)[1] for n, _ in probes}
        assert {"gradient_weights", "err_output"} <= kinds, kinds
        for name, idx in probes:
            a, r, tol = self.kept[name]
            assert within(a, r, tol), name
            assert not within(perturbed(a, r, tol, idx), r, tol), \
                "%s: a change of 2x the tolerance at %s passes the comparison" % (name, idx)
        return [n for n, _ in probes]


def run_checked(model, compute, on_gpu):
    oracle = Oracle(model)
    root.common.engine.precision_type = "float"
    wf = build(model, compute, "cuda" if on_gpu else "numpy")
    chk = StepOracleChecker(wf, oracle, compute == "bf16", on_gpu)
    # a small training set can be learnt without an error within the run, and the decision stops
    # on a zero error; the steps are what is checked here, not the stop rule
    wf.decision.stop_condition = lambda: False
    ld = wf.loader
    per_epoch = -(-N_TRAIN[model] // ld.max_minibatch_size)
    for _ in range(4 * EPOCHS * per_epoch):
        if chk.runs >= EPOCHS * per_epoch:
            break
        wf.run(iterations=1)
    chk.check()
    assert len(chk.steps) == EPOCHS * per_epoch, (len(chk.steps), per_epoch)
    assert chk.ragged == EPOCHS
    assert wf.forwards[-1].output.shape[1] == N_CLASSES[model]
    return wf, chk


def _report(model, compute, chk, t):
    worst = max(((v[0], n) for s in chk.steps for n, v in s.items()), default=(0.0, None))
    sys.stderr.write("step oracle %s/%s: %d steps, %.1f s, worst error/tol %.3f (%s), "
                     "adoptions %s\n" % (model, compute, len(chk.steps), t, worst[0], worst[1],
                                         {k[1] + str(k[0]): v for k, v in chk.adoptions.items()}))


def _adoptions_small(wf, chk):
    # bf16 storage leaves 8 significant bits: pooling windows and ReLU inputs that the exact
    # oracle separates by less than that tie or swap on the device far more often than in fp32
    share = 50 if chk.bf16 else 200
    for (i, name), n in chk.adoptions.items():
        size = wf.forwards[i].output.size * len(chk.steps)
        assert n <= 8 + size // share, "%s: %d adopted decisions of %d" % (name, n, size)


# ------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------
def test_bf16_round_and_comparison_are_sharp():
    x = numpy.array([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -3.14159265, 1e-20])
    r = bf16_round(x)
    assert r[0] == 1.0 and r[1] == 1.0 and r[2] == 1.0 + 2 ** -6
    assert abs(r[3] + 3.140625) < 1e-12
    a = numpy.linspace(-1, 1, 1000)
    assert within(a, a, FP32_TOL)
    assert not within(perturbed(a, a, FP32_TOL, 0), a, FP32_TOL)
    assert not within(perturbed(a, a, FP32_TOL, 999), a, FP32_TOL)


@pytest.mark.parametrize("model", ["mnist_conv", "cifar_caffe", "lstm"])
def test_numpy_step_matches_float64_oracle(model):
    """CPU tier: the numpy float32 workflow as the system under test. Exercises the anchoring,
    the decision alignment, the per-tensor comparison and the self-check without a GPU."""
    t0 = time.time()
    try:
        wf, chk = run_checked(model, "fp32", False)
    finally:
        root.common.engine.precision_type = "float"
        root.common.engine.compute_type = "fp32"
    _report(model, "numpy-fp32", chk, time.time() - t0)
    _adoptions_small(wf, chk)
    assert chk.self_check()


@pytest.mark.gpu
@pytest.mark.parametrize("compute", ["fp32", "bf16"])
@pytest.mark.parametrize("model", ["mnist_conv", "cifar_caffe", "lstm"])
def test_benchmarked_step_matches_float64_oracle(model, compute):
    import torch
    from veles.znicz_b200.kernels import load_extension
    ext = load_extension(required=True)
    halo0, lstm0 = ext.conv_halo_launches(), ext.lstm_persist_launches()
    t0 = time.time()
    alone = {"n": 0}
    try:
        from veles.znicz_b200.kernels import api
        orig = api.evaluate_softmax

        def counting(unit):
            if not unit.__dict__.get("fused_done_", False):
                alone["n"] += 1
            return orig(unit)
        api.evaluate_softmax = counting
        wf, chk = run_checked(model, compute, True)
        torch.cuda.synchronize()
    finally:
        from veles.znicz_b200.kernels import api
        api.evaluate_softmax = orig
        root.common.engine.precision_type = "float"
        root.common.engine.compute_type = "fp32"
    _report(model, compute, chk, time.time() - t0)
    _adoptions_small(wf, chk)
    # the step that was checked is the benchmarked one
    seg = wf.segments_[0]
    assert seg.fused_replays > 0
    assert chk.ragged_replays > 0, "no ragged minibatch ran as a graph replay"
    # (python-side count: the launches issued eagerly or while capturing the step graph)
    assert wf.fused_step_ is not None and wf.fused_step_.launches > 0
    assert wf.forwards[-1].__dict__.get("fused_eval_") is wf.evaluator
    assert alone["n"] == 0, "a stand-alone evaluate_softmax launch ran"
    if model == "cifar_caffe":
        assert ext.conv_halo_launches() > halo0
    if model == "lstm" and compute == "bf16":
        # (the persistent cluster kernels run on the bf16 weight shadow; fp32 steps per time step
        # on split-bf16 GEMMs)
        assert ext.lstm_persist_launches() > lstm0
    assert chk.self_check()
