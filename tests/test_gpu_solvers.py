"""adagrad / adadelta / fast / RProp inside the fused update kernels (csrc/update.cu::step_elem),
checked step by step against the numpy oracle functions (ops.gd.solver_step,
ops.rprop_gd.rprop_step). Each step the reduced gradient the kernel used is read back from the
unit's ``gradient_weights`` / ``gradient_bias``, so the check isolates the update from the bf16
GEMM noise of the gradient itself."""
import glob
import json
import os
import subprocess
import sys

import numpy
import pytest

from veles.znicz_b200.core.config import root
from veles.znicz_b200.core.memory import Array
from veles.znicz_b200.core.workflow import DummyWorkflow, DummyLauncher
from veles.znicz_b200.core.backends import get_device
from veles.znicz_b200.ops import all2all, gd, rprop_gd
from veles.znicz_b200.ops.nn_units import GradientDescentBase
from veles.znicz_b200.models import cifar

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-5
SOLVER_SETS = [("adagrad",), ("adadelta",), ("fast",), ("adagrad", "fast")]


def _close(a, b, what):
    scale = max(float(numpy.abs(b).max()), 1e-30)
    err = float(numpy.abs(a - b).max())
    assert err <= TOL * scale, "%s: max |diff| %.3g > %.1g * %.3g" % (what, err, TOL, scale)


def _parts(u):
    for part in ("weights", "bias"):
        w = getattr(u, part, None)
        if w is not None and w:
            yield part


def _record(units):
    rec = {}
    for u in units:
        for part in _parts(u):
            grad = getattr(u, "gradient_" + part)
            vel = getattr(u, "gradient_%s_with_moment" % part)
            arrays = {"w": getattr(u, part), "grad": grad, "vel": vel}
            for (name, p), a in getattr(u, "solver_state", {}).items():
                if p == part:
                    arrays["s:" + name] = a
            r = {}
            for k, a in arrays.items():
                if isinstance(a, Array) and a:
                    a.map_read()
                    r[k] = a.mem.copy()
            r["hyper"] = u.hyper_values()
            rec[(id(u), part)] = r
    return rec


def _oracle(u, part, pre, post):
    """Apply the shared oracle to the pre-step state with the gradient the kernel used."""
    is_bias = part == "bias"
    h = pre["hyper"]
    lr, wd, l1, moment = (h[9], h[10], h[11], h[12]) if is_bias else (h[0], h[1], h[2], h[3])
    ortho = 0 if is_bias else h[8]
    trans = False if is_bias else bool(u.weights_transposed)
    g = post["grad"]
    step = -GradientDescentBase.numpy_gradient_step(pre["w"], g, lr, wd, l1, ortho, trans)
    vel = step + pre["vel"] * numpy.float32(moment) if "vel" in pre else None
    w = pre["w"].copy()
    state = {k[2:]: v.copy() for k, v in pre.items() if k.startswith("s:")}
    gd.solver_step(w, (vel if vel is not None else step).copy(), vel, state, u.extra_solvers,
                   u.adagrad_epsilon, u.adadelta_momentum, u.adadelta_epsilon,
                   u.fast_learning_rate, u.apply_gradient, trans)
    _close(w, post["w"], "%s %s" % (u.name, part))
    if vel is not None:
        _close(vel, post["vel"], "%s %s velocity" % (u.name, part))
    for k, v in state.items():
        _close(v, post["s:" + k], "%s %s %s" % (u.name, part, k))


class StepChecker(object):
    """Wraps the loader's run: before each minibatch the previous TRAIN step is checked."""

    def __init__(self, wf):
        self.wf = wf
        self.units = [u for u in wf.gds if u is not None]
        self.ld = wf.loader
        self.prev, self.prev_train = None, False
        self.checked = 0
        inner = self.ld.run

        def run():
            self.check()
            r = inner()
            self.prev_train = self.ld.minibatch_class == 2
            self.prev = _record(self.units) if self.prev_train else None
            return r
        self.ld.run = run

    def check(self):
        if self.prev is None:
            return
        post = _record(self.units)
        for u in self.units:
            for part in _parts(u):
                _oracle(u, part, self.prev[(id(u), part)], post[(id(u), part)])
        self.checked += 1
        self.prev = None


def _cifar(solvers, graphs, fused, max_epochs=1, prefix="cifar_solv"):
    layers = cifar.caffe_layers()
    for l in layers:
        if "<-" in l:
            l["<-"].update(learning_rate=0.02, learning_rate_bias=0.02, weights_decay=0.0005,
                           solvers={"momentum"} | set(solvers))
        if l["type"] == "conv":
            l["->"]["weights_stddev"] = 0.05
    root.common.engine.fused_step = fused
    return cifar.build(
        layers=layers, use_graphs=graphs,
        loader_config={"minibatch_size": 20, "n_train": 200, "n_valid": 40,
                       "normalization_type": "internal_mean", "noise": 0.3},
        decision_config={"max_epochs": max_epochs, "fail_iterations": 10},
        snapshotter_config={"prefix": prefix, "interval": 1, "time_interval": 0,
                            "compression": ""})


# every solver on the default engine (fused step, CUDA graphs); adagrad+fast on every combination;
# fp32 and bf16 (tensor-core layers whose bf16 weight shadows the update kernel rewrites)
CIFAR_CASES = [(s, True, True, "fp32") for s in SOLVER_SETS] + \
    [(("adagrad", "fast"), f, g, "fp32") for f, g in ((True, False), (False, False), (False, True))] + \
    [(s, True, True, "bf16") for s in (("adadelta", "fast"), ("adagrad",))]


def _check_shadows(wf):
    """The bf16 shadows of the convolutions (no channel padding) equal the updated fp32 weights."""
    import torch
    from veles.znicz_b200.kernels import api
    n = 0
    for f in wf.forwards:
        lp = getattr(f, "weights_lp_", None)
        if lp is None or not hasattr(f, "kx") or api.lp_cpad(f):
            continue
        f.weights.map_read()
        w = torch.from_numpy(f.weights.mem).to(lp.device).to(torch.bfloat16)
        assert torch.equal(lp[:w.shape[0], :w.shape[1]], w), f.name
        n += 1
    return n


@pytest.mark.parametrize("solvers,fused,graphs,compute", CIFAR_CASES,
                         ids=["%s-fused%d-graphs%d-%s" % ("+".join(s), f, g, c)
                              for s, f, g, c in CIFAR_CASES])
def test_cifar_solvers_match_oracle(solvers, fused, graphs, compute):
    """CIFAR caffe net (first conv with its channel-padded gradient, conv, FC softmax; ortho on)."""
    from veles.znicz_b200.core import prng
    prng.get(1).seed(1234)
    prng.get(2).seed(5678)
    root.common.disable.snapshotting = True       # (the step checker's hook does not pickle)
    root.common.engine.compute_type = compute
    try:
        wf = _cifar(solvers, graphs, fused)
        wf.initialize(device="cuda")
        gds = [u for u in wf.gds if u is not None and getattr(u, "weights", None)]
        assert gds and all(u.on_cuda for u in gds)
        assert all(u.extra_solvers == set(solvers) for u in gds)
        assert (wf.fused_step_ is not None) == fused
        chk = StepChecker(wf)
        wf.run()
        chk.check()
        assert chk.checked >= 9
        if graphs:
            assert wf.segments_[0].fused_replays > 0        # the fused train-step graph replays
        for u in gds:
            u.weights.map_read()
            assert numpy.isfinite(u.weights.mem).all()
        if compute == "bf16":
            assert _check_shadows(wf) >= 2
    finally:
        root.common.engine.fused_step = True
        root.common.disable.snapshotting = False
        root.common.engine.compute_type = "fp32"


def test_lstm_seq_solvers_match_oracle():
    from veles.znicz_b200.models import lstm_seq
    root.common.disable.snapshotting = True
    try:
        wf = lstm_seq.build(seq_len=6, features=8, hidden=16, n_classes=3,
                            loader_config={"minibatch_size": 16, "n_train": 96, "n_valid": 32,
                                           "noise": 0.2},
                            decision_config={"max_epochs": 1, "fail_iterations": 10})
        for u in wf.gds:
            u.gradient_moment = u.gradient_moment_bias = 0.5
            u.solvers = {"momentum", "adagrad", "fast"}
        wf.initialize(device="cuda")
        assert type(wf.gds[0]).__name__ == "GDLSTMSequence"
        assert all(u.on_cuda for u in wf.gds) and wf.fused_step_ is not None
        chk = StepChecker(wf)
        wf.run()
        chk.check()
        assert chk.checked >= 5
    finally:
        root.common.disable.snapshotting = False


def _fc_pair(gd_cls, device, transposed=False, **gkw):
    wf = DummyWorkflow()
    rs = numpy.random.RandomState(11)
    f = all2all.All2All(wf, output_sample_shape=48, weights_stddev=0.1,
                        weights_transposed=transposed)
    f.input = Array(rs.uniform(-1, 1, (32, 40)).astype(numpy.float32))
    f.initialize(device=device)
    f.run()
    kw = dict(learning_rate=0.05, learning_rate_bias=0.05, weights_decay=0.001,
              gradient_moment=0.9, gradient_moment_bias=0.9, weights_transposed=transposed)
    kw.update(gkw)
    g = gd_cls(wf, **kw)
    g.err_output = Array(rs.uniform(-1, 1, (32, 48)).astype(numpy.float32))
    g.input, g.output, g.weights, g.bias = f.input, f.output, f.weights, f.bias
    g.forward_unit = f
    g.initialize(device=device)
    return f, g, rs


@pytest.mark.parametrize("solvers", SOLVER_SETS, ids="+".join)
@pytest.mark.parametrize("transposed", [False, True])
def test_fc_immediate_update_matches_oracle(solvers, transposed):
    """Stand-alone FC GD unit: the per-tensor kernel (no whole-network step)."""
    root.common.engine.compute_type = "fp32"
    f, g, rs = _fc_pair(gd.GradientDescent, get_device("cuda"), transposed,
                        solvers={"momentum"} | set(solvers))
    assert g.on_cuda and g.step_ is None
    for _ in range(5):
        pre = _record([g])
        g.err_output.map_write()
        g.err_output.mem[...] = rs.uniform(-1, 1, g.err_output.shape)
        g.run()
        post = _record([g])
        for part in _parts(g):
            _oracle(g, part, pre[(id(g), part)], post[(id(g), part)])


@pytest.mark.parametrize("apply", [True, False])
def test_rprop_on_device_matches_oracle(apply):
    root.common.engine.compute_type = "fp32"
    f, g, rs = _fc_pair(rprop_gd.GDRProp, get_device("cuda"), apply_gradient=apply,
                        increase=1.2, decrease=0.5, max_learning_rate=0.05)
    assert g.on_cuda
    for step in range(6):
        recs = {}
        for name, a in (("w", g.weights), ("b", g.bias), ("gw", g.gradient_weights),
                        ("gb", g.gradient_bias), ("lw", g.weight_lrs), ("lb", g.bias_lrs)):
            a.map_read()
            recs[name] = a.mem.copy()
        g.err_output.map_write()
        sign = -1.0 if step % 3 == 2 else 1.0          # flip now and then: rates shrink
        g.err_output.mem[...] = sign * numpy.abs(rs.uniform(-1, 1, g.err_output.shape))
        g.run()
        for w, gr, lr, wa, ga, la in (("w", "gw", "lw", g.weights, g.gradient_weights,
                                       g.weight_lrs),
                                      ("b", "gb", "lb", g.bias, g.gradient_bias, g.bias_lrs)):
            for a in (wa, ga, la):
                a.map_read()
            wt, prev, lrs = recs[w].copy(), recs[gr].copy(), recs[lr].copy()
            rprop_gd.rprop_step(wt, prev, lrs, ga.mem.copy(), g.increase, g.decrease,
                                g.min_learning_rate, g.max_learning_rate, apply)
            _close(lrs, la.mem, "rprop rates " + w)
            _close(wt, wa.mem, "rprop " + w)
    if not apply:
        assert numpy.array_equal(g.weights.mem, recs["w"])


def test_solver_snapshot_resume_continues():
    """k steps, snapshot, restore into a fresh workflow, k more == 2k uninterrupted steps."""
    from veles.znicz_b200.core import prng
    from veles.znicz_b200.core.snapshotter import SnapshotterToFile
    results = []
    for resume in (False, True):
        prng.get(1).seed(4321)
        prng.get(2).seed(8765)
        prefix = "cifar_solv_resume%d" % int(resume)
        for p in glob.glob(os.path.join(root.common.dirs.snapshots, prefix + "_*")):
            os.remove(p)
        wf = _cifar(("adadelta", "fast"), True, True, max_epochs=1 if resume else 2,
                    prefix=prefix)
        wf.initialize(device="cuda")
        wf.run()
        if resume:
            snaps = sorted(glob.glob(os.path.join(root.common.dirs.snapshots, prefix + "_*")),
                           key=os.path.getmtime)
            assert snaps
            wf = SnapshotterToFile.import_file(snaps[-1])
            wf.workflow = DummyLauncher()
            wf.decision.max_epochs = 2
            wf.decision.complete <<= False
            wf.initialize(device="cuda", snapshot=True)
            assert all(isinstance(a, Array) for u in wf.gds if u is not None
                       for a in getattr(u, "solver_state", {}).values())
            wf.run()
        out = []
        for u in wf.gds:
            if u is None or not getattr(u, "weights", None):
                continue
            u.weights.map_read()
            out.append(u.weights.mem.copy())
            for k in sorted(getattr(u, "solver_state", {})):
                u.solver_state[k].map_read()
                out.append(u.solver_state[k].mem.copy())
        results.append(out)
    diffs = [float(numpy.abs(a - b).max()) for a, b in zip(*results)]
    assert all(numpy.array_equal(a, b) for a, b in zip(*results)), diffs


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("algo", [0, 1])
def test_fake_peer_solvers_update_desc_bit_exact(n, algo):
    """N fake ranks on one GPU (one-shot and two-shot reduction) == the single-GPU kernel fed the
    summed gradient, bit for bit, with every solver bit set; likewise for the per-tensor kernel."""
    r = subprocess.run([sys.executable, os.path.join(REPO, "tests", "fake_peer_solver_worker.py"),
                        str(n), str(algo)], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, PYTHONPATH=REPO))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["finite"] and res["state_moved"], res
    assert res["ranks_identical"], res
    assert res["equal_w"] and res["equal_v"] and res["equal_gout"] and res["equal_state"], res
    assert res["per_tensor_equal"], res
