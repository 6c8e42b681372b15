"""Host side of the solvers that run inside the fused update kernels: the flag bits, the device
hyper-vector layout, the solver state as Arrays (snapshots) and the shared numpy oracle."""
import pickle

import numpy
import pytest

from veles.znicz_b200.core.memory import Array
from veles.znicz_b200.core.workflow import DummyWorkflow
from veles.znicz_b200.ops import all2all, gd, rprop_gd
from veles.znicz_b200.ops.nn_units import GradientDescentBase


def _gd_pair(cls=gd.GradientDescent, solvers=(), **gkw):
    wf = DummyWorkflow()
    f = all2all.All2All(wf, output_sample_shape=3, weights_stddev=0.1)
    rs = numpy.random.RandomState(3)
    f.input = Array(rs.uniform(-1, 1, (4, 5)).astype(numpy.float32))
    f.initialize(device=None)
    f.run()
    kw = dict(learning_rate=0.1, learning_rate_bias=0.1, weights_decay=0.0, gradient_moment=0.5,
              gradient_moment_bias=0.5)
    if solvers:
        kw["solvers"] = set(solvers)
    kw.update(gkw)
    g = cls(wf, **kw)
    g.err_output = Array(rs.uniform(-1, 1, (4, 3)).astype(numpy.float32))
    g.input, g.output, g.weights, g.bias = f.input, f.output, f.weights, f.bias
    g.forward_unit = f
    g.initialize(device=None)
    return f, g


@pytest.mark.parametrize("solvers,bits", [
    ((), 0), (("momentum",), 0), (("momentum", "adagrad"), 32), (("momentum", "adadelta"), 64),
    (("momentum", "fast"), 128), (("momentum", "adagrad", "fast"), 32 | 128),
    (("momentum", "adadelta", "fast"), 64 | 128)])
def test_update_flags_solver_bits(solvers, bits):
    _, g = _gd_pair(solvers=solvers)
    for for_bias in (False, True):
        f = g.update_flags(for_bias=for_bias)
        assert f & 0x1e0 == bits
        assert f & 3 == 3                          # apply + momentum stay as they were


def test_rprop_flags_replace_the_sgd_step():
    _, g = _gd_pair(rprop_gd.GDRProp)
    assert g.update_flags() == 256 | 1
    g.apply_gradient = False
    assert g.update_flags(for_bias=True) == 256
    assert not g.force_numpy
    s0, s1, s2 = g.solver_arrays()
    assert s0 is g.weight_lrs and s1 is None and s2 is None
    assert g.solver_arrays(for_bias=True)[0] is g.bias_lrs


def test_hyper_vector_layout():
    fields = GradientDescentBase.HYPER_FIELDS
    assert len(fields) == 24
    assert fields[:13] == ("lr", "wd", "l1_vs_l2", "moment", "acc_alpha", "acc_beta",
                           "gd_alpha", "gd_beta", "factor_ortho", "lr_bias", "wd_bias",
                           "l1_vs_l2_bias", "moment_bias")
    assert fields[13:21] == ("adagrad_epsilon", "adadelta_rho", "adadelta_epsilon", "fast_lr",
                             "rprop_increase", "rprop_decrease", "rprop_min_lr", "rprop_max_lr")
    _, g = _gd_pair(solvers=("momentum", "adagrad", "fast"), adagrad_epsilon=1e-6,
                    adadelta_momentum=0.8, adadelta_epsilon=1e-7, fast_learning_rate=0.03)
    v = g.hyper_values()
    assert len(v) == 24
    assert v[:4] == (0.1, 0.0, 0, 0.5) and v[12] == 0.5
    assert v[13:17] == (1e-6, 0.8, 1e-7, 0.03) and v[17:] == (0.0,) * 7
    _, r = _gd_pair(rprop_gd.GDRProp, increase=1.2, decrease=0.5, min_learning_rate=1e-5,
                    max_learning_rate=0.5)
    v = r.hyper_values()
    assert v[13:17] == (0.0,) * 4 and v[17:21] == (1.2, 0.5, 1e-5, 0.5) and v[21:] == (0.0,) * 3


def test_solver_state_is_arrays_and_pickles():
    f, g = _gd_pair(solvers=("momentum", "adadelta", "fast"))
    assert set(g.solver_state) == {(n, p) for n in ("adadelta", "adadelta_g", "fast")
                                   for p in ("weights", "bias")}
    assert all(isinstance(a, Array) for a in g.solver_state.values())
    g.run()
    g.run()
    state = pickle.loads(pickle.dumps(g.solver_state))
    for k, a in g.solver_state.items():
        assert numpy.array_equal(state[k].mem, a.mem)
    s0, s1, s2 = g.solver_arrays()
    assert s0 is g.solver_state[("adadelta", "weights")]
    assert s1 is g.solver_state[("adadelta_g", "weights")]
    assert s2 is g.solver_state[("fast", "weights")]


def test_parent_format_solver_state_loads_and_continues():
    """Earlier snapshots hold ``solver_state`` as a dict of numpy arrays: re-initialising adopts
    the values, and the next step equals the one of a unit that never left memory."""
    f, g = _gd_pair(solvers=("momentum", "adagrad"))
    g.run()
    g.run()
    ref_f, ref_g = f, g
    snap = {k: a.mem.copy() for k, a in g.solver_state.items()}     # the earlier format
    f2, g2 = _gd_pair(solvers=("momentum", "adagrad"))
    f2.weights.mem[...] = f.weights.mem
    f2.bias.mem[...] = f.bias.mem
    g2.gradient_weights_with_moment.mem[...] = g.gradient_weights_with_moment.mem
    g2.gradient_bias_with_moment.mem[...] = g.gradient_bias_with_moment.mem
    g2.solver_state = pickle.loads(pickle.dumps(snap))
    g2.initialize(device=None)
    assert all(isinstance(a, Array) for a in g2.solver_state.values())
    for k, a in g2.solver_state.items():
        assert numpy.array_equal(a.mem, snap[k])
    ref_g.run()
    g2.run()
    assert numpy.array_equal(f2.weights.mem, ref_f.weights.mem)
    for k, a in g2.solver_state.items():
        assert numpy.array_equal(a.mem, ref_g.solver_state[k].mem)


def test_solver_step_is_the_unit_oracle():
    """numpy_update delegates to the pure solver_step: the same inputs give the same result."""
    f, g = _gd_pair(solvers=("momentum", "adagrad", "fast"))
    w0 = f.weights.mem.copy()
    v0 = g.gradient_weights_with_moment.mem.copy()
    st0 = {n: g.solver_state[(n, "weights")].mem.copy() for n in ("adagrad", "fast")}
    g.run()
    grad = g.gradient_weights.mem
    step = -GradientDescentBase.numpy_gradient_step(w0, grad, 0.1, 0.0, 0, 0, False)
    vel = step + v0 * 0.5
    w = w0.copy()
    gd.solver_step(w, vel.copy(), vel, st0, {"adagrad", "fast"}, g.adagrad_epsilon,
                   g.adadelta_momentum, g.adadelta_epsilon, g.fast_learning_rate)
    assert numpy.array_equal(w, f.weights.mem)
    assert numpy.array_equal(st0["adagrad"], g.solver_state[("adagrad", "weights")].mem)
    assert numpy.array_equal(st0["fast"], g.solver_state[("fast", "weights")].mem)


def test_rprop_rates_survive_reinitialisation():
    f, g = _gd_pair(rprop_gd.GDRProp)
    g.run()
    g.run()
    lrs = g.weight_lrs.mem.copy()
    g.initialize(device=None)
    assert numpy.array_equal(g.weight_lrs.mem, lrs)


def test_non_default_variants_keep_the_host_maths():
    """The update kernels implement variant_gradient / variant_moment_gradient = True only."""
    _, g = _gd_pair(solvers=("momentum", "adagrad"), variant_gradient=False)
    assert g.force_numpy
    _, g = _gd_pair(solvers=("momentum", "fast"), variant_moment_gradient=False)
    assert g.force_numpy
    _, g = _gd_pair(solvers=("momentum", "adagrad"))
    assert not g.force_numpy


@pytest.mark.parametrize("cls,solvers", [(gd.GradientDescent, ("momentum", "adadelta")),
                                         (rprop_gd.GDRProp, ())])
def test_earlier_snapshot_force_numpy_is_cleared(cls, solvers):
    """Units restored from an earlier version's snapshot carry the force_numpy that version set
    for every solver unit; a unit of this version keeps a force_numpy the user asked for."""
    _, g = _gd_pair(cls, solvers=solvers)
    state = g.__getstate__()
    state.pop("solvers_on_device")
    state["_force_numpy"] = True
    old = cls.__new__(cls)
    old.__setstate__(pickle.loads(pickle.dumps(state)))
    old.init_unpickled()
    old.initialize(device=None)
    assert not old.force_numpy and old.solvers_on_device
    _, g = _gd_pair(cls, solvers=solvers, force_numpy=True)
    assert g.force_numpy
