"""RBM contrastive-divergence training on the device (ops/rbm_units.py, csrc/rbm.cu): the hash
sampler against its numpy twin and the binomial bounds, one CD-1 step of the mnist_rbm workflow
against a float64 recomputation from the device's own samples, the bf16 weight copies after the
update, the whole workflow with every RBM numpy path disabled, and determinism across runs and
snapshots."""
import pickle

import numpy
import pytest

from veles.znicz_b200.core import prng
from veles.znicz_b200.core.backends import get_device
from veles.znicz_b200.core.config import root
from veles.znicz_b200.core.memory import Array
from veles.znicz_b200.core.workflow import DummyLauncher, DummyWorkflow
from veles.znicz_b200.models import mnist_rbm
from veles.znicz_b200.ops import rbm_units

pytestmark = pytest.mark.gpu


def _sigmoid(x):
    return 1.0 / (1.0 + numpy.exp(-x))


def _read(a):
    a.map_read()
    return a.mem.astype(numpy.float64).copy()


@pytest.fixture
def rbm_data(tmp_path):
    """mnist_rbm reads its patches from a .mat file: 96 binary samples of 64 visibles (a multiple
    of 8, so the hidden layer and make_h run their bf16 products on the weight copies)."""
    import scipy.io
    rs = numpy.random.RandomState(5)
    patterns = (rs.rand(6, 64) > 0.5).astype(numpy.float32)
    data = patterns[rs.randint(0, 6, 96)]
    flip = rs.rand(*data.shape) < 0.05
    data[flip] = 1 - data[flip]
    path = str(tmp_path / "rbm_patches.mat")
    scipy.io.savemat(path, {"patches": data})
    cfg = root.mnist_rbm.loader
    saved = cfg.data_path
    cfg.data_path = path
    yield data
    cfg.data_path = saved


def _build(compute, v_size=64, h_size=64, minibatch_size=40, n_samples=96, max_epochs=1, lr=0.05):
    root.common.engine.compute_type = compute
    prng.get(1).seed(1234)
    prng.get(2).seed(5678)
    wf = mnist_rbm.build(minibatch_size=minibatch_size, n_samples=n_samples, v_size=v_size,
                         h_size=h_size, max_epochs=max_epochs, learning_rate=lr)
    wf.initialize(device="cuda")
    return wf


# -- 1. the sampler and its numpy twin ----------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
def test_sampler_matches_numpy_twin(dtype):
    import torch
    rows, n, bs = 24, 300, 17
    rs = numpy.random.RandomState(3)
    wf = DummyWorkflow()
    b = rbm_units.Binarization(wf, seed=987654321)
    b.input = Array(rs.rand(rows, n).astype(numpy.float32),
                    dev_dtype=torch.bfloat16 if dtype == "bf16" else None)
    b.batch_size = bs
    b.initialize(device=get_device("cuda"))
    assert b.on_cuda and b.output.devmem.dtype == b.input.devmem.dtype
    p = b.input.devmem.float().cpu().numpy()
    outs = []
    for counter in (0, 1):
        assert b.rng_counter == counter
        b.run()
        out = _read(b.output)
        twin = rbm_units.binarize_twin(p, bs, b.seed, counter)
        assert numpy.array_equal(out[:bs], twin[:bs]), (dtype, counter)
        assert numpy.array_equal(out[bs:], p[bs:]), (dtype, counter)
        outs.append(out)
    assert not numpy.array_equal(outs[0][:bs], outs[1][:bs])


# -- 2. sampler statistics -------------------------------------------------------------------------
def test_sampler_statistics():
    grid = numpy.array([0.0, 1e-3, 0.01, 0.1, 0.25, 0.5, 0.75, 0.9, 0.99, 0.999, 1.0], numpy.float32)
    per_p = 2048
    wf = DummyWorkflow()
    b = rbm_units.Binarization(wf, seed=24680)
    b.input = Array(numpy.repeat(grid[:, None], per_p, axis=1))
    b.batch_size = len(grid)
    b.initialize(device=get_device("cuda"))
    fires = numpy.zeros(len(grid))
    counters = 64
    for _ in range(counters):
        b.run()
        fires += _read(b.output).sum(axis=1)
    trials = counters * per_p
    assert fires[0] == 0 and fires[-1] == trials
    for p, k in zip(grid.astype(numpy.float64), fires):
        sigma = numpy.sqrt(trials * p * (1 - p))
        assert abs(k - trials * p) <= 5 * sigma + 1e-9, (p, k / trials)


# -- 3. one CD-1 step against float64 ----------------------------------------------------------------
# h = sigma(v . W^T + hbias) from the device's v: bf16 activations and weight copies vs split-bf16
# fp32 products. The update is recomputed from the device's own bf16 / fp32 samples, so only the
# fp32 accumulation order and the rounding of W + dW separate it from the device's.
H_TOL = {"bf16": 1.5e-2, "fp32": 1e-4}
UPDATE_RTOL, UPDATE_ATOL = 1e-4, 2e-7


@pytest.mark.parametrize("ct", ["bf16", "fp32"])
def test_cd1_step_matches_float64(rbm_data, ct):
    lr = 0.05
    wf = _build(ct, lr=lr)
    b1, a2a = wf.forwards
    grad, bw0, bw1, gc, upd = wf.gds
    assert all(u.on_cuda for u in (b1, a2a, bw0, bw1, gc, upd, grad.bino_h, grad.bino_v))
    sizes = []
    for _ in range(3):                     # 40, 40 and the ragged 16 of 96 samples
        w0, hb0, vb0 = _read(a2a.weights), _read(a2a.bias), _read(wf.evaluator.vbias)
        wf.run(iterations=1)
        bs = int(wf.loader.minibatch_size)
        sizes.append(bs)
        v0, h0, v1, h1 = (_read(a) for a in (b1.output, a2a.output, grad.v1, grad.h1))
        assert v0.shape[0] == 40
        for v, h in ((v0, h0), (v1, h1)):
            assert set(numpy.unique(v[:bs])) <= {0.0, 1.0}
            err = numpy.abs(h[:bs] - _sigmoid(v[:bs] @ w0.T + hb0)).max()
            assert err < H_TOL[ct], (ct, bs, err)
        w1, hb1, vb1 = _read(a2a.weights), _read(a2a.bias), _read(wf.evaluator.vbias)
        v0, h0, v1, h1 = v0[:bs], h0[:bs], v1[:bs], h1[:bs]
        dw = lr * (v0.T @ h0 - v1.T @ h1).T / bs
        dhb = lr * (h0.mean(axis=0) - h1.mean(axis=0))
        dvb = lr * (v0.mean(axis=0) - v1.mean(axis=0))
        for what, got, want in (("W", w1 - w0, dw), ("hbias", hb1 - hb0, dhb),
                                ("vbias", vb1 - vb0, dvb)):
            bad = numpy.abs(got - want) > UPDATE_ATOL + UPDATE_RTOL * numpy.abs(want)
            assert not bad.any(), (ct, bs, what, float(numpy.abs(got - want).max()))
        assert numpy.abs(dw).max() > 1e-3
    assert sizes == [40, 40, 16]


# -- 4. the forwards read the updated weights ----------------------------------------------------------
def test_forwards_see_updated_weights(rbm_data):
    wf = _build("bf16", lr=0.5, max_epochs=3)
    a2a = wf.forwards[1]
    assert a2a.weights_lp_ is not None and wf.gds[0].make_h.weights_lp_ is not None
    w_init = _read(a2a.weights)
    for _ in range(6):
        w, hb = _read(a2a.weights), _read(a2a.bias)
        wf.run(iterations=1)
    bs = int(wf.loader.minibatch_size)
    v0, h0 = _read(wf.forwards[0].output)[:bs], _read(a2a.output)[:bs]
    assert numpy.abs(h0 - _sigmoid(v0 @ w.T + hb)).max() < H_TOL["bf16"]
    # the weights moved far enough that a forward on a stale copy would be caught
    assert numpy.abs(h0 - _sigmoid(v0 @ w_init.T + hb)).max() > 10 * H_TOL["bf16"]


# -- 5. the whole workflow, no RBM numpy path ---------------------------------------------------------
@pytest.mark.parametrize("ct", ["bf16", "fp32"])
def test_mnist_rbm_trains_on_device(monkeypatch, ct):
    def host_path(self):
        raise AssertionError("%s ran its numpy path" % self)

    for cls in (rbm_units.Binarization, rbm_units.BatchWeights, rbm_units.GradientsCalculator,
                rbm_units.WeightsUpdater):
        monkeypatch.setattr(cls, "numpy_run", host_path)
    wf = _build(ct, v_size=196, h_size=1000, n_samples=240, max_epochs=10)
    data = wf.loader.original_data.mem.astype(numpy.float64)
    a2a = wf.forwards[1]

    def recon_err():
        w, hb, vb = _read(a2a.weights), _read(a2a.bias), _read(wf.evaluator.vbias)
        h = _sigmoid(data @ w.T + hb)
        return float(((_sigmoid(h @ w + vb) - data) ** 2).mean())

    e0 = recon_err()
    downloaded = set()
    real = Array._download

    def download(self):
        downloaded.add(id(self))
        return real(self)

    monkeypatch.setattr(Array, "_download", download)
    wf.run()
    assert bool(wf.decision.complete)
    grad = wf.gds[0]
    stay = [a2a.weights, a2a.bias, wf.evaluator.vbias, wf.forwards[0].output, a2a.output,
            grad.v1, grad.h1, wf.evaluator.binarization.output, wf.evaluator.output]
    stay += [getattr(u, n) for u in wf.gds[1:3] for n in ("weights_batch", "hbias_batch",
                                                          "vbias_batch")]
    stay += [getattr(wf.gds[3], n) for n in ("weights_grad", "hbias_grad", "vbias_grad")]
    assert not [a for a in stay if id(a) in downloaded], "host round trip in the training loop"
    monkeypatch.setattr(Array, "_download", real)
    assert numpy.isfinite(_read(a2a.weights)).all()
    assert recon_err() < 0.7 * e0


# -- 6. determinism ---------------------------------------------------------------------------------
def test_runs_and_snapshots_are_deterministic(rbm_data):
    finals = []
    for _ in range(2):
        wf = _build("bf16", max_epochs=4)
        wf.run()
        finals.append(_read(wf.forwards[1].weights))
    assert numpy.array_equal(finals[0], finals[1])
    wf = _build("bf16", max_epochs=2)
    wf.run()
    wf = pickle.loads(pickle.dumps(wf))
    wf.workflow = DummyLauncher()
    wf.decision.max_epochs = 4
    wf.decision.complete <<= False
    wf.initialize(device="cuda", snapshot=True)
    wf.run()
    assert bool(wf.decision.complete)
    assert numpy.array_equal(_read(wf.forwards[1].weights), finals[0])
