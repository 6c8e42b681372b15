"""fp8 fully connected layers (compute_type "fp8"): the block-128 numerics oracle
(utils/mxfp8.py), its CPU training emulation, and - on the GPU - the quantisers, the fp8 mode
of the persistent GEMM, the layers, weight re-quantisation and end-to-end training."""
import numpy
import pytest

from veles.znicz_b200.core.config import root
from veles.znicz_b200.utils import mxfp8

RS = numpy.random.RandomState(11)


# ------------------------------------------------------------------------------------ CPU
def test_block_exponent_rule():
    a = numpy.array([0.0, 1e-40, 1.0, 1.75, 1.7500001, 224.0, 448.0, 448.00003, 449.0, 3e38],
                    numpy.float32)
    e = mxfp8.block_exponent(a)
    assert e.tolist() == [-127, -127, -8, -8, -7, -1, 0, 1, 1, 120]
    # the definition: the smallest e with amax <= 448 * 2^e
    x = numpy.abs(RS.randn(1000).astype(numpy.float32)) * numpy.float32(2.0) ** RS.randint(-60, 60, 1000)
    e = mxfp8.block_exponent(x).astype(numpy.float64)
    assert (x <= 448.0 * 2.0 ** e).all() and (x > 448.0 * 2.0 ** (e - 1)).all()


def test_row_block_quantiser_properties():
    x = (RS.randn(37, 300) * numpy.array([1e-3, 1.0, 50.0])[RS.randint(0, 3, 37)][:, None])
    x = x.astype(numpy.float32)
    x[5] = 0.0
    q, s = mxfp8.quantize_rows(x)
    assert q.shape == x.shape and s.shape == (3, 128) and s.dtype == numpy.float32
    assert numpy.array_equal(mxfp8._e4m3(q), q)               # codes are e4m3 values
    assert numpy.abs(q).max() <= 448.0
    # powers of two; the block maximum lands in (224, 448] (224 itself after rounding); zero and
    # padding rows get 2^-127
    m, ex = numpy.frexp(s)
    assert (m == 0.5).all()
    assert (s[:, 5] == numpy.float32(2.0) ** -127).all() and (s[:, 37:] == s[0, 5]).all()
    qp = numpy.pad(numpy.abs(q), ((0, 0), (0, 84))).reshape(37, 3, 128).max(axis=2)
    live = numpy.abs(x).sum(axis=1) > 0
    assert ((qp >= 224.0) & (qp <= 448.0))[live].all()     # (224 after rounding)
    back = mxfp8.fake_quant_rows(x, 1)
    blk = numpy.pad(numpy.abs(x), ((0, 0), (0, 84))).reshape(37, 3, 128).max(axis=2)
    err = numpy.pad(numpy.abs(back - x), ((0, 0), (0, 84))).reshape(37, 3, 128).max(axis=2)
    assert (err <= blk * 2.0 ** -4 + 1e-30).all()
    # along the other axis = along the rows of the transpose
    assert numpy.array_equal(mxfp8.fake_quant_rows(x, 0), mxfp8.fake_quant_rows(x.T, 1).T)


def test_tile_quantiser_transposes_share_scales():
    w = (RS.randn(300, 200) * 0.05).astype(numpy.float32)
    w[128:256, 128:] *= 1e3                                     # one tile with its own range
    q, qt, s, st = mxfp8.quantize_tiles(w)
    assert numpy.array_equal(q.T, qt)
    assert s.shape == (2, 384) and st.shape == (3, 256)
    tiles = s[:, ::128]                                         # [kb_in][kb_out]
    assert numpy.array_equal(tiles.T, st[:, ::128])
    assert (s.reshape(2, 3, 128) == tiles[:, :, None]).all()   # expanded per row
    # the same tile quantisation serves W and W^T
    assert numpy.array_equal(mxfp8.fake_quant_tiles(w).T, mxfp8.fake_quant_tiles(w.T))
    top = numpy.pad(numpy.abs(q), ((0, 84), (0, 56))).reshape(3, 128, 2, 128).max(axis=(1, 3))
    assert ((top >= 224.0) & (top <= 448.0)).all()


def _train_mnist(device, compute="fp32", emulate=False, hidden=None):
    from veles.znicz_b200.core import prng
    from veles.znicz_b200.models import mnist
    root.common.engine.fp8_emulation = emulate
    root.common.engine.compute_type = compute
    prng.get(1).seed(1234)
    prng.get(2).seed(5678)
    try:
        layers = mnist.fc_layers()
        if hidden:
            layers[0]["->"]["output_sample_shape"] = hidden
        wf = mnist.build(
            layers=layers, loader_name="synthetic_mnist",
            loader_config={"minibatch_size": 20, "n_train": 400, "n_valid": 200, "noise": 0.6,
                           "normalization_type": "linear"},
            decision_config={"max_epochs": 6, "fail_iterations": 10})
        wf.initialize(device=device)
        wf.run()
        ws = []
        for f in wf.forwards:
            f.weights.map_read()
            ws.append(f.weights.mem.copy())
        return wf.decision.best_n_err_pt[1], ws
    finally:
        root.common.engine.fp8_emulation = False
        root.common.engine.compute_type = "fp32"


def test_block128_emulated_training_converges_like_full_precision():
    err_ref, w_ref = _train_mnist("numpy")
    err_q, w_q = _train_mnist("numpy", emulate=mxfp8.BLOCK128)
    assert err_ref < 15.0, err_ref
    assert err_q < 15.0 and abs(err_q - err_ref) <= 5.0, (err_q, err_ref)
    d = max(float(numpy.abs(a - b).max()) for a, b in zip(w_ref, w_q))
    assert 0 < d < 0.25 * max(float(numpy.abs(a).max()) for a in w_ref)


# ------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def ext():
    from veles.znicz_b200.kernels import load_extension
    return load_extension(required=True)


def _codes(t):
    """Device uint8 codes -> numpy uint8."""
    return t.cpu().numpy()


def _oracle_bytes(q):
    import torch
    return torch.from_numpy(numpy.ascontiguousarray(q)).to(torch.float8_e4m3fn).view(
        torch.uint8).numpy()


def _r16(n):
    return (n + 15) // 16 * 16


def _quant_act_dev(ext, x, rows, cols):
    import torch
    dev = x.device
    kr, kc = -(-rows // 128), -(-cols // 128)
    q = torch.full((rows, _r16(cols)), 0xAA, dtype=torch.uint8, device=dev)
    s = torch.full((kc, kr * 128), float("nan"), device=dev)
    qt = torch.full((cols, _r16(rows)), 0xAA, dtype=torch.uint8, device=dev)
    st = torch.full((kr, kc * 128), float("nan"), device=dev)
    assert ext.fp8_quant(x, rows, cols, 0, q, s, qt, st) == 0
    return q, s, qt, st


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols", [(128, 9216), (100, 4096), (37, 200), (300, 13), (1, 1)])
def test_quant_act_bit_equal_to_oracle(ext, rows, cols):
    import torch
    x = torch.from_numpy((RS.randn(rows, cols) * 3).astype(numpy.float32))
    x[:, :min(cols, 5)] *= 1e-30                     # tiny and subnormal values
    if rows > 3:
        x[3] = 0.0
    xb = x.to(torch.bfloat16)
    q, s, qt, st = _quant_act_dev(ext, xb.cuda(), rows, cols)
    torch.cuda.synchronize()
    xf = xb.float().numpy()
    oq, os_ = mxfp8.quantize_rows(xf)
    oqt, ost = mxfp8.quantize_rows(xf.T)
    assert numpy.array_equal(_codes(q)[:, :cols], _oracle_bytes(oq))
    assert numpy.array_equal(s.cpu().numpy(), os_)
    assert numpy.array_equal(_codes(qt)[:, :rows], _oracle_bytes(oqt))
    assert numpy.array_equal(st.cpu().numpy(), ost)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols", [(4096, 9216), (1000, 4096), (200, 784), (130, 48)])
def test_quant_weight_bit_equal_to_oracle(ext, rows, cols):
    import torch
    w = (RS.randn(rows, cols) * 0.02).astype(numpy.float32)
    w[:128, :128] = 0.0
    kr, kc = -(-rows // 128), -(-cols // 128)
    dev = torch.device("cuda")
    q = torch.empty((rows, _r16(cols)), dtype=torch.uint8, device=dev)
    qt = torch.empty((cols, _r16(rows)), dtype=torch.uint8, device=dev)
    s = torch.empty((kc, kr * 128), device=dev)
    st = torch.empty((kr, kc * 128), device=dev)
    assert ext.fp8_quant(torch.from_numpy(w).cuda(), rows, cols, 1, q, s, qt, st) == 0
    oq, oqt, os_, ost = mxfp8.quantize_tiles(w)
    assert numpy.array_equal(_codes(q)[:, :cols], _oracle_bytes(oq))
    assert numpy.array_equal(_codes(qt)[:, :rows], _oracle_bytes(oqt))
    assert numpy.array_equal(s.cpu().numpy(), os_)
    assert numpy.array_equal(st.cpu().numpy(), ost)


def _dequant(q, s, rows, cols):
    import torch
    v = q[:, :cols].contiguous().view(torch.float8_e4m3fn).double()
    sc = s.double().t()[:rows].repeat_interleave(128, dim=1)[:, :cols]
    return v * sc


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["forward", "dgrad", "wgrad"])
@pytest.mark.parametrize("M,N,K", [(128, 4096, 9216), (100, 1000, 4096), (37, 200, 784),
                                   (4096, 9216, 128), (4096, 9216, 100)])
def test_fp8_gemm_forms(ext, form, M, N, K):
    """out = A . B^T of block-scaled operands in the three forms a layer uses: forward (bf16 out,
    bias; B a tile-quantised weight), dgrad (bf16 out, alpha; B the weight's transpose
    copy), wgrad (fp32 out; both operands quantised along the batch)."""
    import torch
    dev = torch.device("cuda")
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(dev)
    b = (torch.randn(N, K, generator=g) * 0.05).to(dev)
    bias = torch.randn(N, generator=g).to(dev) if form == "forward" else None
    alpha = 0.7 if form == "dgrad" else 1.0
    out_dt = torch.float32 if form == "wgrad" else torch.bfloat16
    aq, asc, _, _ = _quant_act_dev(ext, a.to(torch.bfloat16).contiguous(), M, K)
    kr, kc = -(-N // 128), -(-K // 128)
    if form == "wgrad":
        bq, bsc, _, _ = _quant_act_dev(ext, b.to(torch.bfloat16).contiguous(), N, K)
    else:
        # a weight W [K][N] stored for the dgrad form as W^T: the tile quantiser writes both
        bq = torch.empty((N, _r16(K)), dtype=torch.uint8, device=dev)
        bsc = torch.empty((kc, kr * 128), device=dev)
        bqt = torch.empty((K, _r16(N)), dtype=torch.uint8, device=dev)
        bst = torch.empty((-(-K // 128), -(-N // 128) * 128), device=dev)
        assert ext.fp8_quant(b.contiguous(), N, K, 1, bq, bsc, bqt, bst) == 0
    big = torch.full((2 * M, N), float("nan"), device=dev, dtype=out_dt)
    out = big[:M]
    assert ext.fp8_gemm(aq, asc, bq, bsc, out, M, N, K, bias, 0, alpha) == 0
    torch.cuda.synchronize()
    assert torch.isnan(big[M:]).all(), "write past the output rows"
    deq = _dequant(aq, asc, M, K) @ _dequant(bq, bsc, N, K).t() * alpha
    full = a.double() @ b.double().t() * alpha
    if bias is not None:
        deq = deq + bias.double()
        full = full + bias.double()
    got = out.double()
    e_deq = float((got - deq).norm() / deq.norm())
    e_full = float((got - full).norm() / full.norm())
    print("fp8 gemm %s M=%d N=%d K=%d: rel err vs dequantised %.2e, vs unquantised %.2e" % (
        form, M, N, K, e_deq, e_full))
    # bf16 outputs round to 8 bits: the dequantised bound applies to the fp32 form, the bf16
    # forms are allowed the output rounding on top
    tol = 1e-3 if out_dt == torch.float32 else 4e-3
    assert e_deq < tol and e_full < 5e-2


@pytest.mark.gpu
def test_fp8_gemm_refuses_bad_alignment(ext):
    import torch
    dev = torch.device("cuda")
    a = torch.zeros((64, 24), dtype=torch.uint8, device=dev)      # row pitch 24 % 16 != 0
    b = torch.zeros((64, 32), dtype=torch.uint8, device=dev)
    s = torch.ones((1, 128), device=dev)
    out = torch.full((64, 64), float("nan"), device=dev)
    before = ext.fp8_gemm_launches()
    assert ext.fp8_gemm(a, s, b, s, out, 64, 64, 24, None, 0, 1.0) != 0
    assert ext.fp8_gemm_launches() == before
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


def _fp8_compare(fwd_cls, gd_cls, x, n_out, tol=None):
    """Layer + GD unit on the GPU in fp8 vs the numpy path under block128 emulation."""
    from test_gpu_units import _compare
    root.common.engine.fp8_emulation = mxfp8.BLOCK128
    try:
        return _compare(fwd_cls, gd_cls, x, {"output_sample_shape": n_out, "weights_stddev": 0.05},
                        {}, compute="fp8", tol=tol)
    finally:
        root.common.engine.fp8_emulation = False


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["", "Tanh", "RELU", "StrictRELU", "Sigmoid", "Softmax"])
def test_fp8_layers_match_block128_emulation(ext, name):
    from veles.znicz_b200.ops import all2all, gd
    from veles.znicz_b200.kernels import api
    fwd_cls = getattr(all2all, "All2All" + name)
    gd_cls = getattr(gd, ("GD" + name) if name else "GradientDescent")
    x = RS.uniform(-1, 1, (100, 256)).astype(numpy.float32)
    before = ext.fp8_gemm_launches()
    api.paths.clear()
    # the device quantises the bf16 input, numpy the fp32 one: a few codes differ by one step,
    # and a strict ReLU gate at |y| ~ 0 then opens on one side only (err_input moves most)
    _fp8_compare(fwd_cls, gd_cls, x, 200, tol=0.12 if name == "StrictRELU" else None)
    # forward, dgrad and wgrad: three fp8 GEMMs. The softmax layer's GD unit gets fp32 errors from
    # this harness (the probabilities are fp32), so its backward takes the fp32 path as in bf16 mode
    assert ext.fp8_gemm_launches() - before == (1 if name == "Softmax" else 3)
    assert not any("fp8:declined" in t for ts in api.paths.values() for t in ts), api.paths


@pytest.mark.gpu
def test_fp8_declined_shape_uses_bf16(ext):
    from veles.znicz_b200.ops import all2all, gd
    from veles.znicz_b200.kernels import api
    from test_gpu_units import _compare
    api.paths.clear()
    before = ext.fp8_gemm_launches()
    x = RS.uniform(-1, 1, (37, 13)).astype(numpy.float32)
    _compare(all2all.All2AllTanh, gd.GDTanh, x, {"output_sample_shape": 40, "weights_stddev": 0.3},
             compute="fp8")
    assert ext.fp8_gemm_launches() == before
    assert any("fp8:declined(n_in % 16)" in t for ts in api.paths.values() for t in ts), api.paths


def _check_weights_q(fwd):
    fwd.weights.map_read()
    oq, oqt, os_, ost = mxfp8.quantize_tiles(fwd.weights.mem)
    n_out, n_in = fwd.weights.shape
    assert numpy.array_equal(_codes(fwd.weights_q_)[:, :n_in], _oracle_bytes(oq))
    assert numpy.array_equal(_codes(fwd.weights_qt_)[:, :n_out], _oracle_bytes(oqt))
    assert numpy.array_equal(fwd.weights_qs_.cpu().numpy(), os_)
    assert numpy.array_equal(fwd.weights_qts_.cpu().numpy(), ost)


def _fc_net_layers():
    return [{"type": "all2all_tanh", "->": {"output_sample_shape": 128, "weights_stddev": 0.05},
             "<-": {"learning_rate": 0.05, "gradient_moment": 0.9}},
            {"type": "all2all_tanh", "->": {"output_sample_shape": 64, "weights_stddev": 0.05},
             "<-": {"learning_rate": 0.05, "gradient_moment": 0.9}},
            {"type": "softmax", "->": {"output_sample_shape": 10, "weights_stddev": 0.05},
             "<-": {"learning_rate": 0.05, "gradient_moment": 0.9}}]


@pytest.mark.gpu
def test_fp8_weights_requantised_after_graph_steps_and_rollback(ext):
    from veles.znicz_b200.models import mnist
    root.common.engine.compute_type = "fp8"
    try:
        wf = mnist.build(
            layers=_fc_net_layers(), loader_name="synthetic_mnist", use_graphs=True,
            loader_config={"minibatch_size": 20, "n_train": 200, "n_valid": 40, "noise": 0.6,
                           "normalization_type": "linear"},
            decision_config={"max_epochs": 2, "fail_iterations": 10})
        wf.initialize(device="cuda")
        fwds = [f for f in wf.forwards if getattr(f, "weights_q_", None) is not None]
        assert len(fwds) == 2
        for f in fwds:
            f.weights.map_read()
        w0 = [f.weights.mem.copy() for f in fwds]
        wf.run()
        import torch
        torch.cuda.synchronize()
        assert any(s.replays > 0 for s in wf.segments_)
        for f, w in zip(fwds, w0):
            _check_weights_q(f)
            assert not numpy.array_equal(f.weights.mem, w)
        # an NNRollback restore (workflow/nn_rollback.py) writes the fp32 master and refreshes
        # the shadows
        for f, w in zip(fwds, w0):
            f.weights.map_invalidate()
            f.weights.mem[...] = w
            f.weights.unmap()
            f.refresh_shadows()
        torch.cuda.synchronize()
        for f in fwds:
            _check_weights_q(f)
    finally:
        root.common.engine.compute_type = "fp32"


@pytest.mark.gpu
def test_mnist_fc_fp8_trains_like_bf16():
    """MNIST FC net with a 128-wide hidden layer (the fc_layers() width 100 gives 200-byte bf16
    output rows, which the fp8 GEMM's TMA-store epilogue declines); the 10-way softmax layer is a
    few-output layer and stays on its fused bf16 kernel."""
    from veles.znicz_b200.kernels import api
    api.paths.clear()
    err_bf, _ = _train_mnist("cuda", "bf16", hidden=128)
    err_f8, _ = _train_mnist("cuda", "fp8", hidden=128)
    assert not any("fp8:declined" in t for t in api.paths.get("fc_tanh1_forward", ())), api.paths
    print("MNIST FC on the GPU: best validation error bf16 %.2f %%, fp8 %.2f %%" % (err_bf, err_f8))
    assert abs(err_f8 - err_bf) <= 5.0, (err_f8, err_bf)


@pytest.mark.gpu
def test_alexnet_fp8_steps(ext):
    from veles.znicz_b200.models import alexnet
    from veles.znicz_b200.kernels import api
    root.common.engine.compute_type = "fp8"
    api.paths.clear()
    before = ext.fp8_gemm_launches()
    try:
        wf = alexnet.build(
            loader_name="synthetic_imagenet", layers=alexnet.alexnet_layers(n_classes=20),
            loader_config={"minibatch_size": 8, "shape": (227, 227, 3), "n_classes": 20,
                           "n_train": 24, "n_valid": 8, "noise": 0.3,
                           "normalization_type": "internal_mean"},
            decision_config={"max_epochs": 1, "fail_iterations": 5},
            snapshotter_config={"prefix": "inet_f8", "interval": 1000, "time_interval": 1e9})
        wf.initialize(device="cuda")
        fc = [f for f in wf.forwards if getattr(f, "weights_q_", None) is not None]
        wf.run()
        assert bool(wf.decision.complete)
        for f in wf.forwards:
            if getattr(f, "weights", None):
                f.weights.map_read()
                assert numpy.isfinite(f.weights.mem).all(), f.name
        wf.forwards[-1].output.map_read()
        out = wf.forwards[-1].output.mem
        assert numpy.isfinite(out).all() and abs(float(out[0].sum()) - 1.0) < 1e-2
        # FC6, FC7 and FC8 (the softmax layer, 20 outputs) run in fp8
        assert len(fc) == 3, [f.name for f in wf.forwards]
        assert ext.fp8_gemm_launches() > before
    finally:
        root.common.engine.compute_type = "fp32"
