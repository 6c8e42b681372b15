"""numpy-oracle vs sm_90a path for every unit (oracle style (b) of SURVEY §4;
/root/reference/tests/unit/test_all2all.py:138-152, test_gd.py:158-175), in fp32 and bf16,
with the 2x-NaN out-of-bounds guard idea applied to device buffers."""
import numpy
import pytest

from veles.znicz_b200.core.config import root
from veles.znicz_b200.core.memory import Array
from veles.znicz_b200.core.workflow import DummyWorkflow
from veles.znicz_b200.core.backends import get_device
from veles.znicz_b200.ops import (all2all, gd, conv, gd_conv, pooling, gd_pooling, activation,
                                  normalization, dropout, cutter, multiplier, summator)

pytestmark = pytest.mark.gpu
RS = numpy.random.RandomState(5)


def _pair(fwd_cls, gd_cls, x, fkw, gkw, device, links=("weights", "bias"), extra=(), mask=None):
    wf = DummyWorkflow()
    f = fwd_cls(wf, **fkw)
    f.input = Array(x.copy())
    if device is not None and device.is_cuda:
        from veles.znicz_b200.ops.nn_units import torch_act_dtype
        f.input.dev_dtype = torch_act_dtype()
    f.initialize(device=device)
    f.run()
    kw = dict(learning_rate=0.1, learning_rate_bias=0.1, weights_decay=0.01,
              gradient_moment=0.9, gradient_moment_bias=0.9)
    kw.update(gkw)
    g = gd_cls(wf, **kw)
    rs = numpy.random.RandomState(9)
    err = rs.uniform(-1, 1, f.output.shape).astype(numpy.float32)
    if mask is not None:
        err[mask.reshape(err.shape)] = 0
    g.err_output = Array(err)
    g.err_output.dev_dtype = f.output.dev_dtype
    g.input, g.output = f.input, f.output
    for a in links:
        if getattr(f, a, None) is not None:
            setattr(g, a, getattr(f, a))
    for a in extra:
        setattr(g, a, getattr(f, a))
    g.forward_unit = f
    g.initialize(device=device)
    g.run()
    return f, g


def _compare(fwd_cls, gd_cls, x, fkw=None, gkw=None, links=("weights", "bias"), extra=(),
             compute="fp32", tol=None):
    fkw, gkw = fkw or {}, gkw or {}
    root.common.engine.compute_type = "fp32"
    from veles.znicz_b200.core import prng
    prng.get(1).seed(77)
    fn, gn = _pair(fwd_cls, gd_cls, x, fkw, gkw, None, links, extra)
    mask = None
    if compute == "fp32" and "StrictRELU" in fwd_cls.__name__:
        # a hard gate at |y| ~ 1e-6 may open on one side only (the split-bf16 tensor-core product
        # differs from numpy in the 6th digit): no error is injected at such outputs
        mask = numpy.abs(fn.output.mem) < 1e-4
        prng.get(1).seed(77)
        fn, gn = _pair(fwd_cls, gd_cls, x, fkw, gkw, None, links, extra, mask)
    root.common.engine.compute_type = compute
    prng.get(1).seed(77)
    dev = get_device("cuda")
    fc, gc = _pair(fwd_cls, gd_cls, x, fkw, gkw, dev, links, extra, mask)
    tol = tol or (2e-4 if compute == "fp32" else 6e-2)
    res = {}
    for name, a, b in (("output", fn.output, fc.output), ("err_input", gn.err_input, gc.err_input),
                       ("weights", getattr(fn, "weights", None), getattr(fc, "weights", None)),
                       ("bias", getattr(fn, "bias", None), getattr(fc, "bias", None))):
        if a is None or not a:
            continue
        b.map_read()
        if compute == "fp32":
            scale = max(1e-6, float(numpy.abs(a.mem).max()))
            res[name] = float(numpy.abs(a.mem - b.mem.reshape(a.mem.shape)).max()) / scale
        else:   # bf16: relative L2 (a relu gate may flip for |y| ~ 0 under rounding)
            d = (a.mem - b.mem.reshape(a.mem.shape)).astype(numpy.float64)
            res[name] = float(numpy.sqrt((d * d).sum()) /
                              max(1e-12, numpy.sqrt((a.mem.astype(numpy.float64) ** 2).sum())))
        assert numpy.isfinite(b.mem).all(), name
        # (bias gradients of tiny layers are sums over a few hundred gated pixels: a ReLU gate
        # that flips under bf16 rounding moves them more than the weights)
        lim = tol * (1.5 if (name == "bias" and compute != "fp32") else 1.0)
        assert res[name] < lim, (name, res, compute)
    root.common.engine.compute_type = "fp32"
    return res


@pytest.mark.parametrize("compute", ["fp32", "bf16"])
@pytest.mark.parametrize("fwd,bwd", [
    (all2all.All2All, gd.GradientDescent), (all2all.All2AllTanh, gd.GDTanh),
    (all2all.All2AllRELU, gd.GDRELU), (all2all.All2AllStrictRELU, gd.GDStrictRELU),
    (all2all.All2AllSigmoid, gd.GDSigmoid)])
def test_fc(fwd, bwd, compute):
    x = RS.uniform(-1, 1, (100, 64)).astype(numpy.float32)
    _compare(fwd, bwd, x, {"output_sample_shape": 48, "weights_stddev": 0.2},
             {"factor_ortho": 0.001}, compute=compute)


@pytest.mark.parametrize("compute", ["fp32", "bf16"])
def test_fc_odd_shapes_and_softmax(compute):
    x = RS.uniform(-1, 1, (37, 13)).astype(numpy.float32)     # K % 8 != 0 -> SIMT path
    _compare(all2all.All2AllTanh, gd.GDTanh, x, {"output_sample_shape": 7,
                                                 "weights_stddev": 0.3}, compute=compute)
    x = RS.uniform(-1, 1, (50, 1024)).astype(numpy.float32)
    _compare(all2all.All2AllSoftmax, gd.GDSoftmax, x, {"output_sample_shape": 10,
                                                       "weights_stddev": 0.05},
             compute=compute)


@pytest.mark.parametrize("compute", ["fp32", "bf16"])
@pytest.mark.parametrize("fwd,bwd", [
    (conv.Conv, gd_conv.GradientDescentConv), (conv.ConvTanh, gd_conv.GDTanhConv),
    (conv.ConvStrictRELU, gd_conv.GDStrictRELUConv)])
@pytest.mark.parametrize("geom", [
    ((6, 16, 16, 32), 32, 5, 5, (2, 2, 2, 2), (1, 1)),
    ((5, 32, 32, 3), 32, 5, 5, (2, 2, 2, 2), (1, 1)),
    ((3, 11, 9, 8), 24, 3, 2, (1, 0, 2, 1), (2, 1)),
    ((6, 12, 12, 64), 87, 5, 5, (0, 0, 0, 0), (1, 1)),      # n_kernels % 8 != 0 (MNIST conv)
    ((4, 14, 14, 3), 27, 3, 3, (1, 1, 1, 1), (1, 1)),
    ((2, 13, 13, 96), 64, 3, 3, (1, 1, 1, 1), (1, 1)),      # 96 -> 128 channel padding (tap mode)
    ((3, 9, 9, 24), 16, 5, 5, (2, 2, 2, 2), (1, 1))])       # 24 -> 32
def test_conv(fwd, bwd, geom, compute):
    shape, f, ky, kx, pad, sl = geom
    x = RS.uniform(-1, 1, shape).astype(numpy.float32)
    kw = {"n_kernels": f, "kx": kx, "ky": ky, "padding": pad, "sliding": sl,
          "weights_stddev": 0.1}
    gkw = dict(kw)
    gkw.pop("weights_stddev")
    gkw["factor_ortho"] = 0.001
    _compare(fwd, bwd, x, kw, gkw, compute=compute)


@pytest.mark.parametrize("compute", ["fp32", "bf16"])
@pytest.mark.parametrize("fwd,bwd,links", [
    (pooling.MaxPooling, gd_pooling.GDMaxPooling, ("input_offset",)),
    (pooling.MaxAbsPooling, gd_pooling.GDMaxAbsPooling, ("input_offset",)),
    (pooling.AvgPooling, gd_pooling.GDAvgPooling, ())])
@pytest.mark.parametrize("k,s", [((2, 2), (2, 2)), ((3, 3), (2, 2))])
def test_pooling(fwd, bwd, links, k, s, compute):
    x = RS.uniform(-1, 1, (4, 17, 16, 32)).astype(numpy.float32)
    if compute == "bf16":   # keep argmax ties identical on both paths
        import torch
        x = torch.from_numpy(x).bfloat16().float().numpy()
    kw = {"kx": k[0], "ky": k[1], "sliding": s}
    _compare(fwd, bwd, x, kw, kw, links=(), extra=links, compute=compute)


@pytest.mark.parametrize("compute", ["fp32", "bf16"])
def test_lrn(compute):
    x = RS.uniform(-1, 1, (4, 8, 8, 32)).astype(numpy.float32)
    kw = {"alpha": 0.00005, "beta": 0.75, "n": 3, "k": 1}
    _compare(normalization.LRNormalizerForward, normalization.LRNormalizerBackward, x, kw, kw,
             links=(), compute=compute)
    kw = {"alpha": 0.01, "beta": 0.75, "n": 5, "k": 2}
    _compare(normalization.LRNormalizerForward, normalization.LRNormalizerBackward, x, kw, kw,
             links=(), compute=compute)


@pytest.mark.parametrize("compute", ["fp32", "bf16"])
@pytest.mark.parametrize("name", ["Tanh", "Sigmoid", "RELU", "StrictRELU", "Log", "TanhLog",
                                  "SinCos", "Mul"])
def test_activation(name, compute):
    x = RS.uniform(-4, 4, (16, 40)).astype(numpy.float32)
    fkw = {"factor": 0.37} if name == "Mul" else {}
    _compare(getattr(activation, "Forward" + name), getattr(activation, "Backward" + name), x,
             fkw, fkw, links=(), compute=compute,
             tol=None if compute == "fp32" else 6e-2)


def test_cutter_and_dropout():
    x = RS.uniform(-1, 1, (3, 9, 8, 4)).astype(numpy.float32)
    kw = {"padding": (1, 2, 3, 1)}
    _compare(cutter.Cutter, cutter.GDCutter, x, kw, kw, links=())
    # dropout: identical hash-based mask on both paths
    dev = get_device("cuda")
    outs = []
    for d in (None, dev):
        wf = DummyWorkflow()
        f = dropout.DropoutForward(wf, dropout_ratio=0.4, seed=1234)
        f.input = Array(x.copy())
        f.minibatch_class = 2
        f.initialize(device=d)
        f.run()
        f.output.map_read()
        f.mask.map_read()
        outs.append((f.output.mem.copy(), f.mask.mem.copy()))
    assert numpy.array_equal(outs[0][1], outs[1][1])
    assert numpy.abs(outs[0][0] - outs[1][0]).max() < 1e-6
    frac = float((outs[1][1] == 0).mean())
    assert 0.3 < frac < 0.5


def test_stochastic_pooling_gpu_valid():
    x = RS.uniform(-1, 1, (2, 8, 8, 16)).astype(numpy.float32)
    dev = get_device("cuda")
    wf = DummyWorkflow()
    f = pooling.StochasticPooling(wf, kx=2, ky=2, sliding=(2, 2), seed=99)
    f.input = Array(x.copy())
    f.initialize(device=dev)
    f.run()
    f.output.map_read()
    f.input_offset.map_read()
    flat = x.reshape(-1)
    assert numpy.allclose(flat[f.input_offset.mem.ravel()], f.output.mem.ravel())
    # chosen elements are positive whenever the window has a positive element
    win_max = x.reshape(2, 4, 2, 4, 2, 16).max(axis=(2, 4))
    assert ((f.output.mem > 0) | (win_max <= 0)).all()


@pytest.mark.parametrize("compute", ["fp32", "bf16"])
@pytest.mark.parametrize("seq", [True, False])
def test_lstm_sequence(compute, seq):
    from veles.znicz_b200.ops import lstm_seq
    x = RS.uniform(-1, 1, (16, 6, 24)).astype(numpy.float32)        # [batch, T, features]
    _compare(lstm_seq.LSTMSequence, lstm_seq.GDLSTMSequence, x,
             {"output_sample_shape": 40, "weights_stddev": 0.2, "return_sequences": seq},
             {"gradient_moment": 0.0, "gradient_moment_bias": 0.0},
             extra=("gates", "cells", "hidden", "xh"), compute=compute,
             tol=None if compute == "fp32" else 8e-2)
    # odd sizes: (I + H) % 8 != 0 -> SIMT GEMMs even in bf16 mode
    x = RS.uniform(-1, 1, (5, 3, 7)).astype(numpy.float32)
    _compare(lstm_seq.LSTMSequence, lstm_seq.GDLSTMSequence, x,
             {"output_sample_shape": 6, "weights_stddev": 0.3, "return_sequences": seq},
             {"gradient_moment": 0.0, "gradient_moment_bias": 0.0},
             extra=("gates", "cells", "hidden", "xh"), compute=compute,
             tol=None if compute == "fp32" else 8e-2)


@pytest.mark.parametrize("seq", [True, False])
@pytest.mark.parametrize("shape,hidden", [((40, 7, 64), 64), ((150, 5, 128), 256)])
def test_lstm_persistent_kernels(seq, shape, hidden):
    """Whole-sequence cluster kernels (csrc/lstm_persist.cu: W resident in shared memory, gates GEMM
    on wgmma, cell math on the register accumulators, h exchanged through L2 under barrier.cluster) against the
    numpy oracle; batch 150 = two clusters with a ragged second tile; ZNICZ_LSTM_PERSIST=0 is the
    per-step path and must agree as well."""
    import os
    from veles.znicz_b200.ops import lstm_seq
    from veles.znicz_b200.kernels import load_extension
    ext = load_extension(required=True)
    x = RS.uniform(-1, 1, shape).astype(numpy.float32)
    kw = ({"output_sample_shape": hidden, "weights_stddev": 0.1, "return_sequences": seq},
          {"gradient_moment": 0.0, "gradient_moment_bias": 0.0})
    before = ext.lstm_persist_launches()
    res = _compare(lstm_seq.LSTMSequence, lstm_seq.GDLSTMSequence, x, *kw,
                   extra=("gates", "cells", "hidden", "xh"), compute="bf16", tol=8e-2)
    assert ext.lstm_persist_launches() - before == 2, "persistent kernels did not run"
    # rows per cluster: the default spreads 32-row clusters over the SMs; 64 / 128 rows per
    # cluster (fewer, fatter CTAs) must give the same numbers
    for rows in ("64", "128"):
        os.environ["ZNICZ_LSTM_ROWS"] = rows
        try:
            res_r = _compare(lstm_seq.LSTMSequence, lstm_seq.GDLSTMSequence, x, *kw,
                             extra=("gates", "cells", "hidden", "xh"), compute="bf16", tol=8e-2)
        finally:
            del os.environ["ZNICZ_LSTM_ROWS"]
        for k in res:
            assert abs(res_r[k] - res[k]) < 1e-3, (rows, k, res, res_r)
    before = ext.lstm_persist_launches() - 2
    os.environ["ZNICZ_LSTM_PERSIST"] = "0"
    try:
        res0 = _compare(lstm_seq.LSTMSequence, lstm_seq.GDLSTMSequence, x, *kw,
                        extra=("gates", "cells", "hidden", "xh"), compute="bf16", tol=8e-2)
        assert ext.lstm_persist_launches() - before == 2
    finally:
        del os.environ["ZNICZ_LSTM_PERSIST"]
    for k in res:
        assert res[k] < max(2.5 * res0[k], 2e-2), (k, res, res0)


def test_lstm_persistent_forward_then_per_step_backward():
    """err_input_alpha != 1 keeps the backward pass on the per-step kernels: the gates / cells the
    persistent forward kernel left in its private lane-major layout are unpacked into the unit's
    public arrays first (lstm_unpack_state)."""
    from veles.znicz_b200.ops import lstm_seq
    from veles.znicz_b200.kernels import load_extension
    ext = load_extension(required=True)
    x = RS.uniform(-1, 1, (40, 6, 64)).astype(numpy.float32)
    before = ext.lstm_persist_launches()
    _compare(lstm_seq.LSTMSequence, lstm_seq.GDLSTMSequence, x,
             {"output_sample_shape": 64, "weights_stddev": 0.1, "return_sequences": True},
             {"gradient_moment": 0.0, "gradient_moment_bias": 0.0, "err_input_alpha": 0.5},
             extra=("gates", "cells", "hidden", "xh"), compute="bf16", tol=8e-2)
    assert ext.lstm_persist_launches() - before == 1          # forward only


@pytest.mark.parametrize("geom", [
    ((4, 35, 35, 3), 16, 11, 11, (0, 0, 0, 0), (4, 4)),            # AlexNet conv1 in small
    ((3, 21, 25, 3), 24, 5, 5, (2, 2, 2, 2), (2, 2)),              # padding, 12 channels per pixel
    ((2, 30, 30, 4), 8, 9, 7, (1, 0, 2, 1), (3, 3))])              # ImagenetAE-like 9 x 9 / 3
def test_strided_first_layer_conv_runs_in_space_to_depth_form(geom):
    """Strided convolution over an image-like input = stride-1 convolution over the space-to-depth
    tensor (csrc/s2d.cu): forward, weight gradient (unpacked from the transformed tap order) and
    bias against the numpy oracle."""
    from veles.znicz_b200.kernels import api
    shape, f, ky, kx, pad, sl = geom
    x = RS.uniform(-1, 1, shape).astype(numpy.float32)
    kw = {"n_kernels": f, "kx": kx, "ky": ky, "padding": pad, "sliding": sl, "weights_stddev": 0.1}
    gkw = dict(kw)
    gkw.pop("weights_stddev")
    before = api.counters.get("s2d", 0)
    _compare(conv.ConvTanh, gd_conv.GDTanhConv, x, kw, gkw, compute="bf16")
    assert api.counters.get("s2d", 0) == before + 1
    root.common.engine.conv_s2d = False
    try:
        _compare(conv.ConvTanh, gd_conv.GDTanhConv, x, kw, gkw, compute="bf16")
        assert api.counters.get("s2d", 0) == before + 1
    finally:
        root.common.engine.conv_s2d = True
