"""Cross-framework golden data: Caffe blob dumps shipped with the reference Znicz test suite
(``tests/functional/data/*.txt`` and ``tests/data/gd_conv_data/gd_conv3.*`` there) vs our numpy
units - the reference's ``tests/functional/test_caffe.py`` strategy (SURVEY §4, "cross-framework
golden data"). The blobs are stored under ``tests/golden/caffe/<dump>.npz`` as float32 NHWC
arrays, all images (tools/make_caffe_golden.py regenerates them)."""
import os

import numpy
import pytest

from veles.znicz_b200.core.config import root
from veles.znicz_b200.core.memory import Array
from veles.znicz_b200.core.workflow import DummyWorkflow
from veles.znicz_b200.ops import conv, gd_conv, gd_pooling, normalization, pooling

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "caffe")


def _golden(dump):
    """{blob name: float64 array} of one Caffe dump."""
    with numpy.load(os.path.join(GOLDEN, dump + ".npz")) as z:
        return {k: z[k].astype(numpy.float64) for k in z.files}


def _rel(a, b):
    return float(numpy.abs(a - b).sum() / max(numpy.abs(b).sum(), 1e-30))


@pytest.fixture(autouse=True)
def _double():
    root.common.engine.precision_type = "double"
    yield
    root.common.engine.precision_type = "float"


def _conv_unit(wf, bottom, weights, n_kernels):
    u = conv.Conv(wf, kx=5, ky=5, padding=(2, 2, 2, 2), sliding=(1, 1), n_kernels=n_kernels)
    u.input = Array(bottom.copy())
    u.initialize(device="numpy")
    u.weights.mem[:] = weights.reshape(n_kernels, -1)
    u.bias.mem[:] = 0
    u.run()
    return u


def test_conv_forward_matches_caffe():
    d = _golden("conv")
    bottom, weights, top = d["bottom"], d["weights"], d["top"]
    u = _conv_unit(DummyWorkflow(), bottom, weights, 2)
    assert _rel(u.output.mem, top) < 1e-2      # dumps carry 6 decimals of ~1e-4 weights


def test_conv_backward_matches_caffe():
    d = _golden("conv_grad")
    bottom, weights, top = d["bottom"], d["weights"], d["top"]
    top_err, bot_err = d["top_diff"], d["bottom_diff"]
    wf = DummyWorkflow()
    u = _conv_unit(wf, bottom, weights, 2)
    assert _rel(u.output.mem, top) < 1e-2      # dumps carry 6 decimals of ~1e-4 weights
    g = gd_conv.GradientDescentConv(wf, kx=5, ky=5, padding=(2, 2, 2, 2), sliding=(1, 1),
                                    n_kernels=2, learning_rate=0.0, weights_decay=0.0,
                                    apply_gradient=False, gradient_moment=0.0)
    g.err_output = Array(top_err.copy())
    g.link_attrs(u, "input", "output", "weights", "bias")
    g.initialize(device="numpy")
    g.run()
    assert _rel(g.err_input.mem, bot_err) < 1e-2


@pytest.mark.parametrize("fname", ["pool.txt", "pool_grad.txt"])
def test_max_pooling_matches_caffe(fname):
    d = _golden(fname[:-4])
    bottom, top = d["bottom"], d["top"]
    wf = DummyWorkflow()
    u = pooling.MaxPooling(wf, kx=3, ky=3, sliding=(2, 2))
    u.input = Array(bottom.copy())
    u.initialize(device="numpy")
    u.run()
    assert _rel(u.output.mem, top) < 1e-6
    if fname == "pool_grad.txt":
        top_err, bot_err = d["top_diff"], d["bottom_diff"]
        g = gd_pooling.GDMaxPooling(wf, kx=3, ky=3, sliding=(2, 2))
        g.err_output = Array(top_err.copy())
        g.link_attrs(u, "input", "input_offset", "output")
        g.initialize(device="numpy")
        g.run()
        # errors of ~1e-6 printed with 6 decimals + tie-breaking between equal maxima
        assert _rel(g.err_input.mem, bot_err) < 0.03


def test_lrn_matches_caffe():
    d = _golden("norm_gd")
    bottom, top, top_err, bot_err = d["bottom"], d["top"], d["top_diff"], d["bottom_diff"]
    wf = DummyWorkflow()
    f = normalization.LRNormalizerForward(wf, k=1)
    f.input = Array(bottom.copy())
    f.initialize(device="numpy")
    f.run()
    assert _rel(f.output.mem, top) < 0.02          # the reference allows 2 %
    b = normalization.LRNormalizerBackward(wf, k=1)
    b.input, b.output = f.input, f.output
    b.err_output = Array(top_err.copy())
    b.initialize(device="numpy")
    b.run()
    assert _rel(b.err_input.mem, bot_err) < 0.02


def test_conv3_golden_arrays_forward_and_err_input():
    """The reference ships golden arrays of the CIFAR net's conv3 (5 x 5, pad 2, 32 -> 64 channels,
    3 images) under tests/data/gd_conv_data (SURVEY Appendix C): forward output and err_input of
    the numpy oracle against them (relative max error; the arrays come from a Caffe fp32 run)."""
    d = _golden("gd_conv3")
    x, w, b, y, eo, ei = [d[n] for n in ("input", "weights", "bias", "output", "err_output", "err_input")]
    wf = DummyWorkflow()
    kw = dict(n_kernels=64, kx=5, ky=5, padding=(2, 2, 2, 2), sliding=(1, 1))
    c = conv.Conv(wf, weights_stddev=0.1, **kw)
    c.input = Array(x.copy())
    c.initialize(device=None)
    c.weights.map_write()
    c.bias.map_write()
    c.weights.mem[...] = w
    c.bias.mem[...] = b
    c.run()
    assert c.output.mem.shape == y.shape
    assert numpy.abs(c.output.mem - y).max() / numpy.abs(y).max() < 1e-2
    g = gd_conv.GradientDescentConv(wf, learning_rate=0, learning_rate_bias=0, **kw)
    g.err_output = Array(eo.copy())
    g.input, g.output, g.weights, g.bias = c.input, c.output, c.weights, c.bias
    g.initialize(device=None)
    g.run()
    assert numpy.abs(g.err_input.mem - ei).max() / numpy.abs(ei).max() < 1e-3


def _conv_relu(wf, bottom, weights):
    u = conv.ConvStrictRELU(wf, kx=5, ky=5, padding=(2, 2, 2, 2), sliding=(1, 1), n_kernels=2)
    u.input = Array(bottom.copy())
    u.initialize(device="numpy")
    u.weights.mem[:] = weights.reshape(2, -1)
    u.bias.mem[:] = 0
    u.run()
    return u


def test_conv_relu_forward_matches_caffe():
    """The reference's tests/functional/test_caffe.py (conv + ReLU pair, `conv_relu.txt`)."""
    d = _golden("conv_relu")
    bottom, weights, relu_top = d["conv_bottom"], d["conv_weights"], d["relu_top_flat"]
    u = _conv_relu(DummyWorkflow(), bottom, weights)
    assert _rel(u.output.mem, relu_top) < 5e-3        # weights printed with 6 decimals


def test_conv_relu_backward_matches_caffe():
    """`conv_relu_grad.txt`: the fused conv + ReLU GD unit against Caffe's ReLU backward followed
    by its conv backward - err_input and the raw weight gradient."""
    g = _golden("conv_relu_grad")
    assert _rel(g["relu_top_diff"] * (g["relu_bottom"] > 0), g["relu_bottom_diff"]) < 1e-9
    wf = DummyWorkflow()
    u = _conv_relu(wf, g["conv_bottom"], g["conv_weights"])
    assert _rel(u.output.mem, g["relu_top_flat"]) < 1e-4
    gd = gd_conv.GDStrictRELUConv(wf, kx=5, ky=5, padding=(2, 2, 2, 2), sliding=(1, 1), n_kernels=2,
                                  learning_rate=0.0, weights_decay=0.0, apply_gradient=False,
                                  gradient_moment=0.0)
    gd.err_output = Array(g["relu_top_diff"].copy())
    gd.link_attrs(u, "input", "output", "weights", "bias")
    gd.initialize(device="numpy")
    gd.run()
    assert _rel(gd.err_input.mem, g["conv_bottom_diff"]) < 1e-5
    assert _rel(gd.gradient_weights.mem.reshape(2, 5, 5, 3), g["conv_weight_delta"]) < 1e-3


def test_softmax_and_loss_gradient_match_caffe():
    """`softmax.txt`: softmax of the logits and the SoftmaxWithLoss gradient (p - onehot) / batch."""
    from veles.znicz_b200.ops import all2all
    from veles.znicz_b200.workflow import evaluator
    d = _golden("softmax")
    labels = d["labels"].astype(numpy.int32)
    logits, top, bottom_diff = d["sm_bottom"], d["sm_top"], d["sm_bottom_diff"]
    wf = DummyWorkflow()
    f = all2all.All2AllSoftmax(wf, output_sample_shape=10, weights_stddev=0.1)
    f.input = Array(logits.copy())
    f.initialize(device="numpy")
    f.weights.mem[:] = numpy.eye(10)
    f.bias.mem[:] = 0
    f.run()
    assert numpy.abs(f.output.mem - top).max() < 2e-6
    ev = evaluator.EvaluatorSoftmax(wf)
    ev.output, ev.max_idx = f.output, f.max_idx
    ev.labels = Array(labels.copy())
    ev.batch_size = 2
    ev.initialize(device="numpy")
    ev.run()
    assert numpy.abs(ev.err_output.mem - bottom_diff).max() < 2e-6
