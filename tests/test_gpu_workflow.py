"""End-to-end StandardWorkflow on a real H100: eager + CUDA-graph segments, fp32 + bf16."""
import numpy
import pytest

from veles.znicz_b200.core.config import root
from veles.znicz_b200.models import cifar, mnist

pytestmark = pytest.mark.gpu


def _fast_layers():
    layers = cifar.caffe_layers()
    for l in layers:
        if "<-" in l:
            l["<-"].update(learning_rate=0.02, learning_rate_bias=0.02, weights_decay=0.0005)
        if l["type"] == "conv":
            l["->"]["weights_stddev"] = 0.05
    return layers


@pytest.mark.parametrize("compute,graphs", [("fp32", False), ("bf16", False), ("bf16", True)])
def test_cifar_trains_on_gpu(compute, graphs):
    root.common.engine.compute_type = compute
    try:
        wf = cifar.build(
            layers=_fast_layers(), use_graphs=graphs,
            loader_config={"minibatch_size": 20, "n_train": 400, "n_valid": 100,
                           "normalization_type": "internal_mean", "noise": 0.3},
            decision_config={"max_epochs": 5, "fail_iterations": 50},
            snapshotter_config={"prefix": "cifar_g", "interval": 1, "time_interval": 0})
        wf.initialize(device="cuda")
        wf.run()
        dec = wf.decision
        assert bool(dec.complete)
        assert dec.best_n_err_pt[1] < 50.0, dec.best_n_err_pt
        wf.forwards[0].weights.map_read()
        assert numpy.isfinite(wf.forwards[0].weights.mem).all()
        if graphs:
            assert all(s.replays > 0 for s in wf.segments_), [
                (s.name, s.replays, s.eager_runs) for s in wf.segments_]
    finally:
        root.common.engine.compute_type = "fp32"


def test_mnist_conv_fp32_gpu():
    """The genetically tuned MnistConv hyper-parameters need the full 60k dataset to
    converge (the same tiny run gives ~80% error on the numpy backend too), so this only
    checks that the conv/pool/relu/softmax GPU chain trains to completion with finite
    weights; learning on the GPU is asserted by the LeNet run below."""
    wf = mnist.build(
        loader_config={"minibatch_size": 6, "n_train": 120, "n_valid": 36,
                       "normalization_type": "linear", "noise": 0.3},
        decision_config={"max_epochs": 3, "fail_iterations": 10},
        snapshotter_config={"prefix": "mnist_g", "interval": 1, "time_interval": 0,
                            "compression": ""})
    wf.initialize(device="cuda")
    wf.run()
    assert bool(wf.decision.complete)
    for f in wf.forwards:
        if getattr(f, "weights", None):
            f.weights.map_read()
            assert numpy.isfinite(f.weights.mem).all(), f.name


@pytest.mark.parametrize("compute", ["fp32", "bf16"])
def test_mnist_lenet_gpu(compute):
    root.common.engine.compute_type = compute
    try:
        wf = mnist.build(
            layers=mnist.caffe_layers(),
            loader_config={"minibatch_size": 12, "n_train": 240, "n_valid": 60,
                           "normalization_type": "linear", "noise": 0.3},
            decision_config={"max_epochs": 4, "fail_iterations": 10},
            snapshotter_config={"prefix": "lenet_g", "interval": 1, "time_interval": 0,
                                "compression": ""})
        wf.initialize(device="cuda")
        wf.run()
        assert bool(wf.decision.complete)
        assert wf.decision.best_n_err_pt[1] < 25.0, wf.decision.best_n_err_pt
    finally:
        root.common.engine.compute_type = "fp32"


def test_fused_step_equals_per_layer_updates():
    """One whole-network step launch == per-tensor update launches (same weights after a few
    minibatches, fp32 so the comparison is tight)."""
    results = []
    from veles.znicz_b200.core import prng
    for fused in (False, True):
        root.common.engine.fused_step = fused
        prng.get(1).seed(1234)
        prng.get(2).seed(5678)
        try:
            wf = cifar.build(
                layers=_fast_layers(), use_graphs=False,
                loader_config={"minibatch_size": 20, "n_train": 200, "n_valid": 40,
                               "normalization_type": "internal_mean", "noise": 0.3},
                decision_config={"max_epochs": 1, "fail_iterations": 10},
                snapshotter_config={"prefix": "cifar_fs", "interval": 100,
                                    "time_interval": 1e9})
            wf.initialize(device="cuda")
            assert (wf.fused_step_ is not None) == fused
            wf.run()
            if fused:
                assert wf.fused_step_.launches == 10      # one per train minibatch
            ws = []
            for f in wf.forwards:
                if getattr(f, "weights", None):
                    f.weights.map_read()
                    f.bias.map_read()
                    ws.append((f.weights.mem.copy(), f.bias.mem.copy()))
            results.append(ws)
        finally:
            root.common.engine.fused_step = True
    for (wa, ba), (wb, bb) in zip(*results):
        assert numpy.abs(wa - wb).max() <= 1e-4 * max(1.0, numpy.abs(wa).max())
        assert numpy.abs(ba - bb).max() <= 1e-4 * max(1.0, numpy.abs(ba).max())


def test_fp32_tensor_core_training_matches_simt():
    """10 fp32 training steps with the split-bf16 tensor-core layers (kernels/fp32x.py, stacked
    operands handed from the forward to the backward units from step 2 on) end at the same
    weights as the SIMT fp32 kernels."""
    from veles.znicz_b200.core import prng
    from veles.znicz_b200.kernels import fp32x
    results = []
    for tc in (False, True):
        root.common.engine.fp32_tensor_cores = tc
        prng.get(1).seed(1234)
        prng.get(2).seed(5678)
        before = fp32x.counters["gemms"]
        try:
            wf = cifar.build(
                layers=_fast_layers(), use_graphs=False,
                loader_config={"minibatch_size": 20, "n_train": 200, "n_valid": 40,
                               "normalization_type": "internal_mean", "noise": 0.3},
                decision_config={"max_epochs": 1, "fail_iterations": 10},
                snapshotter_config={"prefix": "cifar_x3", "interval": 100,
                                    "time_interval": 1e9})
            wf.initialize(device="cuda")
            wf.run()
            assert (fp32x.counters["gemms"] > before) == tc
            ws = []
            for f in wf.forwards:
                if getattr(f, "weights", None):
                    f.weights.map_read()
                    ws.append(f.weights.mem.copy())
            results.append(ws)
        finally:
            root.common.engine.fp32_tensor_cores = True
    for wa, wb in zip(*results):
        assert numpy.isfinite(wb).all()
        assert numpy.abs(wa - wb).max() <= 2e-3 * numpy.abs(wa).max()


@pytest.mark.parametrize("compute,tol", [("fp32", 2e-4), ("bf16", 4e-2)])
def test_activation_fusion_equals_separate_units(compute, tol):
    """conv→relu / maxpool→relu / conv→relu folded into the producers' kernels (forward), the
    derivative folded into the pooling backward and - bf16 - the bias gradient delivered by the
    wgmma wgrad kernel must train like the stand-alone units (eager)."""
    from veles.znicz_b200.core import prng
    results, counts = [], []
    for fuse in (False, True):
        root.common.engine.fuse_activations = fuse
        root.common.engine.compute_type = compute
        prng.get(1).seed(1234)
        prng.get(2).seed(5678)
        try:
            wf = cifar.build(
                layers=_fast_layers(), use_graphs=False,
                loader_config={"minibatch_size": 20, "n_train": 200, "n_valid": 40,
                               "normalization_type": "internal_mean", "noise": 0.3},
                decision_config={"max_epochs": 1, "fail_iterations": 10},
                snapshotter_config={"prefix": "cifar_fa", "interval": 100,
                                    "time_interval": 1e9})
            wf.initialize(device="cuda")
            counts.append(wf.fused_activations_)
            from veles.znicz_b200.kernels import api
            n0 = api.counters["launches"]
            wf.run()
            launches = api.counters["launches"] - n0
            ws = []
            for f in wf.forwards:
                if getattr(f, "weights", None):
                    f.weights.map_read()
                    ws.append(f.weights.mem.copy())
            results.append((ws, launches, wf.decision.epoch_n_err[2]))
        finally:
            root.common.engine.fuse_activations = True
            root.common.engine.compute_type = "fp32"
    assert counts == [0, 3]
    (wa, la, ea), (wb, lb, eb) = results
    assert lb < la                       # fewer launches per training step
    for a, b in zip(wa, wb):
        assert numpy.abs(a - b).max() <= tol * max(1.0, numpy.abs(a).max())
    if compute == "fp32":
        assert ea == eb


@pytest.mark.parametrize("family", ["alexnet", "nin", "vgga"])
def test_imagenet_models_step_on_gpu(family):
    """Full-size AlexNet (grouped) / NiN / 13-conv VGG, bf16, a few training steps on synthetic
    227x227 (224 for VGG) images: exercises stride-4 11x11 convs on the channel-padded path,
    3x3/1x1 convs with 64..1024 channels, 9216x4096 FC layers, dropout, LRN, ZeroFiller."""
    from veles.znicz_b200.models import alexnet
    root.common.engine.compute_type = "bf16"
    try:
        side = 224 if family == "vgga" else 227
        layers = {"alexnet": alexnet.alexnet_layers, "nin": alexnet.nin_layers,
                  "vgga": alexnet.vgga_layers}[family](n_classes=20)
        wf = alexnet.build(
            loader_name="synthetic_imagenet", layers=layers,
            loader_config={"minibatch_size": 8, "shape": (side, side, 3), "n_classes": 20,
                           "n_train": 24, "n_valid": 8, "noise": 0.3,
                           "normalization_type": "internal_mean"},
            decision_config={"max_epochs": 1, "fail_iterations": 5},
            snapshotter_config={"prefix": "inet_g", "interval": 1000, "time_interval": 1e9})
        wf.initialize(device="cuda")
        wf.run()
        assert bool(wf.decision.complete)
        for f in wf.forwards:
            if getattr(f, "weights", None):
                f.weights.map_read()
                assert numpy.isfinite(f.weights.mem).all(), f.name
        wf.forwards[-1].output.map_read()
        out = wf.forwards[-1].output.mem
        assert numpy.isfinite(out).all() and abs(float(out[0].sum()) - 1.0) < 1e-2
    finally:
        root.common.engine.compute_type = "fp32"


@pytest.mark.parametrize("compute", ["fp32", "bf16"])
@pytest.mark.parametrize("on_device", [False, True])
def test_loader_minibatch_on_device_matches_host(compute, on_device):
    """Streaming (packed pinned slot filled by the native gather, one H2D per step) and
    device-resident (index upload + gather kernel) loaders must both deliver
    original_data[indices] / labels[indices] on the device, padded tail zero / -1."""
    from veles.znicz_b200.core.workflow import DummyWorkflow
    from veles.znicz_b200.loader.synthetic import SyntheticImageLoader
    root.common.engine.compute_type = compute
    try:
        wf = DummyWorkflow()
        ld = SyntheticImageLoader(wf, minibatch_size=32, shape=(8, 8, 3), n_classes=5,
                                  n_train=80, n_valid=40, n_test=0, on_device=on_device)
        ld.initialize(device="cuda")
        if not on_device:
            assert ld._packed_ is not None and ld.h2d_bytes_per_step < 2 * 32 * 192 * 4
        for _ in range(7):              # 40 = 32 + 8 (short minibatch), then train 32 + 32 + 16
            ld.run()
            n = int(ld.minibatch_size)
            idx = ld.minibatch_indices.mem[:n].copy()
            ref = ld.original_data.mem[idx]
            ld.minibatch_data.map_read()
            got = ld.minibatch_data.mem
            tol = 0 if compute == "fp32" else 1e-2
            assert numpy.abs(got[:n] - ref).max() <= tol * max(1.0, numpy.abs(ref).max())
            assert not got[n:].any()
            ld.minibatch_labels.map_read()
            lab = ld.minibatch_labels.mem
            numpy.testing.assert_array_equal(lab[:n], ld._mapped_original_labels.mem[idx])
            assert (lab[n:] == -1).all()
    finally:
        root.common.engine.compute_type = "fp32"
