"""The whole-sequence LSTM unit (ops/lstm_seq.py) in the native runtime: packages exported from
trained ``lstm_seq`` workflows run on the CPU executor (checked against the workflow's own forward
chain) and on the sm_90a executor (split-bf16 wgmma per time step, checked against the CPU)."""
import json
import os
import subprocess
import zipfile

import numpy
import pytest

from veles.znicz_b200 import native
from veles.znicz_b200.core.config import root
from veles.znicz_b200.models import lstm_seq

GD = {"learning_rate": 0.05, "learning_rate_bias": 0.05, "gradient_moment": 0.9,
      "gradient_moment_bias": 0.9, "weights_decay": 0.0}


def _lstm(hidden, seq=False):
    return {"type": "lstm_seq", "<-": dict(GD),
            "->": {"output_sample_shape": hidden, "return_sequences": seq, "weights_stddev": 0.3}}


def _softmax(n):
    return {"type": "softmax", "<-": dict(GD),
            "->": {"output_sample_shape": n, "weights_stddev": 0.1}}


# name -> (seq_len, features, layers); the last one has I + H = 33 >= 32 inputs per gate row, so the
# CUDA executor splits it for the tensor cores with padding (K8 = 40) and N = 4H = 52
SHAPES = {
    "single": (5, 7, [_lstm(12), _softmax(4)]),
    "sequences": (5, 7, [_lstm(12, True), _softmax(4)]),
    "stack": (5, 7, [_lstm(12, True), _lstm(9, True), _softmax(4)]),
    "padded": (5, 20, [_lstm(13), _softmax(4)]),
}


def _train(seq_len, features, layers, batch=8):
    """One numpy epoch of a tiny lstm_seq workflow."""
    root.common.disable.snapshotting = True
    wf = lstm_seq.build(seq_len=seq_len, features=features, n_classes=layers[-1]["->"]["output_sample_shape"],
                        layers=layers,
                        loader_config={"minibatch_size": batch, "n_train": 2 * batch, "n_valid": batch,
                                       "noise": 0.2},
                        decision_config={"max_epochs": 1, "fail_iterations": 10})
    wf.initialize(device="numpy")
    wf.run()
    return wf


def _workflow_forward(wf):
    x = wf.loader.minibatch_data.mem.copy()
    for u in wf.forwards:
        u.run()
    return x, wf.forwards[-1].output.mem.copy()


def _rewrite(pkg, dst, edit):
    """Copies a zip package to ``dst`` with ``edit(contents)`` applied to contents.json."""
    with zipfile.ZipFile(pkg) as src, zipfile.ZipFile(dst, "w") as out:
        for name in src.namelist():
            data = src.read(name)
            if name == "contents.json":
                contents = json.loads(data.decode())
                edit(contents)
                data = json.dumps(contents).encode()
            out.writestr(name, data)
    return dst


@pytest.mark.parametrize("precision", [32, 16])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_native_lstm_cpu_matches_workflow(tmp_path, shape, precision):
    wf = _train(*SHAPES[shape])
    pkg = str(tmp_path / "lstm.zip")
    wf.package_export(pkg, precision=precision)
    eng = native.NativeEngine(pkg)
    assert eng.num_units == len(wf.forwards)
    x, ref = _workflow_forward(wf)
    assert x.ndim == 3
    y = eng.run(x)
    assert y.shape == ref.shape
    assert numpy.abs(y - ref).max() < (1e-5 if precision == 32 else 2e-3)
    # a sample may also come flattened to [n, T * I]
    assert numpy.array_equal(eng.run(x.reshape(len(x), -1)), y)


def test_native_lstm_shapes(tmp_path):
    wf = _train(*SHAPES["stack"])
    pkg = str(tmp_path / "lstm.zip")
    wf.package_export(pkg)
    eng = native.NativeEngine(pkg)
    assert [f.output.shape for f in wf.forwards] == [(8, 5, 12), (8, 5, 9), (8, 4)]
    # only the stack's first unit: the [T][H] sequence of every sample
    first = native.NativeEngine(_rewrite(pkg, str(tmp_path / "first.zip"),
                                         lambda c: c.update(units=c["units"][:1])))
    x, _ = _workflow_forward(wf)
    h = first.run(x)
    assert h.shape == (8, 5, 1, 12)
    assert numpy.abs(h.reshape(8, 5, 12) - wf.forwards[0].output.mem).max() < 1e-5
    with pytest.raises(ValueError):
        eng.run(numpy.zeros((2, 13), numpy.float32))     # 13 is not a multiple of I = 7


def test_native_lstm_rejects_transposed_weights(tmp_path):
    wf = _train(*SHAPES["single"])
    pkg = str(tmp_path / "lstm.zip")
    wf.package_export(pkg)

    def transpose(contents):
        contents["units"][0]["data"]["weights_transposed"] = True
    bad = _rewrite(pkg, str(tmp_path / "bad.zip"), transpose)
    with pytest.raises(RuntimeError, match="LSTMSequence.*weights_transposed"):
        native.NativeEngine(bad)


def _functional(tmp_path, pkg, x, ref):
    from veles.znicz_b200.native import _build_impl
    _build_impl.build(verbose=False)
    numpy.save(str(tmp_path / "x.npy"), x)
    numpy.save(str(tmp_path / "ref.npy"), ref.astype(numpy.float32))
    r = subprocess.run([_build_impl.TEST_BIN, pkg, str(tmp_path / "x.npy"), str(tmp_path / "ref.npy")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
    assert "0 failures" in r.stdout and "functional cpu" in r.stdout, r.stdout
    return r.stdout


def test_native_lstm_cpp_functional(tmp_path):
    wf = _train(*SHAPES["stack"])
    pkg = str(tmp_path / "lstm.zip")
    wf.package_export(pkg)
    _functional(tmp_path, pkg, *_workflow_forward(wf))


# ------------------------------------------------------------------------------------------ GPU
def _tc_off():
    os.environ["ZNICZ_NATIVE_TC"] = "0"


def _tc_restore():
    del os.environ["ZNICZ_NATIVE_TC"]


def _cuda_matches_cpu(pkg, x):
    eng = native.NativeEngine(pkg)
    cpu = eng.run(x, "cpu")
    assert numpy.abs(eng.run(x, "cuda") - cpu).max() < 1e-4
    _tc_off()
    try:
        simt = native.NativeEngine(pkg)
        assert numpy.abs(simt.run(x, "cuda") - cpu).max() < 1e-4
        assert simt.tensor_core_launches == 0
    finally:
        _tc_restore()
    return eng, cpu


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_native_lstm_cuda_matches_cpu(tmp_path, shape):
    wf = _train(*SHAPES[shape])
    pkg = str(tmp_path / "lstm.zip")
    wf.package_export(pkg)
    x = numpy.random.RandomState(3).uniform(-1, 1, wf.loader.minibatch_data.shape).astype(numpy.float32)
    _cuda_matches_cpu(pkg, x)


BENCH = dict(seq_len=32, features=128, hidden=256, n_classes=10)


def _bench_package(tmp_path, seq):
    # the benchmark model's own layers and weight scales: the 3-part split leaves ~2^-16 |x| |w| per
    # product, so its error grows with |z| (weights 6x the model's, |z| ~ 10, land near 1e-4)
    layers = lstm_seq.layers(BENCH["hidden"], BENCH["n_classes"])
    layers[0]["->"]["return_sequences"] = seq
    wf = _train(BENCH["seq_len"], BENCH["features"], layers, batch=128)
    pkg = str(tmp_path / ("lstm_seq.zip" if seq else "lstm.zip"))
    wf.package_export(pkg)
    return wf, pkg


@pytest.mark.gpu
@pytest.mark.parametrize("seq", [False, True])
def test_native_lstm_cuda_benchmark_shape(tmp_path, seq):
    wf, pkg = _bench_package(tmp_path, seq)
    for batch in (128, 130):           # 130 rows span two M tiles of the GEMM
        x = numpy.random.RandomState(batch).uniform(-1, 1, (batch, BENCH["seq_len"], BENCH["features"]))
        eng, cpu = _cuda_matches_cpu(pkg, x.astype(numpy.float32))
        assert cpu.shape == (batch, BENCH["n_classes"])
        # T tensor-core GEMMs for the LSTM unit and one for the softmax layer, on every run
        before = eng.tensor_core_launches
        eng.run(x, "cuda")
        assert eng.tensor_core_launches - before == BENCH["seq_len"] + 1
    # the LSTM unit's own output, before the softmax flattens it
    lstm_only = _rewrite(pkg, str(tmp_path / "first.zip"), lambda c: c.update(units=c["units"][:1]))
    x = numpy.random.RandomState(7).uniform(-1, 1, (128, BENCH["seq_len"], BENCH["features"]))
    _cuda_matches_cpu(lstm_only, x.astype(numpy.float32))


@pytest.mark.gpu
def test_native_lstm_cpp_functional_cuda(tmp_path):
    wf, pkg = _bench_package(tmp_path, False)
    out = _functional(tmp_path, pkg, *_workflow_forward(wf))
    assert "functional cuda" in out, out
