"""Reference arm: drives the UNMODIFIED Samsung/veles.znicz CIFAR-10 sample
(``oracle/_ref/veles/znicz/samples/CIFAR10/cifar.py`` + ``cifar_caffe_config.py``) through
its own public API — ``run(load, main)`` → ``CifarWorkflow`` (StandardWorkflow) →
``initialize(device)`` → ``run()`` — on the stock ``cuda_run`` path of its units (NVRTC build of
its ``cuda/*.cu``, cuBLAS SGEMM). The absent Veles core / cuda4py / zope.interface are the shim
under ``baseline/veles_core``. Nothing of veles.znicz_b200 is imported in this process.

What is synthetic: the dataset (CIFAR-10 python pickles of random uint8 images written to a
temporary directory, read by the reference's own CifarLoader) and the launcher (the core's
``python -m veles`` CLI is replaced by ``launch()`` below).
"""
import importlib.util
import os
import pickle
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
CORE = os.path.join(HERE, "veles_core")
ORACLE = os.path.join(os.path.dirname(HERE), "oracle")
REF = os.path.join(ORACLE, "_ref", "veles", "znicz")


def ensure_reference():
    if not os.path.isfile(os.path.join(REF, "MANIFEST.sha256.json")):
        sys.path.insert(0, ORACLE)
        import install_reference
        install_reference.install()


def setup_path():
    ensure_reference()
    # the shim's ``veles`` must win over the product's ``veles`` package at the repo root
    sys.path[:] = [CORE] + [p for p in sys.path if os.path.abspath(p or ".") !=
                            os.path.dirname(HERE)]
    mod = sys.modules.get("veles")
    if mod is not None and not os.path.abspath(mod.__file__).startswith(CORE):
        raise RuntimeError("the product's veles package is already imported (%s): the reference "
                           "arm must run in its own process" % mod.__file__)


def write_synthetic_cifar(root_dir, n_train=50000, n_valid=10000, seed=1):
    """cifar-10-batches-py layout: data_batch_1..5 + test_batch, 10000 rows each (the
    reference's CifarLoader reshapes every pickle to (10000, 3, 32, 32))."""
    import numpy
    d = os.path.join(root_dir, "cifar-10-batches-py")
    os.makedirs(d, exist_ok=True)
    rs = numpy.random.RandomState(seed)
    protos = rs.randint(0, 256, (10, 3072)).astype(numpy.float32)

    protos = protos.astype(numpy.uint8) // 2

    def batch(path, n):
        labels = rs.randint(0, 10, n)
        data = protos[labels] + rs.randint(0, 128, (n, 3072), dtype=numpy.uint8)
        with open(path, "wb") as f:
            pickle.dump({"data": data, "labels": labels.tolist()}, f, protocol=2)
    assert n_train % 10000 == 0 and n_valid == 10000
    for i in range(1, 6):
        batch(os.path.join(d, "data_batch_%d" % i), 10000)
    batch(os.path.join(d, "test_batch"), n_valid)
    return d


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def launch(backend="cuda", data_dir=None, force_numpy_loader=False, layers=None,
           minibatch_size=None, pinned=False, log_level=None, loader_name=None):
    """The launcher's job: execute the config, let the sample build its workflow via
    ``run(load, main)``, initialise it on the device. Returns the workflow (not yet run)."""
    setup_path()
    import logging
    from veles.logger import setup_logging
    setup_logging(log_level if log_level is not None else logging.WARNING)
    from veles.config import root
    from veles.backends import CUDADevice, NumpyDevice
    from veles.dummy import DummyLauncher
    import veles.znicz  # noqa: F401  (adds its cuda/ dir to root.common.engine.source_dirs)

    data_dir = data_dir or os.environ.get("ZNICZ_REF_DATA_DIR") or \
        tempfile.mkdtemp(prefix="ref_cifar_")
    root.common.dirs.datasets = data_dir
    if loader_name is None and not os.path.isdir(os.path.join(data_dir, "cifar-10-batches-py")):
        write_synthetic_cifar(data_dir)
    root.common.engine.backend = backend
    root.common.disable.snapshotting = True
    root.common.disable.plotting = True

    sample_dir = os.path.join(REF, "samples", "CIFAR10")
    _load_module("cifar_caffe_config", os.path.join(sample_dir, "cifar_caffe_config.py"))
    # launcher-level overrides (what ``python -m veles ... root.cifar.x=y`` does)
    root.cifar.add_plotters = False
    root.cifar.image_saver.do = False
    root.cifar.loader.force_numpy = bool(force_numpy_loader)
    if minibatch_size:
        root.cifar.loader.minibatch_size = minibatch_size
    if layers is not None:
        root.cifar.layers = layers
    if loader_name is not None:          # tests: a tiny registered loader instead of the pickles
        root.cifar.loader_name = loader_name
    cifar = _load_module("cifar_sample", os.path.join(sample_dir, "cifar.py"))

    state = {}

    def load(workflow_class, **kwargs):
        launcher = DummyLauncher()
        wf = workflow_class(launcher, **kwargs)
        state["workflow"] = wf
        return wf, False

    def main(**kwargs):
        wf = state["workflow"]
        device = CUDADevice(pinned=pinned) if backend == "cuda" else NumpyDevice()
        wf.initialize(device=device, **kwargs)
        state["device"] = device

    cifar.run(load, main)
    return state["workflow"], state["device"]


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="cuda")
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    wf, dev = launch(args.backend)
    n = wf.run(iterations=args.steps)
    dev.sync()
    wf.evaluator.n_err.map_read()
    print("ran %d minibatches; n_err %s" % (n, wf.evaluator.n_err.mem))
