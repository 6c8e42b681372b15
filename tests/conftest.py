import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs an H100 GPU")
    config.addinivalue_line("markers", "slow: long-running test")


def _has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_cuda():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _fresh_config(tmp_path):
    from veles.znicz_b200.core.config import root
    from veles.znicz_b200.core import prng
    root.common.dirs.snapshots = str(tmp_path / "snapshots")
    root.common.engine.backend = "numpy"
    root.common.engine.precision_type = "float"
    root.common.engine.compute_type = "fp32"
    prng.get(1).seed(1234)
    prng.get(2).seed(5678)
    disable = {k: root.common.disable.get(k) for k in ("plotting", "snapshotting", "publishing")}
    yield
    for k, v in disable.items():
        setattr(root.common.disable, k, v)
