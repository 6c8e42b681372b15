"""multi_update_k MODE 1/2 (cross-rank reduce + update) on ONE GPU with 2 / 4 / 8 fake peers,
one-shot and two-shot, bit for bit against the single-GPU kernel fed the summed gradient."""
import json
import os
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("algo", [0, 1])
def test_fake_peer_update_desc_bit_exact(n, algo):
    r = subprocess.run([sys.executable, os.path.join(REPO, "tests", "fake_peer_worker.py"),
                        str(n), str(algo)], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, PYTHONPATH=REPO))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["finite"]
    assert res["oracle_vs_torch"] < 1e-5
    assert res["ranks_identical"], res
    assert res["equal_w"] and res["equal_v"], res
