"""The persistent halo conv kernel (``conv_halo_persist_k``: filter resident in shared memory, one
8x8 pixel block per work item) against the one-tile-per-CTA halo kernel it replaces
(ZNICZ_CONV_HALO_PERSIST=0) and against the tap-mode gather (ZNICZ_CONV_HALO=0), for fprop and
dgrad: the same products in the same order, so bit-identical results.

Each reference comes from a subprocess (the switches are read once per process); every process
computes the same seeded inputs with ``_run_cases``. The kernels that ran are read from
``torch.profiler``, so that shapes the persistent kernel must not take are checked too."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PERSIST = "conv_halo_persist_k"

# N, H, W, C, F, k, pad (stride 1)
CASES = [
    (100, 32, 32, 8, 32, 5, 2),      # CIFAR conv1 (3 channels padded to 8): 1600 items
    (100, 16, 16, 32, 32, 5, 2),     # CIFAR conv2: fprop and dgrad
    (100, 8, 8, 32, 64, 5, 2),       # CIFAR conv3: F = 64 as two 32-column items per block
    (3, 20, 20, 8, 32, 5, 2),        # ragged: 20x20 is not a multiple of the 8x8 block
    (3, 20, 20, 32, 16, 5, 2),       # ragged dgrad (C = 32), 16-column fprop
    (2, 10, 10, 16, 16, 3, 1),       # 3x3, C = F = 16 (its dgrad stays on A_HALO: C <= 16)
    (6, 28, 28, 8, 64, 5, 0),        # MNIST conv1-like: pad 0, 24x24 output
    (1, 16, 16, 32, 32, 5, 2),       # 4 items: fewer than the SMs
    (2, 16, 16, 64, 32, 5, 2),       # dgrad C = 64: two 32-column items per block
    (9, 32, 32, 8, 32, 5, 2),        # 144 items: just above 132 SMs
    (600, 16, 16, 32, 32, 5, 2),     # 2400 items: many per CTA, the halo ring wraps
    # N = 128 (fprop F = 128; dgrad C = 128): A_HALO, not the persistent kernel
    (2, 16, 16, 32, 128, 5, 2),
    (2, 16, 16, 128, 32, 5, 2),
]


def _persist_fprop(c, f):
    return c in (8, 16, 32) and f <= 64


def _persist_dgrad(c, f):
    return f in (16, 32) and 16 < c <= 64


def _ran_persist(prof):
    return any(PERSIST in e.name for e in prof.events())


def _run_cases(ext):
    """Every case's fprop (bias + strict ReLU), dgrad (alpha 0.5) and dgrad with the folded
    strict-ReLU derivative, whether the NaN guard behind each output stayed NaN, and whether the
    persistent kernel ran for the fprop / the dgrads."""
    from torch.profiler import ProfilerActivity, profile
    res = {}
    for i, (n, h, w, c, f, k, pad) in enumerate(CASES):
        gen = torch.Generator().manual_seed(300 + i)
        oh, ow = h + 2 * pad - k + 1, w + 2 * pad - k + 1
        kw = k * k * c
        x = torch.randn(n, h, w, c, generator=gen).bfloat16().cuda()
        wl = (torch.randn(f, kw, generator=gen) / kw ** 0.5).bfloat16().cuda()
        wd = (torch.randn(k * k * f, c, generator=gen) / (k * k * f) ** 0.5).bfloat16().cuda()
        bias = torch.randn(f, generator=gen).cuda()
        eo = torch.randn(n, oh, ow, f, generator=gen).bfloat16().cuda()
        xin = torch.randn(n, h, w, c, generator=gen).bfloat16().cuda()
        g = [n, h, w, c, oh, ow, f, k, k, 1, 1, pad, pad]
        big = torch.full((2 * n, oh, ow, f), float("nan"), device="cuda", dtype=torch.bfloat16)
        bei = torch.full((2 * n, h, w, c), float("nan"), device="cuda", dtype=torch.bfloat16)
        bei2 = torch.full_like(bei, float("nan"))
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as pf:
            assert ext.conv_fprop(x, wl, kw, False, bias, big[:n], g, 3, 1) == 0
            torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as pd:
            assert ext.conv_dgrad(eo, wd, c, False, bei[:n], g, 0.5, 0.0, 1, None, 0) == 0
            assert ext.conv_dgrad(eo, wd, c, False, bei2[:n], g, 1.0, 0.0, 1, xin, 3) == 0
            torch.cuda.synchronize()
        res[i] = {"fprop": big[:n].cpu(), "dgrad": bei[:n].cpu(), "dgrad_f": bei2[:n].cpu(),
                  "guards": bool(torch.isnan(big[n:]).all() and torch.isnan(bei[n:]).all() and
                                 torch.isnan(bei2[n:]).all()),
                  "persist_fprop": _ran_persist(pf), "persist_dgrad": _ran_persist(pd)}
    return res


def _ext():
    from veles.znicz_b200.kernels import load_extension
    return load_extension(required=True)


def _reference(tmp_path, name, **env):
    out = str(tmp_path / (name + ".pt"))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), out],
                       env=dict(os.environ, PYTHONPATH=ROOT, **env), cwd=ROOT,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    return torch.load(out)


@pytest.mark.gpu
def test_persistent_halo_matches_halo_and_gather_bit_for_bit(tmp_path):
    assert os.environ.get("ZNICZ_CONV_HALO", "1") != "0", "run with the halo kernels enabled"
    assert os.environ.get("ZNICZ_CONV_HALO_PERSIST", "1") != "0", "run with the persistent kernel"
    refs = {"halo": _reference(tmp_path, "halo", ZNICZ_CONV_HALO_PERSIST="0"),
            "gather": _reference(tmp_path, "gather", ZNICZ_CONV_HALO="0")}
    got = _run_cases(_ext())
    for i, case in enumerate(CASES):
        c, f = case[3], case[4]
        assert got[i]["persist_fprop"] == _persist_fprop(c, f), case
        assert got[i]["persist_dgrad"] == _persist_dgrad(c, f), case
        assert got[i]["guards"], case
        for name, ref in refs.items():
            assert not ref[i]["persist_fprop"] and not ref[i]["persist_dgrad"], (name, case)
            assert ref[i]["guards"], (name, case)
            for key in ("fprop", "dgrad", "dgrad_f"):
                a, b = got[i][key], ref[i][key]
                assert not torch.isnan(a.float()).any(), (name, case, key)
                # bit patterns, not values: -0 vs +0 or a NaN payload would count as a difference
                assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (name, case, key)


if __name__ == "__main__":
    torch.save(_run_cases(_ext()), sys.argv[1])
