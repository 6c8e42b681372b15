"""The band A operand of the wgmma conv weight gradient (stride 1, 8 / 16 / 32 input channels)
against the tap-mode gather it replaces: the same products in the same pixel order, so the
split-K partials and the bias partials are bit-identical.

The gather outputs come from a subprocess with ZNICZ_CONV_HALO=0 (the switch is read once per
process); both processes compute the same seeded inputs with ``_run_cases``."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# N, H, W, C, F, k, pad, stride
CASES = [
    (100, 32, 32, 8, 32, 5, 2, 1),     # CIFAR conv1 (3 channels padded to 8)
    (100, 16, 16, 32, 32, 5, 2, 1),    # CIFAR conv2
    (100, 8, 8, 32, 64, 5, 2, 1),      # CIFAR conv3
    (4, 16, 16, 16, 16, 3, 1, 1),      # 3x3, C = F = 16: a CTA that holds only the bias group
    (2, 6, 128, 8, 32, 5, 2, 1),       # OW = 128: k-blocks are 64-pixel row segments
    (3, 12, 12, 8, 16, 5, 0, 1),       # pad 0, 8x8 output
    # not served by the band kernel
    (6, 28, 28, 8, 64, 5, 0, 1),       # OW = 24
    (2, 15, 13, 8, 16, 3, 1, 2),       # strided
    (2, 8, 8, 64, 32, 3, 1, 1),        # C = 64
]


def _band(c, f, k, ow, oh, s):
    rows = ow % 8 == 0 and 64 % ow == 0
    return (s == 1 and c in (8, 16, 32) and f <= 64 and k <= 8 and (rows or ow % 64 == 0)
            and (oh * ow) % 64 == 0)


def _geometry(case):
    n, h, w, c, f, k, pad, s = case
    oh, ow = (h + 2 * pad - k) // s + 1, (w + 2 * pad - k) // s + 1
    return oh, ow, k * k * c


def _split_counts(ext, case):
    """1, the count the training step uses, 64, and one that leaves empty trailing splits."""
    n, h, w, c, f, k, pad, s = case
    oh, ow, kw = _geometry(case)
    kb = (n * oh * ow + 63) // 64
    counts = [1, int(ext.pick_splits(kw, f, n * oh * ow, 64)), 64]
    for sp in range(3, kb + 1):
        per = (kb + sp - 1) // sp
        if (kb + per - 1) // per < sp:
            counts.append(sp)
            break
    return counts


def _run_cases(ext):
    """Every case's partials and bias partials at each split count (return code and whether the
    guard slab behind each output stayed NaN), and the band launches each case made."""
    res = {}
    for i, case in enumerate(CASES):
        n, h, w, c, f, k, pad, s = case
        oh, ow, kw = _geometry(case)
        gen = torch.Generator().manual_seed(200 + i)
        x = torch.randn(n, h, w, c, generator=gen).bfloat16().cuda()
        eo = torch.randn(n, oh, ow, f, generator=gen).bfloat16().cuda()
        g = [n, h, w, c, oh, ow, f, k, k, s, s, pad, pad]
        h0 = ext.conv_halo_launches()
        runs = []
        for splits in _split_counts(ext, case):
            parts = torch.full((splits + 1, f, kw), float("nan"), device="cuda")
            bparts = torch.full((splits + 1, f), float("nan"), device="cuda")
            r = int(ext.conv_wgrad(eo, x, parts[:splits], splits, g, False, 1, bparts[:splits]))
            torch.cuda.synchronize()
            runs.append({"splits": splits, "r": r, "parts": parts[:splits].cpu(),
                         "bias": bparts[:splits].cpu(),
                         "guards": bool(torch.isnan(parts[splits:]).all() and
                                        torch.isnan(bparts[splits:]).all())})
        res[i] = {"runs": runs, "halo": ext.conv_halo_launches() - h0}
    return res


def _ext():
    from veles.znicz_b200.kernels import load_extension
    return load_extension(required=True)


@pytest.mark.gpu
def test_band_wgrad_matches_gather_bit_for_bit(tmp_path):
    assert os.environ.get("ZNICZ_CONV_HALO", "1") != "0", "run with the halo kernels enabled"
    out = str(tmp_path / "gather.pt")
    env = dict(os.environ, ZNICZ_CONV_HALO="0", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), out], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    ref = torch.load(out)
    got = _run_cases(_ext())
    for i, case in enumerate(CASES):
        n, h, w, c, f, k, pad, s = case
        oh, ow, _ = _geometry(case)
        want = len(got[i]["runs"]) if _band(c, f, k, ow, oh, s) else 0
        assert got[i]["halo"] == want, (case, got[i]["halo"], want)
        assert ref[i]["halo"] == 0, case
        for a, b in zip(got[i]["runs"], ref[i]["runs"]):
            sp = a["splits"]
            assert a["splits"] == b["splits"] and a["r"] == b["r"] and a["r"] in (0, 1), (case, sp)
            assert a["guards"] and b["guards"], (case, sp)
            assert not torch.isnan(a["parts"]).any(), (case, sp)
            # bit patterns, not values: -0 vs +0 or a NaN payload would count as a difference
            assert torch.equal(a["parts"].view(torch.int32), b["parts"].view(torch.int32)), (case, sp)
            if a["r"] == 1:
                assert not torch.isnan(a["bias"]).any(), (case, sp)
                assert torch.equal(a["bias"].view(torch.int32), b["bias"].view(torch.int32)), (case, sp)


@pytest.mark.gpu
def test_band_wgrad_matches_reference():
    """The band path against fp32 torch (the bit-exact test above only compares it with the
    gather kernel)."""
    got = _run_cases(_ext())
    for i, case in enumerate(CASES):
        n, h, w, c, f, k, pad, s = case
        oh, ow, kw = _geometry(case)
        gen = torch.Generator().manual_seed(200 + i)
        x = torch.randn(n, h, w, c, generator=gen).bfloat16().float()
        eo = torch.randn(n, oh, ow, f, generator=gen).bfloat16().float()
        wg = torch.nn.grad.conv2d_weight(x.permute(0, 3, 1, 2), (f, c, k, k),
                                         eo.permute(0, 3, 1, 2), stride=s, padding=pad)
        wg = wg.permute(0, 2, 3, 1).reshape(f, kw)        # [f][(ky * KX + kx) * C + c]
        bg = eo.reshape(-1, f).sum(0)
        for run in got[i]["runs"]:
            a = run["parts"].sum(0)
            err = float((a - wg).abs().max() / (wg.abs().max() + 1e-12))
            assert err < 5e-3, (case, run["splits"], err)
            if run["r"] == 1:
                b = run["bias"].sum(0)
                err = float((b - bg).abs().max() / (bg.abs().max() + 1e-12))
                assert err < 5e-3, (case, run["splits"], "bias", err)


if __name__ == "__main__":
    torch.save(_run_cases(_ext()), sys.argv[1])
