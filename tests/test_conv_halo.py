"""The halo-tile A operand of the wgmma conv kernel (stride 1, 8 / 16 / 32 inner channels) against
the tap-mode gather it replaces: the same products in the same order, so bit-identical results.

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
    (100, 8, 8, 32, 64, 5, 2, 1),      # CIFAR conv3 (its dgrad has F = 64: TMA im2col)
    (3, 20, 20, 8, 32, 5, 2, 1),       # ragged: 20x20 is not a multiple of the 8x8 block
    (2, 10, 10, 16, 16, 3, 1, 1),      # 3x3, C = F = 16, odd number of blocks
    (6, 28, 28, 8, 64, 5, 0, 1),       # MNIST conv1-like: pad 0, 24x24 output
    # not served by the halo kernel
    (2, 9, 9, 64, 64, 3, 1, 1),        # C % 64 == 0: TMA im2col
    (2, 15, 13, 8, 16, 3, 1, 2),       # strided
]


def _halo_fprop(c, stride):
    return stride == 1 and c in (8, 16, 32)


def _halo_dgrad(f, stride):
    return stride == 1 and f in (16, 32)


def _run_cases(ext):
    """Every case's fprop (bias + strict ReLU) and dgrad (plain and with the folded strict-ReLU
    derivative), the halo launches each made, and whether the guard behind each output stayed
    NaN."""
    res = {}
    for i, (n, h, w, c, f, k, pad, s) in enumerate(CASES):
        gen = torch.Generator().manual_seed(100 + i)
        oh, ow = (h + 2 * pad - k) // s + 1, (w + 2 * pad - k) // s + 1
        kw = k * k * c
        x = torch.randn(n, h, w, c, generator=gen).bfloat16().cuda()
        wl = (torch.randn(f, kw, generator=gen) / kw ** 0.5).bfloat16().cuda()
        wd = (torch.randn(k * k * f, c, generator=gen) / (k * k * f) ** 0.5).bfloat16().cuda()
        bias = torch.randn(f, generator=gen).cuda()
        eo = torch.randn(n, oh, ow, f, generator=gen).bfloat16().cuda()
        xin = torch.randn(n, h, w, c, generator=gen).bfloat16().cuda()
        g = [n, h, w, c, oh, ow, f, k, k, s, s, pad, pad]
        h0 = ext.conv_halo_launches()
        big = torch.full((2 * n, oh, ow, f), float("nan"), device="cuda", dtype=torch.bfloat16)
        assert ext.conv_fprop(x, wl, kw, False, bias, big[:n], g, 3, 1) == 0
        bei = torch.full((2 * n, h, w, c), float("nan"), device="cuda", dtype=torch.bfloat16)
        assert ext.conv_dgrad(eo, wd, c, False, bei[:n], g, 1.0, 0.0, 1, None, 0) == 0
        bei2 = torch.full_like(bei, float("nan"))
        assert ext.conv_dgrad(eo, wd, c, False, bei2[:n], g, 1.0, 0.0, 1, xin, 3) == 0
        torch.cuda.synchronize()
        res[i] = {"fprop": big[:n].cpu(), "dgrad": bei[:n].cpu(), "dgrad_f": bei2[:n].cpu(),
                  "guards": bool(torch.isnan(big[n:]).all() and torch.isnan(bei[n:]).all() and
                                 torch.isnan(bei2[n:]).all()),
                  "halo": ext.conv_halo_launches() - h0}
    return res


def _ext():
    from veles.znicz_b200.kernels import load_extension
    return load_extension(required=True)


@pytest.mark.gpu
def test_halo_matches_gather_bit_for_bit(tmp_path):
    assert os.environ.get("ZNICZ_CONV_HALO", "1") != "0", "run with the halo kernel enabled"
    out = str(tmp_path / "gather.pt")
    env = dict(os.environ, ZNICZ_CONV_HALO="0", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), out], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    ref = torch.load(out)
    got = _run_cases(_ext())
    for i, (n, h, w, c, f, k, pad, s) in enumerate(CASES):
        case = CASES[i]
        want = int(_halo_fprop(c, s)) + 2 * int(_halo_dgrad(f, s))
        assert got[i]["halo"] == want, (case, got[i]["halo"], want)
        assert ref[i]["halo"] == 0, case
        assert got[i]["guards"] and ref[i]["guards"], case
        for key in ("fprop", "dgrad", "dgrad_f"):
            a, b = got[i][key], ref[i][key]
            assert not torch.isnan(a.float()).any(), (case, key)
            # bit patterns, not values: -0 vs +0 or a NaN payload would count as a difference
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (case, key)


@pytest.mark.gpu
def test_halo_fprop_dgrad_match_reference():
    """The halo path against fp32 torch convolutions (the bit-exact test above only compares it
    with the gather kernel)."""
    ext = _ext()
    got = _run_cases(ext)
    for i, (n, h, w, c, f, k, pad, s) in enumerate(CASES):
        gen = torch.Generator().manual_seed(100 + i)
        kw = k * k * c
        x = torch.randn(n, h, w, c, generator=gen).bfloat16().float()
        wl = (torch.randn(f, kw, generator=gen) / kw ** 0.5).bfloat16().float()
        wd = (torch.randn(k * k * f, c, generator=gen) / (k * k * f) ** 0.5).bfloat16().float()
        bias = torch.randn(f, generator=gen)
        oh, ow = (h + 2 * pad - k) // s + 1, (w + 2 * pad - k) // s + 1
        eo = torch.randn(n, oh, ow, f, generator=gen).bfloat16().float()
        xin = torch.randn(n, h, w, c, generator=gen).bfloat16().float()
        wt = wl.view(f, k, k, c).permute(0, 3, 1, 2)
        y = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), wt, bias, stride=s, padding=pad)
        y = torch.relu(y).permute(0, 2, 3, 1)
        # dgrad operand [tap][f][c] -> the forward filter it is the transpose of: [f][c][ky][kx]
        wdt = wd.view(k, k, f, c).permute(2, 3, 0, 1)
        ei = torch.nn.grad.conv2d_input((n, c, h, w), wdt, eo.permute(0, 3, 1, 2), stride=s,
                                        padding=pad).permute(0, 2, 3, 1)
        for key, ref in (("fprop", y), ("dgrad", ei), ("dgrad_f", ei * (xin > 0))):
            a = got[i][key].float()
            err = float((a - ref).abs().max() / (ref.abs().max() + 1e-12))
            assert err < 2e-2, (CASES[i], key, err)


if __name__ == "__main__":
    torch.save(_run_cases(_ext()), sys.argv[1])
