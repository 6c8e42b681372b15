"""Micro-benchmark of the five small-channel conv calls of the CIFAR and MNIST conv nets that run
on the halo kernels: CIFAR conv1-3 fprop and conv2 dgrad at batch 100, MNIST conv1 fprop at batch 6
(bench.py's batches). Each call is timed with CUDA events, once with the L2 flushed (a 256 MB
write) before every launch and once hot (back-to-back launches). Beside each time it prints the
least time the data sheet allows (the larger of activation bytes over 3.35 TB/s HBM and the MMA
that conv_halo_persist_k issues over 989 TFLOP/s dense BF16, H100 SXM, 700 W) and that bound as a
fraction of the time.

Run on an H100, once per kernel choice (the switch is read once per process):
    python tools/bench_conv_halo.py
    ZNICZ_CONV_HALO_PERSIST=0 python tools/bench_conv_halo.py      # one-tile-per-CTA halo kernel
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from step_profile import card  # noqa: E402
from veles.znicz_b200.kernels import load_extension  # noqa: E402

HBM_BPS = 3.35e12
BF16_FLOPS = 989e12
# name, kind, N, H, W, C, F, k, pad      (stride 1; dgrad: C = err_input channels, F = err_output's)
CALLS = [("cifar conv1 fprop", "fprop", 100, 32, 32, 8, 32, 5, 2),
         ("cifar conv2 fprop", "fprop", 100, 16, 16, 32, 32, 5, 2),
         ("cifar conv3 fprop", "fprop", 100, 8, 8, 32, 64, 5, 2),
         ("cifar conv2 dgrad", "dgrad", 100, 16, 16, 32, 32, 5, 2),
         ("mnist conv1 fprop", "fprop", 6, 28, 28, 8, 64, 5, 0)]


def bounds(kind, n, h, w, c, f, k, pad):
    """Activation bytes (bf16 in + out), the MMA FLOPs of every k16 step issued over the 8x8 pixel
    blocks, and the data-sheet time bound in us."""
    oh, ow = h + 2 * pad - k + 1, w + 2 * pad - k + 1
    inner, cols, ph, pw = (c, f, oh, ow) if kind == "fprop" else (f, c, h, w)
    kpad = -(-(k * k * inner) // 64) * 64
    rows = n * -(-ph // 8) * -(-pw // 8) * 64
    byts = 2 * (n * h * w * c + n * oh * ow * f)
    flops = 2.0 * rows * max(cols, 16) * kpad
    return byts, flops, max(byts / HBM_BPS, flops / BF16_FLOPS) * 1e6


def timeit(fn, flush, iters=200):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    if flush is None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters * 1000.0
    tot = 0.0
    for _ in range(iters):
        flush.fill_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters * 1000.0


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv_halo.py needs a GPU")
    ext = load_extension(required=True)
    dev = "cuda"
    flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    print("card: %s" % card())
    print("ZNICZ_CONV_HALO=%s ZNICZ_CONV_HALO_PERSIST=%s" % (
        os.environ.get("ZNICZ_CONV_HALO", "1"), os.environ.get("ZNICZ_CONV_HALO_PERSIST", "1")))
    print("| call | L2 flushed us | hot us | MB | MMA GFLOP | bound us | bound / flushed | bound / hot |")
    print("|---|---|---|---|---|---|---|---|")
    for name, kind, n, h, w, c, f, k, pad in CALLS:
        oh, ow = h + 2 * pad - k + 1, w + 2 * pad - k + 1
        g = [n, h, w, c, oh, ow, f, k, k, 1, 1, pad, pad]
        if kind == "fprop":
            kw = k * k * c
            x = torch.randn(n, h, w, c, device=dev, generator=gen).bfloat16()
            wl = (torch.randn(f, kw, device=dev, generator=gen) / kw ** 0.5).bfloat16()
            bias = torch.randn(f, device=dev, generator=gen)
            out = torch.empty(n, oh, ow, f, device=dev, dtype=torch.bfloat16)
            fn = lambda: ext.conv_fprop(x, wl, kw, False, bias, out, g, 3, 1)  # noqa: E731
        else:
            eo = torch.randn(n, oh, ow, f, device=dev, generator=gen).bfloat16()
            wd = (torch.randn(k * k * f, c, device=dev, generator=gen) / (k * k * f) ** 0.5).bfloat16()
            ei = torch.empty(n, h, w, c, device=dev, dtype=torch.bfloat16)
            fn = lambda: ext.conv_dgrad(eo, wd, c, False, ei, g, 1.0, 0.0, 1, None, 0)  # noqa: E731
        byts, flops, bound = bounds(kind, n, h, w, c, f, k, pad)
        t_cold, t_hot = timeit(fn, flush), timeit(fn, None)
        print("| %s | %.2f | %.2f | %.2f | %.3f | %.2f | %.1f %% | %.1f %% |" % (
            name, t_cold, t_hot, byts / 1e6, flops / 1e9, bound, 100 * bound / t_cold,
            100 * bound / t_hot))
    return 0


if __name__ == "__main__":
    sys.exit(main())
