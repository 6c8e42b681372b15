"""bf16 vs fp8 (e4m3) wgmma GEMM on FC-shaped problems (CUDA events, L2 flushed between
launches). Run on an H100:  python tests/bench_fp8_micro.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from veles.znicz_b200.kernels import load_extension  # noqa: E402

ext = load_extension(required=True)
dev = "cuda"
flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
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


for M, N, K in ((128, 4096, 9216), (4096, 4096, 4096), (8192, 8192, 8192)):
    a = torch.randn(M, K, device=dev)
    b = torch.randn(N, K, device=dev) / K ** 0.5
    ab, bb = a.bfloat16(), b.bfloat16()
    qa = (a * 100).to(torch.float8_e4m3fn).view(torch.uint8)
    qb = (b * 100).to(torch.float8_e4m3fn).view(torch.uint8)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    t16 = timeit(lambda: ext.gemm(ab, K, False, bb, K, True, out, N, False, M, N, K, None, 0, 1.0, 0.0,
                                  1, 0, 1))
    t8 = timeit(lambda: ext.gemm_fp8(qa, qb, out, None, 0, 1e-4))
    fl = 2.0 * M * N * K
    print("M=%d N=%d K=%d  bf16 %.1f us (%.0f TFLOP/s)   fp8 %.1f us (%.0f TFLOP/s)   x%.2f" % (
        M, N, K, t16, fl / t16 / 1e6, t8, fl / t8 / 1e6, t16 / t8))
