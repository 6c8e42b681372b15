"""Numerics + throughput of the persistent warp-specialised wgmma GEMM (csrc/gemm_pair.cu) against the
single-CTA kernel (gemm_umma.cu) and cuBLAS (torch.matmul), same process, CUDA events, L2 flushed
between timed launches. usage: python tests/bench_gemm_pair.py [check|bench]"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from veles.znicz_b200.kernels import load_extension  # noqa: E402

ext = load_extension(required=True)
dev = torch.device("cuda:0")


def check():
    torch.manual_seed(1)
    out = []
    for (m, n, k, f32, act, bias) in [(256, 256, 64, False, 0, False), (512, 256, 128, True, 0, True),
                                      (1024, 1024, 512, False, 3, True), (768, 384, 200, False, 0, False),
                                      (300, 130, 72, True, 0, True), (2048, 4096, 1024, False, 0, False),
                                      (8192, 8192, 256, False, 0, False)]:
        a = torch.randn(m, k, device=dev).bfloat16()
        b = torch.randn(n, k, device=dev).bfloat16()
        bs = torch.randn(n, device=dev) if bias else None
        o = torch.full((m * 2, n), float("nan"), device=dev,
                       dtype=torch.float32 if f32 else torch.bfloat16)       # 2x-NaN OOB guard
        r = ext.gemm_pair(a, b, o[:m], bs, act, 0.5)
        torch.cuda.synchronize()
        ref = 0.5 * (a.float() @ b.float().t())
        if bias:
            ref = ref + bs
        if act == 3:
            ref = torch.relu(ref)
        got = o[:m].float()
        err = (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-6)
        l2 = ((got - ref).norm() / ref.norm()).item()
        guard = bool(torch.isnan(o[m:]).all())
        out.append({"shape": [m, n, k], "f32": f32, "rc": int(r), "max_rel": err, "rel_l2": l2,
                    "guard_ok": guard})
        print(out[-1], flush=True)
    return out


def timeit(fn, iters=20):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def bench():
    res = []
    for (m, n, k) in [(8192, 8192, 8192), (4096, 4096, 4096), (16384, 4096, 4096), (2048, 9216, 4096)]:
        a = torch.randn(m, k, device=dev).bfloat16()
        b = torch.randn(n, k, device=dev).bfloat16()
        o = torch.empty(m, n, device=dev, dtype=torch.bfloat16)
        fl = 2.0 * m * n * k
        row = {"shape": [m, n, k]}
        for name, fn in (("pair", lambda: ext.gemm_pair(a, b, o, None, 0, 1.0)),
                         ("single_cta", lambda: ext.gemm(a, k, False, b, k, True, o, n, False, m, n, k,
                                                         None, 0, 1.0, 0.0, 1, 0, 1)),
                         ("cublas", lambda: torch.matmul(a, b.t(), out=o))):
            med, best = timeit(fn)
            row[name + "_ms"] = round(med, 4)
            row[name + "_tflops"] = round(fl / med / 1e9, 1)
            row[name + "_best_tflops"] = round(fl / best / 1e9, 1)
        row["pair_vs_cublas"] = round(row["pair_tflops"] / row["cublas_tflops"], 3)
        res.append(row)
        print(json.dumps(row), flush=True)
    return res


if __name__ == "__main__":
    mode = sys.argv[1] if len(sys.argv) > 1 else "check"
    if mode in ("check", "all"):
        check()
    if mode in ("bench", "all"):
        bench()
