"""Stand-alone first-contact check of the wgmma kernels (run under `timeout`):
prints per-configuration max relative error so a descriptor mistake is visible at once."""
import sys
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from veles.znicz_b200.kernels import load_extension

ext = load_extension()
dev = "cuda"
torch.manual_seed(0)


def rel(a, b):
    return float((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-12))


def run(name, fn):
    try:
        v = fn()
        torch.cuda.synchronize()
        print("%-40s %s" % (name, v), flush=True)
    except Exception as e:  # noqa
        print("%-40s EXC %s" % (name, e), flush=True)


def nt(M, N, K):
    a = torch.randn(M, K, device=dev).bfloat16()
    b = torch.randn(N, K, device=dev).bfloat16()
    out = torch.zeros(M, N, device=dev)
    r = ext.gemm(a, K, False, b, K, True, out, N, False, M, N, K, None, 0, 1.0, 0.0, 1, 0, 1)
    torch.cuda.synchronize()
    return "rc=%d rel=%.2e" % (r, rel(out, a.float() @ b.float().t()))


def nn(M, N, K):
    a = torch.randn(M, K, device=dev).bfloat16()
    b = torch.randn(K, N, device=dev).bfloat16()
    out = torch.zeros(M, N, device=dev)
    r = ext.gemm(a, K, False, b, N, False, out, N, False, M, N, K, None, 0, 1.0, 0.0, 1, 0, 1)
    torch.cuda.synchronize()
    return "rc=%d rel=%.2e" % (r, rel(out, a.float() @ b.float()))


def tn(M, N, K):
    a = torch.randn(K, M, device=dev).bfloat16()
    b = torch.randn(K, N, device=dev).bfloat16()
    out = torch.zeros(M, N, device=dev)
    r = ext.gemm(a, M, True, b, N, False, out, N, False, M, N, K, None, 0, 1.0, 0.0, 1, 0, 1)
    torch.cuda.synchronize()
    return "rc=%d rel=%.2e" % (r, rel(out, a.float().t() @ b.float()))


def tt(M, N, K):
    a = torch.randn(K, M, device=dev).bfloat16()
    b = torch.randn(N, K, device=dev).bfloat16()
    out = torch.zeros(M, N, device=dev)
    r = ext.gemm(a, M, True, b, K, True, out, N, False, M, N, K, None, 0, 1.0, 0.0, 1, 0, 1)
    torch.cuda.synchronize()
    return "rc=%d rel=%.2e" % (r, rel(out, a.float().t() @ b.float().t()))


for shp in [(128, 128, 64), (128, 64, 64), (128, 16, 64), (128, 32, 128), (256, 128, 256),
            (100, 10, 1024), (300, 200, 520)]:
    run("NT %s" % (shp,), lambda: nt(*shp))
for shp in [(128, 128, 64), (128, 64, 128), (100, 1024, 16), (130, 200, 72)]:
    run("NN %s" % (shp,), lambda: nn(*shp))
for shp in [(128, 128, 64), (64, 1024, 100), (32, 800, 2560)]:
    run("TN %s" % (shp,), lambda: tn(*shp))
run("TT (128,128,64)", lambda: tt(128, 128, 64))
print("done", flush=True)
