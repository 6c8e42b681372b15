"""H2D copy timing from pinned memory (CUDA events), alone and queued behind a kernel.
Run on an H100:  python tests/bench_h2d_micro.py"""
import torch

dev = "cuda"
for nbytes in (4096, 615 * 1024, 1230 * 1024, 16 << 20):
    pin = torch.zeros(nbytes, dtype=torch.uint8).pin_memory()
    dst = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    for _ in range(5):
        dst.copy_(pin, non_blocking=True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 50
    e0.record()
    for _ in range(n):
        dst.copy_(pin, non_blocking=True)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / n
    print("H2D %8d B: %.1f us/copy  %.2f GB/s" % (nbytes, us, nbytes / us / 1e3))
a = torch.randn(4096, 4096, device=dev)
pin = torch.zeros(615 * 1024, dtype=torch.uint8).pin_memory()
dst = torch.zeros(615 * 1024, dtype=torch.uint8, device=dev)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(50):
    dst.copy_(pin, non_blocking=True)
    b = a * 2.0
e1.record()
torch.cuda.synchronize()
print("copy + 64 MB elementwise kernel interleaved: %.1f us/iter" % (e0.elapsed_time(e1) * 1e3 / 50))
e0.record()
for _ in range(50):
    b = a * 2.0
e1.record()
torch.cuda.synchronize()
print("kernel alone: %.1f us/iter" % (e0.elapsed_time(e1) * 1e3 / 50))

import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from veles.znicz_b200.kernels import load_extension  # noqa: E402
ext = load_extension(required=True)
for nbytes in (4096, 615 * 1024, 1230 * 1024):
    pin = torch.arange(nbytes, dtype=torch.int64).to(torch.uint8).pin_memory()
    dst = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    ext.pull_from_host(pin, dst)
    torch.cuda.synchronize()
    assert torch.equal(dst.cpu(), pin)
    e0.record()
    for _ in range(50):
        ext.pull_from_host(pin, dst)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / 50
    print("pull %8d B: %.1f us/launch  %.2f GB/s" % (nbytes, us, nbytes / us / 1e3))
pin = torch.zeros(615 * 1024, dtype=torch.uint8).pin_memory()
dst = torch.zeros(615 * 1024, dtype=torch.uint8, device=dev)
e0.record()
for _ in range(50):
    ext.pull_from_host(pin, dst)
    b = a * 2.0
e1.record()
torch.cuda.synchronize()
print("pull + 64 MB elementwise kernel interleaved: %.1f us/iter" % (e0.elapsed_time(e1) * 1e3 / 50))
