"""Workload for `ncu --set full`: one 8192^3 bf16 GEMM on the persistent kernel, one AlexNet conv2
fprop / wgrad on the same kernel with the TMA im2col operand (a few launches each)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from veles.znicz_b200.kernels import load_extension  # noqa: E402

ext = load_extension(required=True)
dev = "cuda"
torch.manual_seed(0)
a = torch.randn(8192, 8192, device=dev).bfloat16()
b = torch.randn(8192, 8192, device=dev).bfloat16()
o = torch.empty(8192, 8192, device=dev, dtype=torch.bfloat16)
for _ in range(3):
    ext.gemm_pair(a, b, o, None, 0, 1.0)
n, h, w, c, f, k, pad = 128, 27, 27, 128, 256, 5, 2
g = [n, h, w, c, h, w, f, k, k, 1, 1, pad, pad]
kw = k * k * c
x = torch.randn(n, h, w, c, device=dev).bfloat16()
wl = torch.randn(f, kw, device=dev).bfloat16()
out = torch.empty(n, h, w, f, device=dev, dtype=torch.bfloat16)
eo = torch.randn(n, h, w, f, device=dev).bfloat16()
splits = int(ext.pick_splits(kw, f, n * h * w, 64))
parts = torch.empty(splits, f, kw, device=dev)
for _ in range(3):
    ext.conv_fprop(x, wl, kw, False, None, out, g, 3, 1)
    ext.conv_wgrad(eo, x, parts, splits, g, False, 1, None)
torch.cuda.synchronize()
print("done")
