"""Block-scaled fp8 (MX format: e4m3 elements, one UE8M0 power-of-two scale per 32 consecutive
elements of the reduction dimension) - the numerics reference of north-star config 4.

Block-scaled tensor-core MMAs multiply e4m3 operands whose 32-element K-blocks carry an 8-bit
exponent scale each; the H100 has no such instruction (its e4m3 GEMM here uses one per-tensor
scale) and this tree builds no device path for the format. This module is its host-side oracle
and an EMULATION switch for the numpy backend:

* ``quantize`` / ``dequantize`` / ``fake_quant`` implement the format exactly (round-to-nearest-even
  to e4m3 via torch's float8 type, saturation at +-448, scale = 2^ceil(log2(amax / 448)));
* ``matmul`` is the product a block-scaled tensor-core GEMM would return (fp32 accumulation of the
  de-quantised operands);
* with ``root.common.engine.fp8_emulation = True`` the numpy paths of the fully connected layers
  (forward, err_input, weight gradient) pass their GEMM operands through ``fake_quant`` along the
  reduction dimension of each product, so the effect of block-scaled fp8 on convergence can be
  measured on the CPU before any kernel exists (``tests/test_mxfp8.py``).
"""
from __future__ import annotations

import numpy

from ..core.config import root

BLOCK = 32
E4M3_MAX = 448.0


def _e4m3(x):
    """fp32 array -> the nearest e4m3 values (as fp32), saturating."""
    import torch
    t = torch.from_numpy(numpy.ascontiguousarray(numpy.clip(x, -E4M3_MAX, E4M3_MAX), dtype=numpy.float32))
    return t.to(torch.float8_e4m3fn).to(torch.float32).numpy()


def quantize(x, axis=-1, block=BLOCK):
    """-> (q, e): ``q`` e4m3 values (stored as fp32, same shape as ``x`` with ``axis`` padded to a
    multiple of ``block``), ``e`` int8 exponents of the per-block scales (shape: blocks along
    ``axis``). x ~= q * 2^e per block."""
    x = numpy.moveaxis(numpy.asarray(x, dtype=numpy.float32), axis, -1)
    n = x.shape[-1]
    pad = (-n) % block
    if pad:
        x = numpy.concatenate([x, numpy.zeros(x.shape[:-1] + (pad,), numpy.float32)], axis=-1)
    xb = x.reshape(x.shape[:-1] + (-1, block))
    amax = numpy.abs(xb).max(axis=-1)
    with numpy.errstate(divide="ignore"):
        e = numpy.where(amax > 0, numpy.ceil(numpy.log2(amax / E4M3_MAX)), -127.0)
    e = numpy.clip(e, -127, 127).astype(numpy.int8)
    scale = numpy.exp2(e.astype(numpy.float32))[..., None]
    q = _e4m3(xb / scale)
    return q.reshape(x.shape), e, n


def dequantize(q, e, n, axis=-1, block=BLOCK):
    qb = q.reshape(q.shape[:-1] + (-1, block))
    x = (qb * numpy.exp2(e.astype(numpy.float32))[..., None]).reshape(q.shape)[..., :n]
    return numpy.moveaxis(x, -1, axis)


def fake_quant(x, axis=-1, block=BLOCK):
    """x -> the values a block-scaled e4m3 operand would carry (same shape, fp32)."""
    q, e, n = quantize(x, axis, block)
    return dequantize(q, e, n, axis, block)


def matmul(a, b):
    """a [M, K] . b [K, N] as a block-scaled fp8 tensor-core GEMM would compute it."""
    return fake_quant(a, axis=1).astype(numpy.float32).dot(fake_quant(b, axis=0).astype(numpy.float32))


def enabled():
    return bool(root.common.engine.get("fp8_emulation", False))


def operand(x, axis):
    """GEMM operand hook of the numpy layer paths: identity unless the emulation is switched on."""
    if not enabled():
        return x
    return fake_quant(x, axis).astype(x.dtype, copy=False)
