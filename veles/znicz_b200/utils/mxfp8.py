"""Block-scaled fp8 numerics: the MX format and the 128-element block scheme of the device's fp8
fully connected layers (compute_type "fp8") - the numerics reference of north-star config 4.

MX (e4m3 elements, one UE8M0 power-of-two scale per 32 consecutive elements of the reduction
dimension) needs block-scaled tensor-core MMAs the H100 does not have; it exists here only as a
CPU emulation. The device scheme ("block128") is what ``csrc/fp8.cu`` and the fp8 mode of
``csrc/gemm_pair.cu`` compute:

* activations and errors: one scale per 1 x 128 block along the reduction dimension of the product
  they feed; weights: one scale per 128 x 128 tile, so W and W^T carry the same quantised values;
* scale 2^e, e the smallest integer with amax <= 448 * 2^e, from the bits of amax
  (``block_exponent``), clamped to [-127, 127]; an all-zero block gets e = -127;
* codes: the e4m3 value of x * 2^-e (exact power-of-two division, round to nearest even,
  saturating): ``quantize_rows`` / ``quantize_tiles`` return the device's codes bit for bit and
  its scales in the device layout [k-block][rows rounded up to 128];
* the GEMM sums the per-k-block products in fp32, so its result is the fp32 product of the
  dequantised operands up to accumulation order.

MX reference:

* ``quantize`` / ``dequantize`` / ``fake_quant`` implement the format exactly (round-to-nearest-even
  to e4m3 via torch's float8 type, saturation at +-448, scale = 2^ceil(log2(amax / 448)));
* ``matmul`` is the product a block-scaled tensor-core GEMM would return (fp32 accumulation of the
  de-quantised operands);
* with ``root.common.engine.fp8_emulation = True`` the numpy paths of the fully connected layers
  (forward, err_input, weight gradient) pass their GEMM operands through ``fake_quant`` along the
  reduction dimension of each product, so the effect of MX fp8 on convergence can be measured on
  the CPU (``tests/test_mxfp8.py``); with ``fp8_emulation = "block128"`` they apply the device
  scheme instead (weights by tiles), the numpy reference of the device's fp8 layers.
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


TILE = 128
BLOCK128 = "block128"


def block_exponent(amax):
    """Smallest integer e with amax <= 448 * 2^e, from the exponent and mantissa bits of the fp32
    ``amax`` (448 = 1.75 * 2^8), clamped to [-127, 127]; zero and subnormal maxima give -127."""
    b = numpy.ascontiguousarray(amax, dtype=numpy.float32).view(numpy.uint32).astype(numpy.int64)
    ef = (b >> 23) & 0xFF
    e = ef - 127 - 8 + ((b & 0x7FFFFF) > 0x600000)
    return numpy.where(ef == 0, -127, numpy.clip(e, -127, 127)).astype(numpy.int32)


def _pow2(e):
    return numpy.ldexp(numpy.float32(1.0), e).astype(numpy.float32)


def _codes(x, e):
    """e4m3 values of x * 2^-e (fp32 product, exact for power-of-two scales)."""
    return _e4m3((x * _pow2(-e)).astype(numpy.float32))


def _pad2(x, rows, cols):
    out = numpy.zeros((rows, cols), numpy.float32)
    out[:x.shape[0], :x.shape[1]] = x
    return out


def quantize_rows(x):
    """x [rows][cols] in 1 x 128 blocks along cols -> (q, s): q [rows][cols] e4m3 values (fp32),
    s [ceil(cols / 128)][round_up(rows, 128)] fp32 scales (padding rows: 2^-127)."""
    x = numpy.asarray(x, dtype=numpy.float32)
    rows, cols = x.shape
    kb, rp = -(-cols // TILE), -(-rows // TILE) * TILE
    xb = _pad2(x, rp, kb * TILE).reshape(rp, kb, TILE)
    e = block_exponent(numpy.abs(xb).max(axis=2))                       # [rp][kb]
    q = _codes(xb, e[..., None]).reshape(rp, kb * TILE)[:rows, :cols]
    return q, numpy.ascontiguousarray(_pow2(e).T)


def quantize_tiles(w):
    """w [rows][cols] in 128 x 128 tiles -> (q, qt, s, st): q [rows][cols] e4m3 values, qt = q^T,
    s [ceil(cols / 128)][round_up(rows, 128)] and st [ceil(rows / 128)][round_up(cols, 128)]: the
    tile scales expanded to the per-row scale layout of each operand form."""
    w = numpy.asarray(w, dtype=numpy.float32)
    rows, cols = w.shape
    kr, kc = -(-rows // TILE), -(-cols // TILE)
    wb = _pad2(w, kr * TILE, kc * TILE).reshape(kr, TILE, kc, TILE)
    e = block_exponent(numpy.abs(wb).max(axis=(1, 3)))                  # [kr][kc]
    q = _codes(wb, e[:, None, :, None]).reshape(kr * TILE, kc * TILE)[:rows, :cols]
    sc = _pow2(e)
    s = numpy.ascontiguousarray(numpy.repeat(sc, TILE, axis=0).T)       # [kc][kr * 128]
    st = numpy.ascontiguousarray(numpy.repeat(sc.T, TILE, axis=0).T)    # [kr][kc * 128]
    return q, numpy.ascontiguousarray(q.T), s, st


def _expand(s, rows, cols):
    """Scales [kb][rows_pad] -> the [rows][cols] array of each element's scale."""
    return numpy.repeat(s.T[:rows], TILE, axis=1)[:, :cols]


def fake_quant_rows(x, axis):
    """2-D x -> the values of its device fp8 codes, 1 x 128 blocks along ``axis``."""
    x = numpy.asarray(x, dtype=numpy.float32)
    x2 = x if axis in (1, -1) else x.T
    q, s = quantize_rows(x2)
    d = q * _expand(s, *x2.shape)
    return d if axis in (1, -1) else d.T


def fake_quant_tiles(w):
    """2-D w -> the values of its device fp8 codes (128 x 128 tiles; symmetric in w and w^T)."""
    q, _, s, _ = quantize_tiles(w)
    return q * _expand(s, *numpy.shape(w))


def matmul(a, b):
    """a [M, K] . b [K, N] as a block-scaled fp8 tensor-core GEMM would compute it."""
    return fake_quant(a, axis=1).astype(numpy.float32).dot(fake_quant(b, axis=0).astype(numpy.float32))


def enabled():
    return bool(root.common.engine.get("fp8_emulation", False))


def operand(x, axis, tile=False):
    """GEMM operand hook of the numpy layer paths: identity unless the emulation is switched on.
    ``tile``: ``x`` is a weight matrix (the "block128" scheme quantises it by 128 x 128 tiles)."""
    mode = root.common.engine.get("fp8_emulation", False)
    if not mode:
        return x
    if mode == BLOCK128:
        q = fake_quant_tiles(x) if tile else fake_quant_rows(x, axis)
        return q.astype(x.dtype, copy=False)
    return fake_quant(x, axis).astype(x.dtype, copy=False)
