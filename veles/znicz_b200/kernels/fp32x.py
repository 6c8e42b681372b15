"""fp32 layers on the wgmma tensor cores ("split-bf16", SURVEY §6 config 2).

``compute_type: "fp32"`` keeps activations, errors and weights in fp32 - the reference's only
precision (/root/reference/all2all.py:262-275 calls SGEMM, conv.py:330-352 its fp32 im2col GEMM).
The tensor cores have no fp32 operand type, so each fp32 operand is written as
``hi + lo`` (two bf16 numbers = 16 mantissa bits, kernels/csrc/split.cu) and the product

    x . w  ~=  hi.hi + hi.lo + lo.hi (+ lo.lo)

is evaluated by ONE bf16 wgmma GEMM / implicit-GEMM convolution whose reduction dimension holds
the parts side by side; the fp32 accumulator sums the partial products. The same kernels as
the bf16 path run (gemm_umma.cu: TMA, tap-mode im2col gather, split-K), on 3-4x the reduction
length - still several times faster than the SIMT fp32 kernels, at ~1e-5 relative error per
product instead of bf16's 4e-3.

Layouts (A side pattern 0 = [hi|hi|lo|lo], B side pattern 1 = [hi|lo|hi|lo]):

* FC fprop:   x  -> [batch][3 K8]           w -> [n_out][3 K8]          (parts along K)
* FC dgrad:   err-> [batch][3 N8]           w -> [3 N8][n_in8]          (parts along n_out)
* FC wgrad:   x  -> [3 batch][n_in8]        err->[3 batch][n_out8]      (parts along the batch)
* conv fprop: x  -> NHW[4 Cp]               w -> [F][tap][4 Cp]         (4 parts keep the tap-mode
  gather's power-of-two / multiple-of-64 channel counts; the 4th carries lo.lo)
* conv dgrad: err-> NHW[4 Fp]               w -> [tap][4 Fp][C8]
* conv wgrad: x  -> [3 N]HW[Cw]             err->[3 N]HW[F8]            (parts along the images)

Switch: ``root.common.engine.fp32_tensor_cores`` (default True) or ``ZNICZ_FP32_TC=0``;
off = SIMT fp32 kernels.
"""
import os

import torch

from ..core.config import root

counters = {"gemms": 0, "splits": 0}


def enabled(unit):
    from ..ops.nn_units import compute_dtype_name
    return (compute_dtype_name() == "fp32" and
            bool(root.common.engine.get("fp32_tensor_cores", True)) and
            os.environ.get("ZNICZ_FP32_TC", "1") != "0" and
            not getattr(unit, "weights_transposed", False))


def _r(n, a):
    return (n + a - 1) // a * a


def _tmp(unit, name, shape, zero=False):
    key = "tmp_x3_%s_" % name
    t = unit.__dict__.get(key)
    if t is None or tuple(t.shape) != tuple(shape):
        t = (torch.zeros if zero else torch.empty)(shape, dtype=torch.bfloat16,
                                                   device=unit.device.torch_device)
        unit.__dict__[key] = t
    return t


def _cpad4(c):
    """Per-part channel count such that 4 parts per pixel suit the tap-mode gather
    (32 / 64 channels per tap, or a multiple of 64)."""
    if c <= 8:
        return 8
    return _r(c, 16)


def _wgrad_cpad(c):
    from .api import _fprop_cpad
    return _fprop_cpad(c) or c


def _from_forward(gd_unit, which, shape):
    """Row-stacked operand the forward unit produced beside its own split this step (None = it
    did not; the request flag makes it do so from the next step on)."""
    fwd = gd_unit.forward_unit
    if fwd is None:
        return None
    fwd.__dict__["x3_train_"] = True
    ready = fwd.__dict__.get("x3_ready_")
    if not ready or ready[which] is None or tuple(ready[which].shape) != tuple(shape):
        return None
    return ready[which]


def _f32(*tensors):
    return all(t.dtype == torch.float32 and t.is_contiguous() for t in tensors)


def _count_split():
    from .api import counters as api_counters
    counters["splits"] += 1
    api_counters["launches"] += 1


def _split(ext, src, rows, length, a, da, b=None, db=()):
    ext.split_parts(src, rows, length, a, list(da), b, list(db))
    _count_split()


# ------------------------------------------------------------------------------------------
# fully connected
# ------------------------------------------------------------------------------------------
def fc_forward(unit, ext, x, out, bias, act, batch, n_in, n_out):
    """out[batch][n_out] = act(x . W^T + bias). True when the tensor cores took it."""
    w = unit.weights.dev
    if not _f32(x, w, out) or n_in < 32:
        return False
    k8 = _r(n_in, 8)
    x3 = _tmp(unit, "fc_x", (batch, 3 * k8))
    w3 = _tmp(unit, "fc_w", (n_out, 3 * k8))
    xs = ws = None
    dxs = dws = ()
    if unit.__dict__.get("x3_train_"):
        # a GD unit consumed this layer last step: its row-stacked operands (wgrad's x, dgrad's
        # W) come out of the same two launches
        n8 = _r(n_out, 8)
        xs = _tmp(unit, "fc_xs", (3 * batch, k8))
        ws = _tmp(unit, "fc_ws", (3 * n8, k8), zero=True)  # rows n_out..n8 of a part stay zero
        dxs = (k8, batch * k8, k8, 3, 1)
        dws = (k8, n8 * k8, k8, 3, 1)
    _split(ext, x, batch, n_in, x3, (3 * k8, k8, k8, 3, 0), xs, dxs)
    _split(ext, w, n_out, n_in, w3, (3 * k8, k8, k8, 3, 1), ws, dws)
    unit.__dict__["x3_ready_"] = (xs, ws)
    r = ext.gemm(x3, 3 * k8, False, w3, 3 * k8, True, out, n_out, False,
                 batch, n_out, 3 * k8, bias, act, 1.0, 0.0, 1, 0, 1)
    if r != 0:
        return False
    counters["gemms"] += 1
    return True


def fc_split_err(unit, ext, err, batch, n_out, want_concat, want_stack):
    """err_output -> (concatenated [batch][3 N8], stacked [3 batch][N8]) in one launch."""
    n8 = _r(n_out, 8)
    ec = _tmp(unit, "fc_ec", (batch, 3 * n8)) if want_concat else None
    es = _tmp(unit, "fc_es", (3 * batch, n8)) if want_stack else None
    dc = (3 * n8, n8, n8, 3, 0)
    ds = (n8, batch * n8, n8, 3, 0)
    if ec is not None:
        _split(ext, err, batch, n_out, ec, dc, es, ds if es is not None else ())
    elif es is not None:
        _split(ext, err, batch, n_out, es, ds)
    return ec, es


def fc_dgrad(unit, ext, ec, ei, batch, n_in, n_out, alpha, beta):
    """err_input = alpha * err . W + beta * err_input from the concatenated err parts."""
    w = unit.weights.dev
    n8 = _r(n_out, 8)
    i8 = _r(n_in, 8)
    ws = _from_forward(unit, 1, (3 * n8, i8))
    if ws is None:
        ws = _tmp(unit, "fc_ws", (3 * n8, i8), zero=True)  # rows n_out..n8 of a part stay zero
        _split(ext, w, n_out, n_in, ws, (i8, n8 * i8, i8, 3, 1))
    r = ext.gemm(ec, 3 * n8, False, ws, i8, False, ei, n_in, False,
                 batch, n_in, 3 * n8, None, 0, float(alpha), float(beta), 1, 0, 1)
    if r != 0:
        return False
    counters["gemms"] += 1
    return True


def fc_wgrad(unit, ext, x, es, gbuf, batch, n_in, n_out):
    """gradW[n_out][n_in] = err^T . x with the parts stacked along the batch."""
    i8 = _r(n_in, 8)
    n8 = _r(n_out, 8)
    xs = _from_forward(unit, 0, (3 * batch, i8))
    if xs is None:
        xs = _tmp(unit, "fc_xs", (3 * batch, i8))
        _split(ext, x, batch, n_in, xs, (i8, batch * i8, i8, 3, 1))
    r = ext.gemm(xs, i8, True, es, n8, False, gbuf, n_in, True,
                 n_in, n_out, 3 * batch, None, 0, 1.0, 0.0, 1, 0, 1)
    if r != 0:
        return False
    counters["gemms"] += 1
    return True


# ------------------------------------------------------------------------------------------
# convolution
# ------------------------------------------------------------------------------------------
def conv_forward(unit, ext, x, out, bias, g, act):
    w = unit.weights.dev
    if not _f32(x, w, out):
        return False
    n, h, wd, c = g[0], g[1], g[2], g[3]
    f, taps = g[6], g[7] * g[8]
    cp = _cpad4(c)
    x4 = _tmp(unit, "cv_x", (n, h, wd, 4 * cp))
    w4 = _tmp(unit, "cv_w", (f, taps * 4 * cp))
    xs = None
    dxs = ()
    if unit.__dict__.get("x3_train_"):
        cw = _wgrad_cpad(c)
        xs = _tmp(unit, "cv_xs", (3 * n, h, wd, cw))
        dxs = (cw, n * h * wd * cw, cw, 3, 1)
    _split(ext, x, n * h * wd, c, x4, (4 * cp, cp, cp, 4, 0), xs, dxs)
    unit.__dict__["x3_ready_"] = (xs, None)
    _split(ext, w, f * taps, c, w4, (4 * cp, cp, cp, 4, 1))
    g4 = list(g)
    g4[3] = 4 * cp
    r = ext.conv_fprop(x4, w4, taps * 4 * cp, False, bias, out, g4, act, 1)
    if r != 0:
        return False
    counters["gemms"] += 1
    return True


def conv_split_err(unit, ext, err, g, pixels, want_concat, want_stack):
    f = g[6]
    fp = _cpad4(f)
    f8 = _r(f, 8)
    ec = _tmp(unit, "cv_ec", (pixels, 4 * fp)) if want_concat else None
    es = _tmp(unit, "cv_es", (3 * pixels, f8)) if want_stack else None
    dc = (4 * fp, fp, fp, 4, 0)
    ds = (f8, pixels * f8, f8, 3, 0)
    if ec is not None:
        _split(ext, err, pixels, f, ec, dc, es, ds if es is not None else ())
    elif es is not None:
        _split(ext, err, pixels, f, es, ds)
    return ec, es


def conv_dgrad(unit, ext, ec, ei, g, alpha, beta):
    fwd_w = unit.weights.dev
    c, f, taps = g[3], g[6], g[7] * g[8]
    fp = _cpad4(f)
    c8 = _r(c, 8)
    wt = _tmp(unit, "cv_wt", (taps * 4 * fp, c8))
    ext.split_conv_wt(fwd_w, wt, f, taps, c, fp, c8, 4, 1)
    _count_split()
    g4 = list(g)
    g4[6] = 4 * fp
    r = ext.conv_dgrad(ec, wt, c8, False, ei, g4, float(alpha), float(beta), 1, None, 0)
    if r != 0:
        return False
    counters["gemms"] += 1
    return True


def conv_wgrad_prepare(unit, ext, x, g, pixels):
    """(stacked input, geometry, kw, channel padding, split count) of the wgrad launch."""
    n, h, wd, c = g[0], g[1], g[2], g[3]
    f, taps = g[6], g[7] * g[8]
    cw = _wgrad_cpad(c)
    f8 = _r(f, 8)
    xs = _from_forward(unit, 0, (3 * n, h, wd, cw))
    if xs is None:
        xs = _tmp(unit, "cv_xs", (3 * n, h, wd, cw))
        _split(ext, x, n * h * wd, c, xs, (cw, n * h * wd * cw, cw, 3, 1))
    g3 = list(g)
    g3[0], g3[3], g3[6] = 3 * n, cw, f8
    kw = taps * cw
    return xs, g3, kw, (cw if cw != c else 0), f8
