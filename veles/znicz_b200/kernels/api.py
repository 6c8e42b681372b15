"""Glue between the unit classes and the sm_90a extension.

Every function takes a unit, pulls the device tensors out of its Arrays
(``.dev`` = read, ``.dev_out`` = about to be overwritten) and launches kernels on the
current CUDA stream. Nothing here synchronises with the host or allocates per call
(temporaries are cached on the unit), so every function is CUDA-graph capturable.

Engine selection is by *shape legality*, not by backend: bf16 activations + TMA-legal
leading dimensions go through the wgmma kernels (``gemm_umma.cu``); everything else
(fp32 compute type, leading dims that are not multiples of 8 elements, transposed weight
storage) runs the exact-fp32 SIMT implicit-GEMM kernels. A wgmma launcher that refuses
a shape raises — there is no silent fallback to PyTorch.
"""
from __future__ import annotations

import contextlib
from typing import NamedTuple, Optional

import numpy
import torch

from ..core.config import root
from ..ops.nn_units import ACT_LINEAR

_MAX_SPLITS = 64
_SMS = {}


def _num_sms():
    """Streaming multiprocessors of the current CUDA device (split-K sizing aims at two CTAs each)."""
    d = torch.cuda.current_device()
    if d not in _SMS:
        _SMS[d] = torch.cuda.get_device_properties(d).multi_processor_count
    return _SMS[d]


counters = {"launches": 0}


from . import fp32x  # noqa: E402


def _ext(unit):
    ext = unit.ext_
    if ext is None:
        raise RuntimeError("%s: the sm_90a extension is not loaded" % unit)
    return ext


def _is_bf16(t):
    return t.dtype == torch.bfloat16


def _tmp(unit, name, shape, dtype, zero=False):
    key = "tmp_%s_" % name
    t = unit.__dict__.get(key)
    if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
        dev = unit.device.torch_device
        t = (torch.zeros if zero else torch.empty)(shape, dtype=dtype, device=dev)
        unit.__dict__[key] = t
    return t


def _roundup(n, a):
    return (n + a - 1) // a * a


def _launch(n=1):
    counters["launches"] += n


paths = {}          # unit name -> kernel families its eager launches used (diagnostics)


def _path(unit, tag):
    paths.setdefault(unit.name, set()).add(tag)


# ------------------------------------------------------------------------------------------
# weights: fp32 master + bf16 shadows in the layouts the tensor-core kernels consume
# ------------------------------------------------------------------------------------------
def lp_enabled(unit):
    from ..ops.nn_units import compute_dtype_name
    return compute_dtype_name() in ("bf16", "fp8") and not unit.weights_transposed


def _shadow_spec(unit):
    """(rows, cols, ld, conv?, taps, C, c_pad) of the weight matrix of a forward unit.
    For conv layers whose channel count is not a multiple of 8 (the first layer, C = 3) the
    fprop shadow is stored channel-padded ``[F][tap][c_pad]`` so the implicit-GEMM gather can
    move 16-byte chunks (see ``lp_cpad``)."""
    rows, cols = unit.weights.shape
    ld = _roundup(cols, 8)
    if hasattr(unit, "kx") and hasattr(unit, "n_kernels"):
        c = unit._n_channels
        taps = unit.kx * unit.ky
        c_pad = _roundup(c, 8)              # dgrad shadow [tap][f][c_pad]
        cp = _fprop_cpad(c)
        if cp:
            ld = taps * cp                  # fprop shadow [f][tap][cp]
        return rows, cols, ld, True, taps, c, c_pad
    return rows, cols, ld, False, 0, 0, 0


def _fprop_cpad(c):
    """Channel count the tap-mode gather wants for a conv input with ``c`` channels (0 = as is).

    A 64-wide reduction block must cover whole filter taps (8 / 16 / 32 / 64 channels per tap) or
    a 64-channel slice of one tap (c % 64 == 0). Other counts - the first layer's 3, AlexNet
    conv2's 96 - would fall back to the per-chunk table gather, 2-3x slower per k-block, so the
    input is channel-padded once per forward instead (96 -> 128: +33 % MMA work, -60 % time)."""
    if c <= 64:
        for v in (8, 16, 32, 64):
            if c <= v:
                return 0 if v == c else v
    r = _roundup(c, 64)
    return 0 if r == c else r


def lp_cpad(unit):
    """Channel padding of the fprop weight shadow / padded input (0 = none)."""
    if hasattr(unit, "kx") and hasattr(unit, "n_kernels"):
        return _fprop_cpad(unit._n_channels)
    return 0


def ensure_shadows(fwd):
    if fwd.weights_lp_ is not None:
        return
    rows, cols, ld, is_conv, taps, c, c_pad = _shadow_spec(fwd)
    dev = fwd.device.torch_device
    fwd.weights_lp_ = torch.zeros((rows, ld), dtype=torch.bfloat16, device=dev)
    if is_conv:
        # dgrad operand [tap][f_pad][c_pad]: f padded to a multiple of 8 (zero rows) so that a
        # channel-padded err_output can use the 16-byte gather when n_kernels % 8 != 0
        fwd.weights_lp_t_ = torch.zeros((taps * _roundup(rows, 8), c_pad), dtype=torch.bfloat16,
                                        device=dev)


def refresh_weight_shadows(fwd):
    """(Re)build the bf16 (and fp8) copies from the fp32 master (init, rollback, snapshot load)."""
    if not fwd.weights or not lp_enabled(fwd):
        return
    ensure_shadows(fwd)
    rows, cols, ld, is_conv, taps, c, c_pad = _shadow_spec(fwd)
    _ext(fwd).refresh_shadows(fwd.weights.dev, rows, cols, fwd.weights_lp_, ld,
                              fwd.weights_lp_t_ if is_conv else None, taps, c, c_pad,
                              lp_cpad(fwd))
    _launch()
    if _fp8_layer(fwd):
        requantize_weights(fwd)


# ------------------------------------------------------------------------------------------
# fp8 (compute_type "fp8"): fully connected products on block-scaled e4m3 operands
# (csrc/fp8.cu quantisers + the fp8 mode of csrc/gemm_pair.cu; numerics: utils/mxfp8.py)
# ------------------------------------------------------------------------------------------
def _fp8_decline(unit, why):
    """Record that an fp8-mode product of this unit runs on the bf16 path instead."""
    _path(unit, "fp8:declined(%s)" % why)
    key = (id(unit), "fp8:" + why)
    if key not in _WARNED:
        _WARNED.add(key)
        unit.warning("fp8 declined (%s): this product uses the bf16 path", why)


def _fp8_layer(fwd):
    """True when the fully connected unit ``fwd`` runs its products in fp8 (a decline is recorded)."""
    from ..ops.nn_units import compute_dtype_name
    if compute_dtype_name() != "fp8" or not fwd.weights:
        return False
    from ..ops.all2all import All2All, All2AllSoftmax
    if not isinstance(fwd, All2All):
        return False                # convolutions (and LSTM cells) stay bf16 under "fp8"
    n_out, n_in = fwd.weights.shape
    if fwd.weights_transposed:
        why = "weights_transposed"
    elif n_out <= FC_SMALL_MAX_OUT:
        why = "fc_small"
    elif n_in % 16:
        why = "n_in % 16"
    elif n_out % (4 if isinstance(fwd, All2AllSoftmax) else 8):
        why = "output row pitch"    # the TMA-store epilogue writes 16-byte aligned rows (bf16;
                                    # the softmax layer's logits are fp32)
    else:
        return True
    _fp8_decline(fwd, why)
    return False


def requantize_weights(fwd):
    """W_q [n_out][n_in16], W_qt [n_in][n_out16] and their expanded tile scales from the fp32
    master: one launch (init, rollback, broadcast and after every weight update)."""
    n_out, n_in = fwd.weights.shape
    dev = fwd.device.torch_device
    q = fwd.__dict__.get("weights_q_")
    if q is None or tuple(q.shape) != (n_out, _roundup(n_in, 16)):
        kb_in, kb_out = -(-n_in // 128), -(-n_out // 128)
        fwd.weights_q_ = torch.empty((n_out, _roundup(n_in, 16)), dtype=torch.uint8, device=dev)
        fwd.weights_qt_ = torch.empty((n_in, _roundup(n_out, 16)), dtype=torch.uint8, device=dev)
        fwd.weights_qs_ = torch.empty((kb_in, kb_out * 128), dtype=torch.float32, device=dev)
        fwd.weights_qts_ = torch.empty((kb_out, kb_in * 128), dtype=torch.float32, device=dev)
    r = _ext(fwd).fp8_quant(fwd.weights.dev, n_out, n_in, 1, fwd.weights_q_, fwd.weights_qs_,
                            fwd.weights_qt_, fwd.weights_qts_)
    if r != 0:
        raise RuntimeError("%s: fp8 weight quantiser refused (code %d)" % (fwd, r))
    _launch()


def _fp8_quant_act(unit, ext, name, t, rows, cols, rows_form, cols_form):
    """bf16 t [rows][cols] -> (q, s) row-block codes and / or (qt, st) transposed codes in
    buffers cached on the unit (None for a form not asked for)."""
    kr, kc = -(-rows // 128), -(-cols // 128)
    q = s = qt = st = None
    if rows_form:
        q = _tmp(unit, name + "_q", (rows, _roundup(cols, 16)), torch.uint8)
        s = _tmp(unit, name + "_s", (kc, kr * 128), torch.float32)
    if cols_form:
        qt = _tmp(unit, name + "_qt", (cols, _roundup(rows, 16)), torch.uint8)
        st = _tmp(unit, name + "_st", (kr, kc * 128), torch.float32)
    r = ext.fp8_quant(t, rows, cols, 0, q, s, qt, st)
    if r != 0:
        raise RuntimeError("%s: fp8 quantiser refused %s (code %d)" % (unit, name, r))
    _launch()
    return q, s, qt, st


def _fp8_gemm(unit, ext, what, a, sa, b, sb, out, m, n, k, bias, act, alpha):
    r = ext.fp8_gemm(a, sa, b, sb, out, m, n, k, bias, act, float(alpha))
    if r != 0:
        raise RuntimeError("%s: fp8 FC %s refused the shape (code %d)" % (unit, what, r))
    _launch()


# ------------------------------------------------------------------------------------------
# fully connected
# ------------------------------------------------------------------------------------------
def fc_forward(unit, softmax=False):
    ext = _ext(unit)
    x = unit.input.dev
    batch = x.shape[0]
    n_in = x.numel() // batch
    n_out = unit.neurons_number
    bias = unit.bias.dev if (unit.include_bias and unit.bias) else None
    if softmax:
        out = _tmp(unit, "logits", (batch, n_out), torch.float32)
    else:
        out = unit.output.dev_out
    use_lp = lp_enabled(unit) and _is_bf16(x) and n_in % 8 == 0
    act = ACT_LINEAR if softmax else eff_act(unit)
    if _fc_small_ok(unit, n_out) and act <= 4:
        # few outputs: one launch does GEMV x n_out + bias + activation (+ softmax + arg-max)
        ev_args = []
        ev = unit.__dict__.get("fused_eval_") if softmax else None
        if ev is not None and getattr(ev, "on_cuda", False) and not ev.testing and \
                ev.output is unit.output and ev.labels and ev.err_output:
            # softmax evaluator folded into this launch (workflow/fusion.py::fuse_evaluator)
            ev.cuda_prepare()
            ev_args = [ev.labels.dev, ev.err_output.dev_out, ev.batch_dev_, ev.n_err.dev,
                       ev.max_err_output_sum.dev]
            if ev.confusion_matrix:
                ev_args.append(ev.confusion_matrix.dev)
                ev.confusion_matrix.dev_written()
            ev.n_err.dev_written()
            ev.max_err_output_sum.dev_written()
            ev.__dict__["fused_done_"] = True
        ext.fc_small_forward(x, unit.weights.dev, bias, unit.output.dev_out,
                             unit.max_idx.dev_out if softmax else None, batch, n_in, n_out,
                             act, bool(softmax), ev_args)
        _launch()
        return
    if use_lp and unit.weights_q_ is not None and _fp8_layer(unit):
        xq, xs, _, _ = _fp8_quant_act(unit, ext, "fp8_x", x, batch, n_in, True, False)
        _fp8_gemm(unit, ext, "forward", xq, xs, unit.weights_q_, unit.weights_qs_, out, batch,
                  n_out, n_in, bias, act, 1.0)
        if softmax:
            ext.softmax_rows(out, unit.output.dev_out, unit.max_idx.dev_out)
            _launch()
        return
    if use_lp:
        ensure_shadows(unit)
        w = unit.weights_lp_
        r = ext.gemm(x, n_in, False, w, w.shape[1], True, out, n_out, False,
                     batch, n_out, n_in, bias, act, 1.0, 0.0, 1, 0, 1)
        if r != 0:
            raise RuntimeError("%s: wgmma FC forward refused the shape (code %d)" % (unit, r))
    elif fp32x.enabled(unit) and fp32x.fc_forward(unit, ext, x, out, bias, act, batch, n_in,
                                                  n_out):
        pass          # fp32 operands as bf16 hi/lo parts on the tensor cores (kernels/fp32x.py)
    else:
        w = unit.weights.dev
        if unit.weights_transposed:   # stored [in][out]
            ext.gemm(x, n_in, False, w, n_out, False, out, n_out, False,
                     batch, n_out, n_in, bias, act, 1.0, 0.0, 1, 0, 0)
        else:
            ext.gemm(x, n_in, False, w, n_in, True, out, n_out, False,
                     batch, n_out, n_in, bias, act, 1.0, 0.0, 1, 0, 0)
    _launch()
    if softmax:
        ext.softmax_rows(out, unit.output.dev_out, unit.max_idx.dev_out)
        _launch()


def fused_act(unit):
    """Activation code folded into this unit by the workflow fusion pass (0 = none)."""
    return int(getattr(unit, "fused_act_", 0) or 0)


def eff_act(unit):
    """The activation a GEMM-like unit applies: its own or the one fused behind it."""
    return fused_act(unit) or unit.ACT


_WARNED = set()


def _warn_once(unit, what, code):
    key = (id(unit), what)
    if key not in _WARNED:
        _WARNED.add(key)
        unit.warning("wgmma %s kernel declined this shape (code %d): using the SIMT kernel",
                     what, code)


FC_SMALL_MAX_OUT = 16


def _fc_small_ok(unit, n_out):
    """Few-output FC layers use the dedicated kernels of csrc/fc_small.cu."""
    return (n_out <= FC_SMALL_MAX_OUT and not unit.weights_transposed and unit.weights and
            unit.weights.dev.dtype == torch.float32)


# -- weight-gradient overlap ---------------------------------------------------------------------
# dgrad and wgrad of a layer both only *read* err_output, and nothing consumes the weight gradient
# before the optimizer step: the wgrad kernels run on the device's side stream (a parallel branch
# of the captured graph) while the main stream carries the err_input chain down the network. The
# small-grid kernels of small nets (50-200 CTAs) then share the SMs instead of queueing.
def _fork_side(unit):
    dev = unit.device
    if not root.common.engine.get("overlap_wgrad", True) or getattr(dev, "side_stream", None) is None:
        return None
    side = dev.side_stream
    side.wait_stream(torch.cuda.current_stream())
    dev.__dict__["side_pending_"] = True
    return side


def join_side(dev):
    """Main stream waits for the outstanding side-stream work (before gradients are consumed)."""
    if dev.__dict__.get("side_pending_"):
        torch.cuda.current_stream().wait_stream(dev.side_stream)
        dev.__dict__["side_pending_"] = False


def _bias_partials(unit, rows, cols):
    ext = _ext(unit)
    slices = ext.colsum_slices(rows)
    return slices, _grad_buffer(unit, "bias_parts", (slices, cols))


def _grad_buffer(unit, name, shape):
    """fp32 gradient staging buffer; lives in symmetric memory when data-parallel."""
    dp = unit.dp_
    if dp is not None and dp.symm is not None and getattr(unit, "step_", None) is None:
        return dp.symm.buffer(unit, name, shape)
    # with the whole-network FusedStep only the locally reduced gradient crosses NVLink (through
    # the step's own symmetric slot), so the split-K partials live in ordinary HBM
    return _tmp(unit, name, shape, torch.float32)


class UpdateDesc(NamedTuple):
    """One parameter update, as both update kernels read it (``ext.cpp::parse_desc``). Buffers
    are the tensors themselves (None: absent); geometry is in elements."""
    w: torch.Tensor                           # fp32 master weights [rows][cols]
    grad: torch.Tensor                        # this rank's split-K partials
    hyper: torch.Tensor                       # GradientDescentBase.HYPER_FIELDS
    nparts: int
    part_stride: int                          # elements between two partials
    flags: int                                # GradientDescentBase.update_flags
    rows: int
    cols: int
    is_bias: int = 0
    lanes: int = 1                            # threads summing one element's partials (a power of 2)
    grad_out: Optional[torch.Tensor] = None   # the reduced gradient (RProp: also the previous one)
    acc: Optional[torch.Tensor] = None
    vel: Optional[torch.Tensor] = None
    col_sums: Optional[torch.Tensor] = None   # ortho regulariser
    s0: Optional[torch.Tensor] = None         # solver state (adagrad / adadelta / fast / RProp)
    s1: Optional[torch.Tensor] = None
    s2: Optional[torch.Tensor] = None
    g_cpad: int = 0                           # > 0: gradient rows are [tap][g_cpad] channel-padded
    lp: Optional[torch.Tensor] = None         # bf16 shadow [rows][ld], rows [tap][lp_cpad] if lp_cpad
    ld: int = 0
    lp_cpad: int = 0
    lp_conv: Optional[torch.Tensor] = None    # conv dgrad shadow [tap][roundup(rows, 8)][c_pad]
    taps: int = 0
    c: int = 0                                # conv input channels
    c_pad: int = 0


def _update(unit, is_bias, grad_buf, nparts, part_stride, rows, cols, g_cpad=0):
    """Fused (cross-GPU reduce +) SGD step for weights or bias of a GD unit."""
    ext = _ext(unit)
    if is_bias:
        w, gout = unit.bias, unit.gradient_bias
        acc, vel = unit.accumulated_gradient_bias, unit.gradient_bias_with_moment
    else:
        w, gout = unit.weights, unit.gradient_weights
        acc, vel = unit.accumulated_gradient_weights, unit.gradient_weights_with_moment
    flags = unit.update_flags(for_bias=is_bias)
    step = unit.step_
    if step is None:
        join_side(unit.device)       # per-tensor update launches right here: gradients must be in
    colsums = None
    if not is_bias and unit.factor_ortho:
        colsums = unit.col_sums.dev_out
        if step is None:
            ext.col_sums(w.dev, colsums, rows, cols, bool(unit.weights_transposed))
            _launch()
    fwd = unit.forward_unit
    if getattr(fwd, "weights_lp_", None) is None and unit.__dict__.get("shadow_owner_"):
        fwd = unit.__dict__["shadow_owner_"]    # GDDeconv: the tied Conv owns the bf16 shadows
    lp = lp_conv = None
    ld = taps = c = c_pad = cpad_lp = 0
    if not is_bias and fwd is not None and getattr(fwd, "weights_lp_", None) is not None:
        r_, c_, ld, is_conv, taps, c, c_pad = _shadow_spec(fwd)
        lp = fwd.weights_lp_
        lp_conv = fwd.weights_lp_t_ if is_conv else None
        cpad_lp = lp_cpad(fwd)
    elif g_cpad:
        if fwd is None or not hasattr(fwd, "kx"):
            raise RuntimeError("channel-padded gradients need the forward conv unit")
        taps, c = fwd.kx * fwd.ky, fwd._n_channels     # fp32x wgrad: no bf16 shadows to refresh
    wdev = w.dev
    if flags & unit.FLAG_RPROP:
        if not gout:
            raise RuntimeError("%s: RProp keeps the previous gradient in gradient_%s" %
                               (unit, "bias" if is_bias else "weights"))
        gout_dev = gout.dev          # read (previous gradient) and rewritten by the kernel
        gout.dev_written()
    else:
        gout_dev = gout.dev_out if gout else None
    # solver state (adagrad / adadelta / fast / RProp): stepped in the same kernel
    states = [a if a is not None and a else None for a in unit.solver_arrays(for_bias=is_bias)]
    for bit, a in ((unit.FLAG_ADAGRAD | unit.FLAG_ADADELTA | unit.FLAG_RPROP, states[0]),
                   (unit.FLAG_ADADELTA, states[1]), (unit.FLAG_FAST, states[2])):
        if (flags & bit) and a is None:
            raise RuntimeError("%s: solver state missing for flags %#x" % (unit, flags))
    s0, s1, s2 = [a.dev if a is not None else None for a in states]
    lanes = 1                        # whole-network kernel: lane groups for small split-K tensors
    if wdev.numel() <= 16384:
        while lanes * 2 <= min(32, nparts):
            lanes *= 2
    desc = UpdateDesc(w=wdev, grad=grad_buf, hyper=unit.hyper_dev_, nparts=int(nparts),
                      part_stride=int(part_stride), flags=int(flags), rows=int(rows),
                      cols=int(cols), is_bias=int(is_bias), lanes=lanes, grad_out=gout_dev,
                      acc=acc.dev if acc else None, vel=vel.dev if vel else None,
                      col_sums=colsums, s0=s0, s1=s1, s2=s2, g_cpad=int(g_cpad), lp=lp,
                      ld=int(ld), lp_cpad=int(cpad_lp), lp_conv=lp_conv, taps=int(taps),
                      c=int(c), c_pad=int(c_pad))
    dp = unit.dp_
    if step is not None:
        step.submit(unit, is_bias, desc)    # deferred: the whole-network step (ops/fused_step.py)
    else:
        if dp is not None and dp.symm is not None:
            ptrs, flag_ptrs, epoch_ptr, blocks = dp.symm.peers(unit, grad_buf)
            ext.fused_update(desc, ptrs, flag_ptrs, epoch_ptr, dp.rank, blocks)
        else:
            ext.fused_update(desc, [], [], 0, 0, 0)
        _launch()
        if not is_bias and getattr(fwd, "weights_q_", None) is not None:
            requantize_weights(fwd)
    w.dev_written()
    if acc:
        acc.dev_written()
    if vel:
        vel.dev_written()
    for a in states:
        if a is not None:
            a.dev_written()
    if dp is not None and dp.symm is None and dp.world_size > 1 and step is None:
        raise RuntimeError("the NCCL baseline mode needs the fused step (engine.fused_step)")


def fc_backward(unit):
    ext = _ext(unit)
    err = unit.err_output.dev
    batch = err.shape[0]
    n_out = err.numel() // batch
    x = unit.input.dev
    n_in = x.numel() // batch
    need_w = unit.need_gradient_weights and unit.weights
    need_b = need_w and unit.include_bias and unit.bias
    if (_fc_small_ok(unit, n_out) and eff_act(unit) <= 4 and err.dtype == x.dtype and
            (eff_act(unit) == ACT_LINEAR or unit.output.dev.dtype == err.dtype)):
        if unit.forward_unit is not None:
            _fp8_layer(unit.forward_unit)      # (records the fc_small decline in fp8 mode)
        # whole GD step of a few-output layer in one launch (+ the deferred update)
        bsplit = max(1, min(16, batch // 8))
        gbuf = _grad_buffer(unit, "wgrad", (bsplit,) + tuple(unit.weights.shape)) \
            if need_w else None
        parts = _grad_buffer(unit, "bias_parts", (bsplit, n_out)) if need_b else None
        ei = None
        if unit.need_err_input:
            ei = unit.err_input.dev if unit.err_input_beta else unit.err_input.dev_out
        ext.fc_small_backward(err, unit.output.dev if eff_act(unit) != ACT_LINEAR else None, x,
                              unit.weights.dev, ei, gbuf, parts, batch, n_in, n_out, eff_act(unit),
                              float(unit.err_input_alpha), float(unit.err_input_beta), bsplit)
        if ei is not None:
            unit.err_input.dev_written()
        _launch()
        if need_w:
            _update(unit, False, gbuf, bsplit, n_out * n_in, n_out, n_in)
        if need_b:
            _update(unit, True, parts, bsplit, n_out, 1, n_out)
        return
    # 1. err_output *= f'(output) fused with the bias-gradient column sums
    if eff_act(unit) != ACT_LINEAR or need_b:
        parts = None
        if need_b:
            slices, parts = _bias_partials(unit, batch, n_out)
        y = unit.output.dev if eff_act(unit) != ACT_LINEAR else None
        if y is not None and y.dtype != err.dtype:
            raise RuntimeError("%s: output/err_output dtype mismatch" % unit)
        ext.err_act_colsum(err, y, batch, n_out, eff_act(unit), parts)
        unit.err_output.dev_written()
        _launch()
    lp_ok = (lp_enabled(unit) and _is_bf16(err) and _is_bf16(x) and
             unit.forward_unit is not None and
             getattr(unit.forward_unit, "weights_lp_", None) is not None)
    fwd = unit.forward_unit
    fp8 = lp_ok and getattr(fwd, "weights_q_", None) is not None and _fp8_layer(fwd)
    fp8_dgrad = fp8 and unit.need_err_input and not unit.err_input_beta
    if fp8 and unit.need_err_input and unit.err_input_beta:
        _fp8_decline(unit, "err_input_beta")
    eq = es8 = eqt = est = None
    if fp8_dgrad or (fp8 and need_w):
        # err (after f' and the bias sums): 1 x 128 blocks along n_out for dgrad, transposed
        # with blocks along the batch for wgrad - one pass over err for both
        eq, es8, eqt, est = _fp8_quant_act(unit, ext, "fp8_err", err, batch, n_out, fp8_dgrad,
                                           fp8 and need_w)
    # the weight-gradient GEMM runs beside the err_input GEMM (see _fork_side)
    x3 = ((not lp_ok) and fp32x.enabled(unit) and fp32x._f32(err, x) and n_in >= 32 and
          n_out >= 32)
    ec = es = None
    if x3:
        ec, es = fp32x.fc_split_err(unit, ext, err, batch, n_out, unit.need_err_input,
                                    bool(need_w))
    side = _fork_side(unit) if (need_w and unit.need_err_input) else None
    # 2. err_input = alpha * err . W + beta * err_input
    if unit.need_err_input:
        ei = unit.err_input.dev if unit.err_input_beta else unit.err_input.dev_out
        if x3 and fp32x.fc_dgrad(unit, ext, ec, ei, batch, n_in, n_out, unit.err_input_alpha,
                                 unit.err_input_beta):
            pass
        elif fp8_dgrad:
            r = ext.fp8_gemm(eq, es8, fwd.weights_qt_, fwd.weights_qts_, ei, batch, n_in, n_out,
                             None, 0, float(unit.err_input_alpha))
            if r != 0:
                raise RuntimeError("%s: fp8 FC dgrad refused the shape (code %d)" % (unit, r))
        elif lp_ok and n_out % 8 == 0:
            w = unit.forward_unit.weights_lp_
            r = ext.gemm(err, n_out, False, w, w.shape[1], False, ei, n_in, False,
                         batch, n_in, n_out, None, 0, float(unit.err_input_alpha),
                         float(unit.err_input_beta), 1, 0, 1)
            if r != 0:
                raise RuntimeError("%s: wgmma FC dgrad refused (code %d)" % (unit, r))
        else:
            _path(unit, "fc_dgrad:simt(lp_ok=%s,err=%s,x=%s,lp=%s)" % (
                lp_ok, err.dtype, x.dtype,
                getattr(unit.forward_unit, "weights_lp_", None) is not None))
            w = unit.weights.dev
            if unit.weights_transposed:  # stored [in][out] => B(k=out, n=in) = w[n][k]
                ext.gemm(err, n_out, False, w, n_out, True, ei, n_in, False, batch, n_in, n_out,
                         None, 0, float(unit.err_input_alpha), float(unit.err_input_beta), 1, 0, 0)
            else:
                ext.gemm(err, n_out, False, w, n_in, False, ei, n_in, False, batch, n_in, n_out,
                         None, 0, float(unit.err_input_alpha), float(unit.err_input_beta), 1, 0, 0)
        unit.err_input.dev_written()
        _launch()
    if not need_w:
        return
    # 3. gradW[out][in] = err^T . x  (reduction over the batch)
    gbuf = _grad_buffer(unit, "wgrad", (1,) + tuple(unit.weights.shape))
    with (torch.cuda.stream(side) if side is not None else contextlib.nullcontext()):
        r = -1
        if fp8:
            _, _, xqt, xst = _fp8_quant_act(unit, ext, "fp8_xt", x, batch, n_in, False, True)
            r = ext.fp8_gemm(eqt, est, xqt, xst, gbuf.view(n_out, n_in), n_out, n_in, batch,
                             None, 0, 1.0)
            if r != 0:
                raise RuntimeError("%s: fp8 FC wgrad refused the shape (code %d)" % (unit, r))
        elif lp_ok and n_out % 8 == 0 and n_in % 8 == 0 and n_out >= 256 and n_in >= 256 \
                and batch >= 64:
            # large layers: err^T . x on the persistent kernel (both operands MN-major,
            # TMA-store epilogue straight into the [neurons][in] gradient layout)
            r = int(ext.fc_wgrad_pair(err.view(batch, n_out), x.view(batch, n_in),
                                       gbuf.view(n_out, n_in)))
        if r == 0:
            pass
        elif x3 and fp32x.fc_wgrad(unit, ext, x, es, gbuf, batch, n_in, n_out):
            pass
        elif lp_ok and n_out % 8 == 0 and n_in % 8 == 0:
            # computed as (x^T . err) with a transposed store: for a fixed output column the 32
            # lanes of a warp then write 32 consecutive floats of gradW[out][in] (one 128-byte
            # store); the direct form wrote 16-byte pieces 36 KB apart and ran FC6's 151 MB
            # gradient at ~200 GB/s
            r = ext.gemm(x, n_in, True, err, n_out, False, gbuf, n_in, True,
                         n_in, n_out, batch, None, 0, 1.0, 0.0, 1, 0, 1)
            if r != 0:
                raise RuntimeError("%s: wgmma FC wgrad refused (code %d)" % (unit, r))
        else:
            _path(unit, "fc_wgrad:simt")
            ext.gemm(err, n_out, True, x, n_in, False, gbuf,
                     n_out if unit.weights_transposed else n_in,
                     bool(unit.weights_transposed), n_out, n_in, batch, None, 0, 1.0, 0.0, 1, 0, 0)
    _launch()
    rows, cols = (n_out, n_in)
    _update(unit, False, gbuf, 1, 0, rows, cols)
    if need_b:
        _update(unit, True, parts, slices, n_out, 1, n_out)


# ------------------------------------------------------------------------------------------
# convolution
# ------------------------------------------------------------------------------------------
def _conv_geom(u):
    return [u._batch_size, u._sy, u._sx, u._n_channels, u._ky_app, u._kx_app, u.n_kernels,
            u.ky, u.kx, u.sliding[1], u.sliding[0], u.padding[1], u.padding[0]]


_S2D_C = 64          # channels per pixel of the space-to-depth tensor (one 128-byte TMA row)


def _s2d_geom(unit, g):
    """Space-to-depth form of a strided convolution over an image-like input (AlexNet conv1:
    11 x 11, stride 4, C = 3), or None. csrc/s2d.cu explains the transform."""
    import os
    n, h, w, c, oh, ow, f, ky, kx, sy, sx, pt, pl = g
    s = sy
    if sy != sx or s < 2 or c * s * s > _S2D_C or ky < s or kx < s or \
            not root.common.engine.get("conv_s2d", True) or os.environ.get("ZNICZ_CONV_S2D", "1") == "0":
        return None
    kyp, kxp = -(-ky // s), -(-kx // s)
    gs = [n, oh + kyp - 1, ow + kxp - 1, _S2D_C, oh, ow, f, kyp, kxp, 1, 1, 0, 0]
    return {"s": s, "kyp": kyp, "kxp": kxp, "g": gs, "kw": kyp * kxp * _S2D_C, "pt": pt, "pl": pl}


def _conv_forward_s2d(unit, ext, x, out, bias, g):
    sd = _s2d_geom(unit, g)
    if sd is None:
        return False
    n, f, ky, kx, c = g[0], g[6], g[7], g[8], g[3]
    gs = sd["g"]
    ensure_shadows(unit)          # the dgrad operand / update kernel keep their usual shadows
    xs = _tmp(unit, "s2d_x", (n, gs[1], gs[2], _S2D_C), torch.bfloat16)
    ws = _tmp(unit, "s2d_w", (f, sd["kw"]), torch.bfloat16)
    ext.space_to_depth(x, xs, sd["s"], sd["pt"], sd["pl"])
    ext.s2d_pack_weights(unit.weights.dev, ws, f, ky, kx, c, sd["s"], sd["kyp"], sd["kxp"], _S2D_C)
    r = ext.conv_fprop(xs, ws, sd["kw"], False, bias, out, gs, eff_act(unit), 1)
    if r != 0:
        unit.__dict__["s2d_"] = None
        return False
    sd["xs"] = xs
    unit.__dict__["s2d_"] = sd
    counters["s2d"] = counters.get("s2d", 0) + 1
    _launch(3)
    return True


def conv_forward(unit):
    ext = _ext(unit)
    x = unit.input.dev
    out = unit.output.dev_out
    bias = unit.bias.dev if (unit.include_bias and unit.bias) else None
    g = _conv_geom(unit)
    if lp_enabled(unit) and _is_bf16(x) and _conv_forward_s2d(unit, ext, x, out, bias, g):
        return
    if lp_enabled(unit) and _is_bf16(x):
        ensure_shadows(unit)
        w = unit.weights_lp_
        cp = lp_cpad(unit)
        if cp:   # first layer: pad C -> 8 once, fprop and wgrad then gather 16-byte chunks
            shape = tuple(x.shape[:3]) + (cp,)
            ready = unit.input.__dict__.get("padded_dev_") if cp == 8 else None
            if ready is not None and tuple(ready.shape) == shape and ready.dtype == x.dtype:
                xp = ready           # the loader's gather kernel already produced it
                unit.__dict__["tmp_xpad_"] = xp
            else:
                if cp == 8:
                    unit.input.__dict__["pad_request_"] = cp
                xp = _tmp(unit, "xpad", shape, x.dtype)
                ext.pad_channels(x, xp, unit._n_channels, cp)
                _launch()
            x = xp
            g = list(g)
            g[3] = cp
        r = ext.conv_fprop(x, w, w.shape[1], False, bias, out, g, eff_act(unit), 1)
        if r in (-3, -4) and not cp:
            _warn_once(unit, "fprop", r)
            w = unit.weights.dev
            ext.conv_fprop(unit.input.dev, w, w.shape[1], bool(unit.weights_transposed), bias,
                           out, _conv_geom(unit), eff_act(unit), 0)
        elif r != 0:
            raise RuntimeError("%s: wgmma conv fprop refused (code %d)" % (unit, r))
    elif fp32x.enabled(unit) and fp32x.conv_forward(unit, ext, x, out, bias, g, eff_act(unit)):
        pass          # (kernels/fp32x.py counts its split launches itself)
    else:
        w = unit.weights.dev
        ld = w.shape[1]
        ext.conv_fprop(x, w, ld, bool(unit.weights_transposed), bias, out, g, eff_act(unit), 0)
    _launch()


def conv_backward(unit):
    ext = _ext(unit)
    err = unit.err_output.dev
    x = unit.input.dev
    g = _conv_geom(unit)
    f = unit.n_kernels
    pixels = err.numel() // f
    kw = unit._kernel_size
    need_w = unit.need_gradient_weights and unit.weights
    need_b = need_w and unit.include_bias and unit.bias
    fwd = unit.forward_unit
    lp_ok = (lp_enabled(unit) and _is_bf16(err) and _is_bf16(x) and fwd is not None and
             getattr(fwd, "weights_lp_t_", None) is not None)
    act = eff_act(unit)
    if unit.__dict__.get("deriv_upstream_"):
        act = ACT_LINEAR       # the consumer's backward kernel already applied f'(y) (fusion.py)
    # bias gradient: with nothing to multiply into err_output, the wgmma wgrad kernel delivers the
    # column sums as an extra product row (no separate pass over err_output at all)
    bias_row = bool(need_b and act == ACT_LINEAR and lp_ok)
    parts = slices = None
    if act != ACT_LINEAR or (need_b and not bias_row):
        if need_b:
            slices, parts = _bias_partials(unit, pixels, f)
        y = unit.output.dev if act != ACT_LINEAR else None
        ext.err_act_colsum(err, y, pixels, f, act, parts)
        unit.err_output.dev_written()
        _launch()
    f_pad = _roundup(f, 8)
    err_mm, g_mm = err, g
    if lp_ok and f_pad != f:
        # n_kernels % 8 != 0 (e.g. the GA-tuned MNIST conv with 87 kernels): one pad kernel makes
        # err_output [pixels][f_pad] so dgrad and wgrad stay on the tensor cores with 16-byte
        # gathers / TMA instead of the element-wise gather
        err_mm = _tmp(unit, "errpad", (pixels, f_pad), err.dtype)
        ext.pad_channels(err, err_mm, f, f_pad)
        _launch()
        g_mm = list(g)
        g_mm[6] = f_pad
    x3 = (not lp_ok) and fp32x.enabled(unit) and fp32x._f32(err, x)
    ec = es = None
    if x3:
        ec, es = fp32x.conv_split_err(unit, ext, err, g, pixels, unit.need_err_input,
                                      bool(need_w))
    # fork here: everything wgrad needs exists; it runs beside the dgrad launched next
    side = _fork_side(unit) if (need_w and unit.need_err_input) else None
    if unit.need_err_input:
        ei = unit.err_input.dev if unit.err_input_beta else unit.err_input.dev_out
        r = -1
        if x3 and fp32x.conv_dgrad(unit, ext, ec, ei, g, unit.err_input_alpha,
                                   unit.err_input_beta):
            r = 0
        # derivative of the producer layer's activation, folded into this dgrad's epilogue
        # (workflow/fusion.py::fuse_backward_derivatives)
        in_act = int(unit.__dict__.get("in_deriv_act_", 0) or 0)
        folded = False
        if lp_ok:
            wd = fwd.weights_lp_t_
            fold = bool(in_act and _is_bf16(ei) and not unit.err_input_beta)
            r = ext.conv_dgrad(err_mm, wd, wd.shape[1], False, ei, g_mm,
                               float(unit.err_input_alpha), float(unit.err_input_beta), 1,
                               x if fold else None, in_act if fold else 0)
            if r == -5:      # the fold was declined (alignment): plain tensor-core dgrad
                r = ext.conv_dgrad(err_mm, wd, wd.shape[1], False, ei, g_mm,
                                   float(unit.err_input_alpha), float(unit.err_input_beta), 1,
                                   None, 0)
                fold = False
            folded = fold and r == 0
            if r not in (0, -3, -4):
                raise RuntimeError("%s: wgmma conv dgrad refused (code %d)" % (unit, r))
            if r != 0:
                _warn_once(unit, "dgrad", r)
        if r != 0:
            # fp32 / odd shapes the tensor-core kernel declines (alignment, gather table): our own
            # SIMT implicit-GEMM kernel with the fp32 master weights
            w = unit.weights.dev
            ext.conv_dgrad(err, w, w.shape[1], bool(unit.weights_transposed), ei, g,
                           float(unit.err_input_alpha), float(unit.err_input_beta), 0, None, 0)
        unit.err_input.dev_written()
        _launch()
        if in_act and not folded:
            # the tensor-core kernel declined: apply the promised derivative in a separate pass
            ext.err_act_colsum(ei, unit.input.dev, ei.numel() // ei.shape[-1], ei.shape[-1],
                               in_act, None)
            _launch()
    if not need_w:
        return
    use_umma = lp_ok
    g_cp = 0
    f_rows = f                    # rows of one gradient partial
    if x3:
        # fp32 wgrad on the tensor cores: hi/lo parts stacked along the images
        with (torch.cuda.stream(side) if side is not None else contextlib.nullcontext()):
            xs, g3, kw3, cp3, f8 = fp32x.conv_wgrad_prepare(unit, ext, x, g, pixels)
            splits = int(ext.pick_splits(kw3, f8, 3 * pixels, _MAX_SPLITS))
            gbuf = _grad_buffer(unit, "wgrad", (splits, f8, kw3))
            r = ext.conv_wgrad(es, xs, gbuf, splits, g3, False, 1, None)
        if r in (0, 1):
            fp32x.counters["gemms"] += 1
            _launch()
            _update(unit, False, gbuf, splits, f8 * kw3, f, unit._kernel_size, g_cpad=cp3)
            if need_b:
                _update(unit, True, parts, slices, f, 1, f)
            return
        _warn_once(unit, "wgrad", r)
    s2d = fwd.__dict__.get("s2d_") if use_umma else None
    if s2d is not None:
        # first-layer strided convolution in its space-to-depth form (csrc/s2d.cu): the forward
        # pass left the transformed input; the gradient comes out in the transformed tap order
        x = s2d["xs"]
        g = list(s2d["g"])
        g[6] = f_pad
        kw = s2d["kw"]
        f_rows = f_pad
        splits = int(ext.pick_splits(kw, f_rows, pixels, _MAX_SPLITS))
    elif use_umma:
        g_cp = lp_cpad(fwd)
        g = list(g_mm)
        if g_cp:
            xp = fwd.__dict__.get("tmp_xpad_")
            if xp is None:
                raise RuntimeError("%s: padded input of the forward pass is missing" % unit)
            x = xp
            g[3] = g_cp
            kw = unit.kx * unit.ky * g_cp
        f_rows = f_pad            # padded rows (zeros) sit at the end of every partial
        splits = int(ext.pick_splits(kw, f_rows, pixels, _MAX_SPLITS))
    else:
        tiles = ((f + 63) // 64) * ((kw + 63) // 64)
        splits = max(1, min(_MAX_SPLITS, (2 * _num_sms()) // tiles, (pixels + 255) // 256))
    gbuf = _grad_buffer(unit, "wgrad", (splits, f_rows, kw)) if s2d is None else \
        _tmp(unit, "wgrad_s2d", (splits, f_rows, kw), torch.float32)
    brow = None
    if bias_row and use_umma and s2d is None:
        brow = _grad_buffer(unit, "bias_row", (splits, f_rows))
    with (torch.cuda.stream(side) if side is not None else contextlib.nullcontext()):
        if use_umma:
            r = ext.conv_wgrad(err_mm, x, gbuf, splits, g, False, 1, brow)
            if r not in (0, 1):
                raise RuntimeError("%s: wgmma conv wgrad refused (code %d)" % (unit, r))
            if r == 0:
                brow = None
            if s2d is not None:
                g2 = _grad_buffer(unit, "wgrad", (splits, f, unit._kernel_size))
                ext.s2d_unpack_grad(gbuf, g2, splits, f, f_rows, unit.ky, unit.kx, unit._n_channels,
                                    s2d["s"], s2d["kyp"], s2d["kxp"], _S2D_C)
                _launch()
                gbuf, f_rows, kw = g2, f, unit._kernel_size
        else:
            ext.conv_wgrad(err, x, gbuf, splits, g, bool(unit.weights_transposed), 0, None)
        _launch()
        if bias_row and brow is None:
            # geometry without a spare product row (kernel size a multiple of 128): classic
            # column sums
            slices, parts = _bias_partials(unit, pixels, f)
            ext.err_act_colsum(err, None, pixels, f, ACT_LINEAR, parts)
            _launch()
    _update(unit, False, gbuf, splits, f_rows * kw, f, unit._kernel_size, g_cpad=g_cp)
    if need_b:
        if brow is not None:
            _update(unit, True, brow, splits, f_rows, 1, f)
        else:
            _update(unit, True, parts, slices, f, 1, f)


# ------------------------------------------------------------------------------------------
# pooling / depooling / LRN / activations / dropout / glue ops
# ------------------------------------------------------------------------------------------
_POOL_MODES = {"max": 0, "maxabs": 1, "avg": 2, "stochastic": 3, "stochastic_abs": 4,
               "stochastic_depool": 5, "stochastic_abs_depool": 6}


def pooling_forward(unit):
    ext = _ext(unit)
    mode = _POOL_MODES[unit.KERNEL]
    ox, oy = unit.out_sxy
    x = unit.input.dev
    offs = unit.input_offset.dev_out if hasattr(unit, "input_offset") else None
    rng = getattr(unit, "rng_dev_", None)
    if mode >= 5:
        ext.pool_forward(x, None, offs, oy, ox, unit.ky, unit.kx, unit.sliding[1],
                         unit.sliding[0], mode, rng, 0)
        unit.input.dev_written()
    else:
        ext.pool_forward(x, unit.output.dev_out, offs, oy, ox, unit.ky, unit.kx,
                         unit.sliding[1], unit.sliding[0], mode, rng, fused_act(unit))
    _launch()


def pooling_backward(unit):
    ext = _ext(unit)
    ox, oy = unit.out_sxy
    is_avg = unit.KERNEL == "avg"
    offs = None if is_avg else unit.input_offset.dev
    err = unit.err_output.dev
    ei = unit.err_input.dev_out
    act = fused_act(unit)
    y = unit.output.dev if act else None
    in_act = int(unit.__dict__.get("in_deriv_act_", 0) or 0)      # see workflow/fusion.py
    xin = unit.input.dev if in_act else None
    ext.pool_backward(err.view(ei.shape[0], oy, ox, ei.shape[3]), offs, ei, oy, ox, unit.ky,
                      unit.kx, unit.sliding[1], unit.sliding[0], is_avg,
                      y.view(ei.shape[0], oy, ox, ei.shape[3]) if act else None, act,
                      xin, in_act)
    _launch()


def depooling_forward(unit):
    ext = _ext(unit)
    ext.scatter_offsets(unit.input.dev, unit.output_offset.dev, unit.output.dev_out)
    _launch()


def lrn_forward(unit):
    _ext(unit).lrn_forward(unit.input.dev, unit.output.dev_out, unit.n, unit.alpha,
                           unit.beta, unit.k)
    _launch()


def lrn_backward(unit):
    _ext(unit).lrn_backward(unit.err_output.dev, unit.input.dev, unit.err_input.dev_out,
                            unit.n, unit.alpha, unit.beta, unit.k,
                            int(unit.__dict__.get("in_deriv_act_", 0) or 0))
    _launch()


def activation_forward(unit):
    _ext(unit).act_forward(unit.input.dev, unit.output.dev_out, unit.CODE,
                           float(unit.factor if unit.factor is not None else 1.0))
    _launch()


def activation_backward(unit):
    x = unit.input.dev if unit.NEEDS_INPUT else None
    y = unit.output.dev if unit.NEEDS_OUTPUT else None
    _ext(unit).act_backward(unit.err_output.dev, x, y, unit.err_input.dev_out, unit.CODE,
                            float(unit.factor))
    _launch()


def dropout_forward(unit):
    ext = _ext(unit)
    x = unit.input.dev
    if unit.active:
        ext.dropout_forward(x, unit.output.dev_out, unit.mask.dev_out, unit.rng_dev_,
                            min(unit.threshold, 0xFFFFFFFF), 1.0 / (1.0 - unit.dropout_ratio))
    else:
        ext.cast_copy(x, unit.output.dev_out)
    _launch()


def dropout_backward(unit):
    _ext(unit).binary_op(unit.err_output.dev, unit.mask.dev, unit.err_input.dev_out, 0)
    _launch()


def cutter_forward(unit):
    _ext(unit).crop_nhwc(unit.input.dev, unit.output.dev_out, unit.padding[1],
                         unit.padding[0], False)
    _launch()


def cutter_backward(unit):
    err = unit.err_output.dev.view(unit.output_shape)
    _ext(unit).crop_nhwc(err, unit.err_input.dev_out, unit.padding[1], unit.padding[0], True)
    _launch()


def cutter1d_forward(unit):
    out = unit.output.dev if unit.beta else unit.output.dev
    _ext(unit).axpby_2d(unit.input.dev, unit.input_offset, out, unit.output_offset,
                        unit.length, float(unit.alpha), float(unit.beta))
    unit.output.dev_written()
    _launch()


def binary_forward(unit, op):
    _ext(unit).binary_op(unit.x.dev, unit.y.dev, unit.output.dev_out, 0 if op == "mul" else 1)
    _launch()


def multiplier_backward(unit):
    _ext(unit).mul_backward(unit.x.dev, unit.y.dev, unit.err_output.dev, unit.err_x.dev_out,
                            unit.err_y.dev_out)
    _launch()


def zero_filler(unit):
    ext = _ext(unit)
    w = unit.weights.dev
    ext.mask_mul(w, unit.mask.dev)
    unit.weights.dev_written()
    _launch()


# ------------------------------------------------------------------------------------------
# evaluators
# ------------------------------------------------------------------------------------------
def evaluate_softmax(unit):
    if unit.__dict__.pop("fused_done_", False):
        return          # the few-output FC kernel already did this step's evaluation
    ext = _ext(unit)
    y = unit.output.dev
    if y.dtype != torch.float32:
        raise RuntimeError("softmax probabilities must be fp32 on the device")
    conf = unit.confusion_matrix.dev if unit.confusion_matrix else None
    ext.evaluate_softmax(y, unit.max_idx.dev, unit.labels.dev, unit.err_output.dev_out,
                         unit.batch_dev_, unit.n_err.dev, conf, unit.max_err_output_sum.dev)
    unit.n_err.dev_written()
    unit.max_err_output_sum.dev_written()
    if conf is not None:
        unit.confusion_matrix.dev_written()
    _launch()


def evaluate_mse(unit):
    ext = _ext(unit)
    y = unit.output.dev
    t = unit.target.dev
    dm = unit.__dict__.get("denorm_mul_")
    if dm is None:
        co = unit.denorm_coefficients()
        dm = False if co is None else torch.from_numpy(co[0]).to(unit.device.torch_device)
        unit.__dict__["denorm_mul_"] = dm
    ext.evaluate_mse(y, t.view(y.shape), unit.err_output.dev_out, unit.batch_dev_,
                     dm if dm is not False else None, bool(unit.root), unit.metrics.dev,
                     unit.mse.dev_out)
    unit.metrics.dev_written()
    _launch()
    if unit.labels and unit.class_targets:
        ext.mse_find_closest(y, unit.class_targets.dev.float().contiguous(), unit.labels.dev,
                             unit.batch_dev_, unit.n_err.dev)
        unit.n_err.dev_written()
        _launch()


# ------------------------------------------------------------------------------------------
# restricted Boltzmann machines (ops/rbm_units.py; csrc/rbm.cu)
# ------------------------------------------------------------------------------------------
def rbm_sample(unit):
    """Binarization: Bernoulli(input) on the first batch_size rows, input copied on the rest."""
    _ext(unit).rbm_sample(unit.input.dev, unit.output.dev_out, int(unit.batch_size), unit.rng_up_.dev)
    _launch()


def _col_mean(unit, ext, name, x, rows, cols, out):
    """out[1][cols] = mean of the first ``rows`` rows of x: the bias-gradient column sums
    (ACT_LINEAR: x is only read) per row slice, their sum, and the 1/rows scale."""
    slices = ext.colsum_slices(rows)
    parts = _tmp(unit, name + "_parts", (slices, cols), torch.float32)
    sums = _tmp(unit, name + "_sums", (1, cols), torch.float32)
    ext.err_act_colsum(x, None, rows, cols, ACT_LINEAR, parts)
    ext.col_sums(parts, sums, slices, cols, False)
    ext.axpby_2d(sums, 0, out.dev_out.view(1, cols), 0, cols, 1.0 / rows, 0.0)
    _launch(3)


def rbm_batch_stats(unit):
    """BatchWeights: weights_batch[V][H] = v^T h / bs, vbias_batch = <v>, hbias_batch = <h> over the
    first batch_size rows (the GEMM's reduction length is bs, so the rows past it never enter)."""
    ext = _ext(unit)
    v, h = unit.v.dev, unit.h.dev
    bs = int(unit.batch_size)
    nv, nh = v.numel() // v.shape[0], h.numel() // h.shape[0]
    wb = unit.weights_batch.dev_out
    if _is_bf16(v) and _is_bf16(h) and nv % 8 == 0 and nh % 8 == 0:
        # the FC weight-gradient form: (h^T . v) with a transposed store = v^T . h
        r = ext.gemm(h, nh, True, v, nv, False, wb, nh, True, nh, nv, bs, None, 0, 1.0 / bs, 0.0,
                     1, 0, 1)
        if r != 0:
            raise RuntimeError("%s: wgmma v^T h refused the shape (code %d)" % (unit, r))
    else:
        _path(unit, "rbm_stats:simt")
        ext.gemm(v, nv, True, h, nh, False, wb, nh, False, nv, nh, bs, None, 0, 1.0 / bs, 0.0,
                 1, 0, 0)
    _launch()
    _col_mean(unit, ext, "v_mean", v, bs, nv, unit.vbias_batch)
    _col_mean(unit, ext, "h_mean", h, bs, nh, unit.hbias_batch)


def rbm_gradients(unit):
    """GradientsCalculator: grad = positive-phase statistic - negative-phase statistic."""
    ext = _ext(unit)
    for g, s0, s1 in ((unit.vbias_grad, unit.vbias0, unit.vbias1),
                      (unit.hbias_grad, unit.hbias0, unit.hbias1),
                      (unit.weights_grad, unit.weights0, unit.weights1)):
        a, b = s0.dev, s1.dev
        out = g.dev_out
        n = out.numel() // out.shape[0]
        ext.axpby_2d(a, 0, out, 0, n, 1.0, 0.0)
        ext.axpby_2d(b, 0, out, 0, n, -1.0, 1.0)
        _launch(2)


def rbm_apply(unit):
    """WeightsUpdater: W[h][v] += lr * weights_grad[v][h], biases += lr * their gradients."""
    _ext(unit).rbm_apply(unit.weights.dev, unit.weights_grad.dev, unit.hbias.dev, unit.hbias_grad.dev,
                         unit.vbias.dev, unit.vbias_grad.dev, float(unit.learning_rate))
    for a in (unit.weights, unit.hbias, unit.vbias):
        a.dev_written()
    _launch()


# ------------------------------------------------------------------------------------------
# deconvolution (transposed conv = the conv dgrad / fprop / wgrad kernels with swapped roles)
# ------------------------------------------------------------------------------------------
def _deconv_geom(u):
    """Geometry of the *equivalent convolution*: image = deconv output side."""
    return [u._batch_size if hasattr(u, "_batch_size") else u._output_shape[0], u._sy, u._sx,
            u._n_channels, u.input.shape[1], u.input.shape[2], u.n_kernels, u.ky, u.kx,
            u.sliding[1], u.sliding[0], u.padding[1], u.padding[0]]


def _rhits(unit, like):
    """Reciprocal overlap map in the activation dtype (static for a geometry)."""
    t = unit.__dict__.get("rhits_dev_")
    if t is None or t.dtype != like.dtype:
        unit.hits.map_read()
        r = 1.0 / numpy.maximum(unit.hits.mem, 1).astype(numpy.float32)
        t = torch.from_numpy(r).to(like.device).to(like.dtype).contiguous()
        unit.__dict__["rhits_dev_"] = t
    return t


def _deconv_owner(unit):
    """The Conv unit that owns the (tied) weights of a Deconv / GDDeconv: its bf16 operand
    shadows (``weights_lp_`` [F][ld] and ``weights_lp_t_`` [tap][F_pad][C_pad]) are exactly what
    the wgmma kernels need with the roles swapped (deconv forward = conv dgrad, GDDeconv
    err_input = conv fprop, GDDeconv wgrad = conv wgrad with image and error exchanged)."""
    o = unit.__dict__.get("shadow_owner_", False)
    if o is not False:
        return o
    o = None
    cand = [getattr(unit, "forward_unit", None)]
    wf = unit.workflow
    if wf is not None:
        cand += list(getattr(wf, "units", []))
    for u in cand:
        if u is None or u is unit or not hasattr(u, "weights_lp_t_"):
            continue
        if getattr(u, "weights", None) is unit.weights and getattr(u, "on_cuda", False):
            o = u
            break
    unit.__dict__["shadow_owner_"] = o
    return o


def _deconv_lp(unit, *tensors):
    """Owner conv with valid shadows when this deconv call can run on the tensor cores."""
    o = _deconv_owner(unit)
    if o is None or not lp_enabled(o) or not all(_is_bf16(t) for t in tensors):
        return None
    if unit.n_kernels % 8 or unit.weights_transposed:
        return None
    ensure_shadows(o)         # (filled by the owner's initialize() and by every update kernel)
    return o


def deconv_forward(unit):
    ext = _ext(unit)
    x = unit.input.dev                       # [N, oy, ox, F] plays the role of err_out
    out = unit.output.dev_out                # [N, sy, sx, C] plays the role of err_in
    g = _deconv_geom(unit)
    alpha = 1.0 if unit.hits else float(unit.scale)
    o = _deconv_lp(unit, x, out)
    r = -1
    if o is not None:
        wd = o.weights_lp_t_
        r = int(ext.conv_dgrad(x, wd, wd.shape[1], False, out, g, alpha, 0.0, 1, None, 0))
        if r not in (0, -3, -4):
            raise RuntimeError("%s: wgmma deconv (dgrad kernel) refused (code %d)" % (unit, r))
        if r != 0:
            _warn_once(unit, "deconv", r)
    if r != 0:
        w = unit.weights.dev
        ext.conv_dgrad(x, w, w.shape[1], bool(unit.weights_transposed), out, g, alpha, 0.0, 0,
                       None, 0)
    _launch()
    if unit.hits:
        ext.mask_mul(out, _rhits(unit, out))
        _launch()


def deconv_backward(unit):
    ext = _ext(unit)
    err = unit.err_output.dev                # [N, sy, sx, C]
    if unit.unsafe_padding:
        ext.mask_mul(err, _rhits(unit, err))
    else:
        ext.axpby_2d(err.view(err.shape[0], -1), 0, err.view(err.shape[0], -1), 0,
                     err.numel() // err.shape[0], float(unit.scale), 0.0)
    unit.err_output.dev_written()
    _launch()
    g = _deconv_geom(unit)
    f, kw = unit.n_kernels, unit._kernel_size
    xin = unit.input.dev                     # [N, oy, ox, F]: the "error" operand of the wgrad
    o = _deconv_lp(unit, err, xin)
    # first-layer geometry: the owner's fprop shadow is channel-padded [F][tap][cp]; the image
    # operand (= the scaled err_output here) is padded the same way, once, for fprop and wgrad
    cp = lp_cpad(o) if o is not None else 0
    img, g_lp = err, list(g)
    if cp:
        img = _tmp(unit, "errpad", tuple(err.shape[:3]) + (cp,), err.dtype)
        ext.pad_channels(err, img, unit._n_channels, cp)
        _launch()
        g_lp[3] = cp
    if unit.need_err_input:
        alpha, beta = float(unit.err_input_alpha), float(unit.err_input_beta)
        plain = alpha == 1.0 and beta == 0.0
        ei = unit.err_input.dev_out if beta == 0.0 else unit.err_input.dev
        dst = ei if plain else _tmp(unit, "ei", tuple(ei.shape), ei.dtype)
        r = -1
        if o is not None and _is_bf16(ei):
            w = o.weights_lp_
            r = int(ext.conv_fprop(img, w, w.shape[1], False, None, dst, g_lp, 0, 1))
            if r not in (0, -3, -4):
                raise RuntimeError("%s: wgmma GDDeconv err_input refused (code %d)" % (unit, r))
            if r != 0:
                _warn_once(unit, "gd_deconv err_input", r)
        if r != 0:
            w = unit.weights.dev
            ext.conv_fprop(err, w, w.shape[1], bool(unit.weights_transposed), None, dst, g, 0, 0)
        _launch()
        if not plain:
            # err_input = alpha * (im2col(err_output) . W^T) + beta * err_input
            # (/root/reference/gd_deconv.py:340-349)
            n = ei.shape[0]
            ext.axpby_2d(dst.view(n, -1), 0, ei.view(n, -1), 0, ei.numel() // n, alpha, beta)
            _launch()
        unit.err_input.dev_written()
    if not (unit.need_gradient_weights and unit.weights):
        return
    pixels = unit.input.size // f
    if o is not None:
        kw_lp = unit.kx * unit.ky * cp if cp else kw
        splits = int(ext.pick_splits(kw_lp, f, pixels, _MAX_SPLITS))
        gbuf = _grad_buffer(unit, "wgrad", (splits, f, kw_lp))
        r = int(ext.conv_wgrad(xin, img, gbuf, splits, g_lp, False, 1, None))
        if r not in (0, 1):
            raise RuntimeError("%s: wgmma GDDeconv wgrad refused (code %d)" % (unit, r))
        _launch()
        _update(unit, False, gbuf, splits, f * kw_lp, f, kw, g_cpad=cp)
        return
    tiles = ((f + 63) // 64) * ((kw + 63) // 64)
    splits = max(1, min(_MAX_SPLITS, (2 * _num_sms()) // tiles, (pixels + 255) // 256))
    gbuf = _grad_buffer(unit, "wgrad", (splits, f, kw))
    ext.conv_wgrad(unit.input.dev, err, gbuf, splits, g, bool(unit.weights_transposed), 0, None)
    _launch()
    _update(unit, False, gbuf, splits, f * kw, f, kw)


# ------------------------------------------------------------------------------------------
# LSTM over a sequence (ops/lstm_seq.py)
# ------------------------------------------------------------------------------------------
def _lstm_gemm_nt(ext, unit, a, w_lp, w_f32, out, m, n, k, bias, beta):
    """out[m, n] = a[m, k] . W[n, k]^T (+ bias) (+ beta * out); wgmma when a is bf16."""
    if w_lp is not None and _is_bf16(a) and k % 8 == 0:
        r = ext.gemm(a, k, False, w_lp, w_lp.shape[1], True, out, n, False, m, n, k, bias,
                     ACT_LINEAR, 1.0, beta, 1, 0, 1)
        if r != 0:
            raise RuntimeError("%s: wgmma LSTM GEMM refused (code %d)" % (unit, r))
    else:
        ext.gemm(a, k, False, w_f32, k, True, out, n, False, m, n, k, bias, ACT_LINEAR, 1.0,
                 beta, 1, 0, 0)
    _launch()


def _lstm_persist_enabled():
    import os
    return os.environ.get("ZNICZ_LSTM_PERSIST", "1") != "0"


def lstm_seq_forward(unit):
    ext = _ext(unit)
    x = unit.input.dev                       # [B, T, I]
    b, t, i = x.shape
    h = unit.hidden_size
    xh = unit.xh.dev_out                     # [T + 1, B, I + H]
    gates = unit.gates.dev_out
    cells = unit.cells.dev_out
    hidden = unit.hidden.dev_out
    out = unit.output.dev_out
    w = unit.weights.dev
    w_lp = None
    if lp_enabled(unit) and _is_bf16(x) and (i + h) % 8 == 0:
        ensure_shadows(unit)
        w_lp = unit.weights_lp_
    bias = unit.bias.dev if unit.include_bias and unit.bias else None
    # [x_t] part of every step's operand in one strided copy; h_{-1} = 0
    xh_flat = xh.view((t + 1) * b, i + h)
    # x [B][T][I] -> the [x_t] part of xh[t][b][0:I] for every step, one launch
    ext.swap01_2d(x, i, 0, xh, i + h, 0, b, t, i)
    _launch()
    ext.axpby_2d(xh[0], i, xh[0], i, h, 0.0, 0.0)
    _launch()
    seq = unit.return_sequences
    persist = -1
    state = None
    if w_lp is not None and _lstm_persist_enabled():
        # the whole time loop in ONE cluster launch: W resident in shared memory, gates GEMM on
        # wgmma, cell math in the epilogue, h exchanged through distributed shared memory
        # (csrc/lstm_persist.cu)
        nstate = int(ext.lstm_state_floats(t, b, i, h))
        if nstate:
            state = _tmp(unit, "lstm_state", (nstate,), torch.float32)
            persist = int(ext.lstm_fwd_persist(xh, w_lp, bias, state, h, None))
        if persist == 0:
            _launch()
    # gates / cells of this pass live in the kernels' private layout (None: in the public arrays)
    unit.__dict__["lstm_state_"] = state if persist == 0 else None
    z = _tmp(unit, "z", (b, 4 * h), torch.float32) if persist != 0 else None
    for s in range(t if persist != 0 else 0):
        _lstm_gemm_nt(ext, unit, xh[s], w_lp, w, z, b, 4 * h, i + h, bias, 0.0)
        ext.lstm_cell_fwd(z, cells[s - 1] if s else None, cells[s], gates[s],
                          hidden, s * b * h, h, xh, (s + 1) * b * (i + h) + i, i + h, b, h)
        _launch()
    # the unit's output: the whole sequence [B, T, H] or the last step [B, H]
    if persist == 0:
        # the kernel leaves h_t only in the [x | h] operand of step t + 1
        if seq:
            ext.swap01_2d(xh[1:], i + h, i, out, h, 0, t, b, h)
        else:
            ext.axpby_2d(xh[t], i, out, 0, h, 1.0, 0.0)
        _launch()
    elif seq:
        ext.swap01_2d(hidden, h, 0, out, h, 0, t, b, h)      # [T][B][H] -> [B][T][H]
        _launch()
    else:
        ext.axpby_2d(hidden[t - 1], 0, out, 0, h, 1.0, 0.0)
        _launch()
    del xh_flat


def lstm_seq_backward(unit):
    ext = _ext(unit)
    gates = unit.gates.dev
    cells = unit.cells.dev
    xh = unit.xh.dev
    t, b, h4 = gates.shape
    h = h4 // 4
    i = xh.shape[2] - h
    err = unit.err_output.dev
    seq = err.dim() == 3
    dz = unit.dz.dev_out                    # [T, B, 4H] compute dtype
    w = unit.weights.dev
    fwd = unit.forward_unit
    w_lp = getattr(fwd, "weights_lp_", None) if (lp_enabled(unit) and _is_bf16(dz)) else None
    dxh = _tmp(unit, "dxh", (b, i + h), dz.dtype)
    dc = [_tmp(unit, "dc0", (b, h), torch.float32), _tmp(unit, "dc1", (b, h), torch.float32)]
    need_ei = unit.need_err_input
    ei = None
    if need_ei:
        ei = unit.err_input.dev if unit.err_input_beta else unit.err_input.dev_out
    persist = -1
    state = fwd.__dict__.get("lstm_state_") if fwd is not None else None
    if (state is not None and w_lp is not None and _is_bf16(err) and
            (not need_ei or (unit.err_input_alpha == 1 and not unit.err_input_beta))):
        whp = _tmp(unit, "whp", (h, h4), torch.bfloat16)
        part = _tmp(unit, "lstm_part", (int(ext.lstm_part_floats(b, h)),), torch.float32)
        persist = int(ext.lstm_bwd_persist(err, bool(seq), state, part, dz, w_lp, whp, i))
    if persist != 0 and state is not None:
        # per-step fallback after a persistent forward: gates / cells back into the public arrays
        ext.lstm_unpack_state(state, gates, cells)
        _launch()
    if persist == 0:
        _launch(2)
        if need_ei:
            # dx for every step in one GEMM: [T B][4H] . W_x, then [T][B][I] -> [B][T][I]
            dx = _tmp(unit, "dx_all", (t, b, i), ei.dtype)
            r = ext.gemm(dz.view(t * b, h4), h4, False, w_lp, w_lp.shape[1], False, dx, i, False,
                         t * b, i, h4, None, 0, 1.0, 0.0, 1, 0, 1)
            if r != 0:
                raise RuntimeError("%s: wgmma LSTM dx refused (code %d)" % (unit, r))
            ext.swap01_2d(dx, i, 0, ei, i, 0, t, b, i)
            _launch(2)
    for s in range(t - 1 if persist != 0 else -1, -1, -1):
        if seq:
            e_t, e_off, lde = err, s * h, t * h
        else:
            e_t, e_off, lde = (err, 0, h) if s == t - 1 else (None, 0, 0)
        ext.lstm_cell_bwd(e_t, e_off, lde, dxh if s < t - 1 else None, i, i + h,
                          dc[(s + 1) & 1] if s < t - 1 else None, gates[s], cells[s],
                          cells[s - 1] if s else None, dc[s & 1], dz[s], b, h)
        _launch()
        if s > 0 or need_ei:
            # [dx_t | dh_{t-1}] = dz_t . W      (B = W stored [K = 4H][N = I + H], MN-major)
            if w_lp is not None and h4 % 8 == 0:
                r = ext.gemm(dz[s], h4, False, w_lp, w_lp.shape[1], False, dxh, i + h, False,
                             b, i + h, h4, None, 0, 1.0, 0.0, 1, 0, 1)
                if r != 0:
                    raise RuntimeError("%s: wgmma LSTM dgrad refused (code %d)" % (unit, r))
            else:
                ext.gemm(dz[s], h4, False, w, i + h, False, dxh, i + h, False, b, i + h, h4,
                         None, 0, 1.0, 0.0, 1, 0, 0)
            _launch()
            if need_ei:
                ext.axpby_2d(dxh, 0, ei.view(b, t * i), s * i, i,
                             float(unit.err_input_alpha), float(unit.err_input_beta))
                _launch()
    if need_ei:
        unit.err_input.dev_written()
    if not (unit.need_gradient_weights and unit.weights):
        return
    # gradW[4H, I + H] = dZ^T . XH over all T * B rows: one GEMM
    rows = t * b
    dz2 = dz.view(rows, h4)
    xh2 = xh[:t].reshape(rows, i + h) if not xh[:t].is_contiguous() else xh[:t].view(rows, i + h)
    gbuf = _grad_buffer(unit, "wgrad", (1, h4, i + h))
    if w_lp is not None and h4 % 8 == 0 and (i + h) % 8 == 0:
        r = ext.gemm(dz2, h4, True, xh2, i + h, False, gbuf, i + h, False, h4, i + h, rows,
                     None, 0, 1.0, 0.0, 1, 0, 1)
        if r != 0:
            raise RuntimeError("%s: wgmma LSTM wgrad refused (code %d)" % (unit, r))
    else:
        ext.gemm(dz2, h4, True, xh2, i + h, False, gbuf, i + h, False, h4, i + h, rows, None, 0,
                 1.0, 0.0, 1, 0, 0)
    _launch()
    _update(unit, False, gbuf, 1, 0, h4, i + h)
    if unit.include_bias and unit.bias:
        slices, parts = _bias_partials(unit, rows, h4)
        ext.err_act_colsum(dz2, None, rows, h4, ACT_LINEAR, parts)
        _launch()
        _update(unit, True, parts, slices, h4, 1, h4)
