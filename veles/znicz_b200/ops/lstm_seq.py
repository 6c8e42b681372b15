"""LSTM over a whole sequence as ONE forward unit + ONE GD unit (north-star config 5).

The reference only has a single-step cell built from ~12 sub-units and unrolls time by
chaining cells in the unit graph (/root/reference/lstm.py:52-143, SURVEY §5 "long-context"):
graph size, launch count and Python overhead all grow linearly with the sequence length.
Here the same cell (sigmoid gates, scaled-tanh memory maker and output activation, no
peephole = the reference's ``simple`` variant) runs over ``[batch, T, features]`` inside one
unit:

  forward   per step t: z_t = [x_t | h_{t-1}] · Wᵀ + b  (one GEMM, wgmma in bf16 mode) and one
            fused cell kernel (gates, c_t, h_t; h_t is written straight into the output
            sequence and into the [x | h] operand of step t + 1);
  backward  per step (reverse): one fused cell-gradient kernel and one GEMM dz_t · W that yields
            [dx_t | dh_{t-1}]; the weight gradient is ONE GEMM over all T·batch rows at the
            end, the bias gradient one column-sum kernel, then the usual fused update.

2·T GEMMs + 2·T small kernels per direction — captured once in a CUDA graph by
``StandardWorkflow``. Layer DSL: ``{"type": "lstm_seq", "->": {"output_sample_shape": H,
"return_sequences": False}, "<-": {...}}``. Weights ``[4H, I + H]`` in gate order
(input, forget, memory, output), bias ``[4H]``.
"""
from __future__ import annotations

import numpy

from ..core.memory import Array
from . import nn_units
from .gd import GDCommon
from .nn_units import ACT_LINEAR

A, B = 1.7159, 0.6666


def _sigmoid(x):
    return 1.0 / (1.0 + numpy.exp(-x))


def _stanh(x):
    return A * numpy.tanh(B * x)


def _dstanh_y(y):
    return y * y * (-0.388484177) + 1.14381894


class LSTMSequence(nn_units.Forward):
    MAPPING = {"lstm_seq"}
    ACT = ACT_LINEAR
    GD_LINK_ATTRS = ("gates", "cells", "hidden", "xh")   # extra state the GD unit shares

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        h = kwargs.get("output_sample_shape", kwargs.get("hidden_size"))
        self.hidden_size = int(h[0] if isinstance(h, (tuple, list)) else h)
        self.return_sequences = kwargs.get("return_sequences", False)
        self.forget_bias = kwargs.get("forget_bias", 1.0)
        self.gates = Array(shallow_pickle=True)     # [T, B, 4H] activated gates
        self.cells = Array(shallow_pickle=True)     # [T, B, H]
        self.hidden = Array(shallow_pickle=True)    # [T, B, H] every h_t (backward needs them)
        self.xh = Array(shallow_pickle=True)        # [T + 1, B, I + H] GEMM operand per step
        self.exports = ["weights", "bias", "include_bias", "weights_transposed", "hidden_size",
                        "return_sequences"]

    @property
    def neurons_number(self):
        return self.hidden_size

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        super().initialize(device=device, **kwargs)
        if len(self.input.shape) != 3:
            raise ValueError("lstm_seq expects input [batch, time, features], got %s" % (
                self.input.shape,))
        if self.weights_transposed:
            raise ValueError("lstm_seq does not support weights_transposed")
        b, t, i = self.input.shape
        h = self.hidden_size
        dtype = self.input.dtype
        if not self.weights or self.weights.shape != (4 * h, i + h):
            std = self.weights_stddev or min(0.5, 1.0 / numpy.sqrt(i + h))
            w = numpy.zeros((4 * h, i + h), dtype=dtype)
            self.fill_array(self.weights_filling, w, std)
            self.weights.reset(w)
            bias = numpy.zeros(4 * h, dtype=dtype)
            bias[h:2 * h] = self.forget_bias          # remember by default
            self.bias.reset(bias)
        self.make_output((b, t, h) if self.return_sequences else (b, h), dtype)
        for arr, shape in ((self.gates, (t, b, 4 * h)), (self.cells, (t, b, h)),
                           (self.hidden, (t, b, h)), (self.xh, (t + 1, b, i + h))):
            if not arr or arr.shape != shape:
                arr.reset(numpy.zeros(shape, dtype=numpy.float32 if arr is not self.xh and
                                      arr is not self.hidden else dtype))
        if self.on_cuda:
            self.xh.dev_dtype = self.input.dev_dtype
            self.hidden.dev_dtype = self.input.dev_dtype
        self.init_vectors(self.input, self.output, self.weights, self.bias, self.gates,
                          self.cells, self.hidden, self.xh)
        if self.on_cuda:
            self.refresh_shadows()
        return None

    def refresh_shadows(self):
        from ..kernels import api
        api.refresh_weight_shadows(self)

    # -- numpy oracle ---------------------------------------------------------------------------
    def numpy_run(self):
        for a in (self.input, self.weights, self.bias):
            a.map_read()
        for a in (self.output, self.gates, self.cells, self.hidden, self.xh):
            a.map_invalidate()
        x = self.input.mem
        b, t, i = x.shape
        h = self.hidden_size
        w, bias = self.weights.mem, self.bias.mem
        xh = self.xh.mem
        xh[:t, :, :i] = x.transpose(1, 0, 2)
        xh[0, :, i:] = 0
        c_prev = numpy.zeros((b, h), dtype=numpy.float64)
        for s in range(t):
            z = xh[s].astype(numpy.float64).dot(w.T.astype(numpy.float64)) + bias
            ig, fg = _sigmoid(z[:, :h]), _sigmoid(z[:, h:2 * h])
            gg, og = _stanh(z[:, 2 * h:3 * h]), _sigmoid(z[:, 3 * h:])
            c = ig * gg + fg * c_prev
            hv = og * _stanh(c)
            self.gates.mem[s] = numpy.concatenate([ig, fg, gg, og], axis=1)
            self.cells.mem[s] = c
            self.hidden.mem[s] = hv
            xh[s + 1, :, i:] = hv
            c_prev = c
        if self.return_sequences:
            self.output.mem[...] = self.hidden.mem.transpose(1, 0, 2)
        else:
            self.output.mem[...] = self.hidden.mem[t - 1]

    # -- device ---------------------------------------------------------------------------------
    def cuda_run(self):
        from ..kernels import api
        api.lstm_seq_forward(self)


class GDLSTMSequence(GDCommon):
    MAPPING = {"lstm_seq"}
    ACT = ACT_LINEAR

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.demand("weights", "bias", "gates", "cells", "hidden", "xh")
        self.dz = Array(shallow_pickle=True)        # [T, B, 4H]

    def initialize(self, device=None, **kwargs):
        if not self.err_output or not self.input or not self.gates:
            return True
        r = super().initialize(device=device, **kwargs)
        t, b, h4 = self.gates.shape
        if not self.dz or self.dz.shape != (t, b, h4):
            self.dz.reset(numpy.zeros((t, b, h4), dtype=self.input.dtype))
        if self.on_cuda:
            self.dz.dev_dtype = self.input.dev_dtype
        self.init_vectors(self.dz, self.err_output, self.err_input, self.gates, self.cells,
                          self.hidden, self.xh)
        return r

    def numpy_run(self):
        for a in (self.err_output, self.weights, self.gates, self.cells, self.xh):
            a.map_read()
        t, b, h4 = self.gates.shape
        h = h4 // 4
        i = self.xh.shape[2] - h
        w = self.weights.mem.astype(numpy.float64)
        eo = self.err_output.mem.astype(numpy.float64)
        seq = eo.ndim == 3
        dz = numpy.zeros((t, b, h4), dtype=numpy.float64)
        dx = numpy.zeros((b, t, i), dtype=numpy.float64)
        dh_rec = numpy.zeros((b, h))
        dc_next = numpy.zeros((b, h))
        for s in range(t - 1, -1, -1):
            g = self.gates.mem[s].astype(numpy.float64)
            ig, fg, gg, og = g[:, :h], g[:, h:2 * h], g[:, 2 * h:3 * h], g[:, 3 * h:]
            c = self.cells.mem[s].astype(numpy.float64)
            c_prev = self.cells.mem[s - 1].astype(numpy.float64) if s else numpy.zeros((b, h))
            dh = dh_rec + (eo[:, s, :] if seq else (eo if s == t - 1 else 0.0))
            tc = _stanh(c)
            dc = dh * og * _dstanh_y(tc) + dc_next
            dz[s, :, :h] = dc * gg * ig * (1 - ig)
            dz[s, :, h:2 * h] = dc * c_prev * fg * (1 - fg)
            dz[s, :, 2 * h:3 * h] = dc * ig * _dstanh_y(gg)
            dz[s, :, 3 * h:] = dh * tc * og * (1 - og)
            dxh = dz[s].dot(w)
            dx[:, s, :] = dxh[:, :i]
            dh_rec = dxh[:, i:]
            dc_next = dc * fg
        self.dz.map_invalidate()
        self.dz.mem[...] = dz
        if self.need_err_input:
            self.err_input.map_invalidate()
            ei = self.err_input.mem
            ei[...] = (self.err_input_alpha * dx + (self.err_input_beta * ei
                                                    if self.err_input_beta else 0)).reshape(ei.shape)
        if self.need_gradient_weights:
            xh = self.xh.mem[:t].astype(numpy.float64).reshape(t * b, -1)
            self.gradient_weights.map_invalidate()
            self.gradient_weights.mem[...] = dz.reshape(t * b, h4).T.dot(xh)
            self.numpy_update("weights")
            if self.include_bias:
                self.gradient_bias.map_invalidate()
                self.gradient_bias.mem[...] = dz.reshape(t * b, h4).sum(axis=0)
                self.numpy_update("bias")

    def cuda_run(self):
        from ..kernels import api
        api.lstm_seq_backward(self)
