"""Kohonen self-organising map units.

Parity: /root/reference/kohonen.py (KohonenForward :72, KohonenTrainer :259,
KohonenDecision :536, KohonenValidator :585). The reference implements these for OpenCL +
numpy only (``@implementer(IOpenCLUnit, INumpyUnit)`` :71,258 — there is no ``.cu``); here
the device path is CUDA (``csrc/som.cu``): one CTA per sample finds the winner with a
warp-shuffle argmin, one thread per weight applies the batch update.

Training step (batch semantics, :470-500): for every sample find the winner neuron
(min ||w − x||), ``winners[winner] += 1``; gravity(n) = exp(−|c_n − c_winner|² / (2σ²)) on a
hexagonal-ish coordinate grid in [−1, 1]²; ``w += Σ_samples gravity · (x − w) · gmult`` with
``σ = radius_decay(t)·σ0`` and ``gmult = gradient_decay(t)``.
"""
from __future__ import annotations

import threading

import numpy

from ..core import prng
from ..core.accelerated_units import AcceleratedUnit
from ..core.memory import Array
from ..core.units import Unit
from ..workflow.decision import TrivialDecision


def default_gradient_decay(t):
    return 0.1 / (1.0 + t * 0.05)


def default_radius_decay(t):
    return 1.0 / (1.0 + t * 0.05)


class KohonenBase(object):
    @property
    def sample_length(self):
        return self.weights.mem.shape[0 if self.weights_transposed else 1]

    @staticmethod
    def numpy_linalg_norm(dist):
        return (dist * dist).sum(axis=1)


class KohonenForward(KohonenBase, AcceleratedUnit):
    """Winner index for every sample. ``total=True`` also accumulates winners for the whole
    epoch into ``total`` (needs minibatch_offset / minibatch_size / batch_size links)."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.demand("input", "weights")
        self.argmins = None
        self.output = Array()
        self.weights_transposed = False
        self.total = Array() if kwargs.get("total", False) else None
        if self.total is not None:
            self.minibatch_offset = None
            self.minibatch_size = None
            self.batch_size = None

    @property
    def neurons_number(self):
        return self.weights.mem.shape[0]

    def initialize(self, device=None, **kwargs):
        if not self.input or not self.weights:
            return True
        super().initialize(device=device, **kwargs)
        batch = self.input.shape[0]
        if self.input.size // batch != self.sample_length:
            raise ValueError("input sample length != weights sample length")
        self.output.reset(numpy.zeros(batch, dtype=numpy.int32))
        if self.total is not None:
            self.total.reset(numpy.zeros(int(self.batch_size), dtype=numpy.int32))
        self.init_vectors(self.input, self.weights, self.output, self.argmins)
        return None

    def _store_total(self):
        if self.total is None:
            return
        self.output.map_read()
        n = int(self.minibatch_size)
        start = int(self.minibatch_offset) - n
        self.total.map_write()
        self.total.mem[start:start + n] = self.output.mem[:n]

    def numpy_run(self):
        self.output.map_invalidate()
        if self.argmins is not None:
            self.argmins.map_read()
            self.output.mem[:] = self.argmins.mem
        else:
            self.input.map_read()
            self.weights.map_read()
            x = self.input.matrix
            w = self.weights.mem
            d = (x * x).sum(1)[:, None] - 2.0 * x.dot(w.T) + (w * w).sum(1)[None, :]
            self.output.mem[:] = d.argmin(axis=1)
        self._store_total()

    def cuda_run(self):
        if self.argmins is not None:
            self.output.dev_out.copy_(self.argmins.dev)
        else:
            x = self.input.dev
            if x.dtype != self.weights.dev.dtype:
                x = x.float()
            som_winners_device(self, x.view(x.shape[0], -1), self.weights.dev,
                               self.output.dev_out, None)
        self._store_total()


def _som_tmp(unit, name, shape, dtype):
    import torch
    key = "som_%s_" % name
    t = unit.__dict__.get(key)
    if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
        t = torch.zeros(shape, dtype=dtype, device=unit.weights.dev.device)
        unit.__dict__[key] = t
    return t


def som_winners_device(unit, x, w, argmins, winners):
    """Winners of a minibatch. Feature vectors of >= 16 elements on >= 32 neurons: distances as
    ONE wgmma GEMM over bf16 hi/lo split operands (csrc/som.cu), otherwise the scalar kernel.
    Returns the split x operand (reused by the update) or None when the scalar path ran."""
    import torch
    ext = unit.ext_
    batch, length = int(x.shape[0]), int(x.shape[1])
    neurons = int(w.shape[0])
    if length < 16 or neurons < 32:
        ext.som_winners(x, w, argmins, winners)
        return None
    kp = (length + 7) // 8 * 8
    xa = _som_tmp(unit, "xa", (batch, 3 * kp), torch.bfloat16)        # [x_hi | x_hi | x_lo]
    wb = _som_tmp(unit, "wb", (neurons, 3 * kp), torch.bfloat16)      # [w_hi | w_lo | w_hi]
    wn = _som_tmp(unit, "wn", (neurons,), torch.float32)
    dots = _som_tmp(unit, "dots", (batch, neurons), torch.float32)
    ext.som_split(x, xa, batch, length, kp, 3 * kp, kp, 0, None)
    ext.som_split(w.view(neurons, -1), wb, neurons, length, kp, 3 * kp, kp, 1, wn)
    r = ext.gemm(xa, 3 * kp, False, wb, 3 * kp, True, dots, neurons, False, batch, neurons, 3 * kp,
                 None, 0, 1.0, 0.0, 1, 0, 1)
    if r != 0:
        raise RuntimeError("%s: wgmma SOM distance GEMM refused (code %d)" % (unit, r))
    ext.som_argmin(dots, wn, argmins, winners)
    return xa


def som_update_device(unit, x, w, sigma, gmult):
    """w += gmult * (G . x - rowsum(G) o w) with the [neurons x len x batch] product on the
    wgmma GEMM (split operands: G parts along K, x parts stacked along its rows)."""
    import torch
    ext = unit.ext_
    batch, length = int(x.shape[0]), int(x.shape[1])
    neurons = int(w.shape[0])
    bp = (batch + 7) // 8 * 8
    lp = (length + 7) // 8 * 8
    ga = _som_tmp(unit, "ga", (neurons, 3 * bp), torch.bfloat16)      # [G_hi | G_hi | G_lo]
    xs = _som_tmp(unit, "xs", (3 * bp, lp), torch.bfloat16)           # [x_hi ; x_lo ; x_hi]
    rs = _som_tmp(unit, "rowsum", (neurons,), torch.float32)
    m = _som_tmp(unit, "m", (neurons, length), torch.float32)
    ext.som_gravity_split(unit._coords.dev, unit.argmins.dev, ga, rs, batch, bp, sigma)
    ext.som_split(x, xs, batch, length, lp, lp, bp * lp, 1, None)
    r = ext.gemm(ga, 3 * bp, False, xs, lp, False, m, length, False, neurons, length, 3 * bp,
                 None, 0, 1.0, 0.0, 1, 0, 1)
    if r != 0:
        raise RuntimeError("%s: wgmma SOM update GEMM refused (code %d)" % (unit, r))
    ext.som_apply(w, m, rs, gmult)


class KohonenTrainer(KohonenBase, AcceleratedUnit):
    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.argmins = Array()
        self._coords = Array()
        self.weights = Array()
        self.winners = Array()
        self.weights_filling = kwargs.get("weights_filling", "uniform")
        self.weights_stddev = kwargs.get("weights_stddev", None)
        self.weights_transposed = kwargs.get("weights_transposed", False)
        self.time = 0
        self._sigma = 0
        self.gradient_decay = kwargs.get("gradient_decay", default_gradient_decay)
        self.radius_decay = kwargs.get("radius_decay", default_radius_decay)
        self._shape = kwargs.get("shape")
        self.demand("input", "shape")

    @property
    def shape(self):
        return self._shape

    @shape.setter
    def shape(self, value):
        self._shape = value

    @property
    def gravity_radius(self):
        return self.radius_decay(self.time) * self._sigma

    @property
    def gradient_multiplier(self):
        return self.gradient_decay(self.time)

    def _get_weights_magnitude(self):
        d = self.input.max_supposed * self._sample_length
        return 9.0 / d

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        if self.weights_transposed:
            raise NotImplementedError("transposed SOM weights are not supported")
        super().initialize(device=device, **kwargs)
        self._neurons_number = self.shape[0] * self.shape[1]
        self._sample_length = self.input.size // self.input.shape[0]
        if self.weights_stddev is None:
            self.weights_stddev = min(self._get_weights_magnitude(), 0.05)
        if not self.weights:
            w = numpy.zeros((self._neurons_number, self._sample_length),
                            dtype=numpy.float32)
            if self.weights_filling == "uniform":
                prng.get().fill(w, -self.weights_stddev, self.weights_stddev)
            elif self.weights_filling == "gaussian":
                prng.get().fill_normal_real(w, 0, self.weights_stddev)
            else:
                raise ValueError("Invalid weights filling %s" % self.weights_filling)
            self.weights.reset(w)
        elif self.weights.shape != (self._neurons_number, self._sample_length):
            raise ValueError("weights shape mismatch")
        self.winners.reset(numpy.zeros(self._neurons_number, numpy.int32))
        batch = self.input.shape[0]
        self.argmins.reset(numpy.zeros(batch, dtype=numpy.int32))
        sz = self._neurons_number
        rows = int(numpy.round(numpy.sqrt(sz)))
        cols = sz // rows + (1 if sz % rows else 0)
        coords = numpy.zeros((sz, 2), dtype=numpy.float32)
        x_step = 2.0 / (cols - 1) if cols > 1 else 0
        y_step = 2.0 / (rows - 1) if rows > 1 else 0
        offs = 0
        for r in range(rows):
            x = -1.0 + (x_step * 0.5 if r & 1 else 0)
            for _c in range(cols):
                if offs < sz:
                    coords[offs] = (x, -1.0 + r * y_step)
                offs += 1
                x += x_step
        self._coords.reset(coords)
        self._sigma = float(coords.max() - coords.min()) * 1.42
        self.init_vectors(self.input, self.weights, self.winners, self.argmins,
                          self._coords)
        return None

    def numpy_run(self):
        self.time += 1
        sigma = self.gravity_radius
        gmult = self.gradient_multiplier
        self.input.map_read()
        self.weights.map_write()
        self.winners.map_write()
        self.argmins.map_invalidate()
        x = self.input.matrix.astype(self.weights.dtype)
        w = self.weights.mem
        d = (x * x).sum(1)[:, None] - 2.0 * x.dot(w.T) + (w * w).sum(1)[None, :]
        win = d.argmin(axis=1)
        self.argmins.mem[:] = win
        numpy.add.at(self.winners.mem, win, 1)
        c = self._coords.mem
        dc = ((c[:, None, :] - c[None, win, :]) ** 2).sum(axis=2)      # [neurons, batch]
        gravity = numpy.exp(dc / (-2 * sigma * sigma))
        grad = gravity.dot(x) - gravity.sum(axis=1)[:, None] * w
        w += grad * gmult

    def cuda_run(self):
        self.time += 1
        x = self.input.dev
        if x.dtype != self.weights.dev.dtype:
            x = x.float()
        x = x.view(x.shape[0], -1)
        w = self.weights.dev
        split = som_winners_device(self, x, w, self.argmins.dev_out, self.winners.dev)
        self.winners.dev_written()
        if split is None:
            self.ext_.som_update(x, w, self._coords.dev, self.argmins.dev,
                                 float(self.gravity_radius), float(self.gradient_multiplier))
        else:
            som_update_device(self, x, w, float(self.gravity_radius),
                              float(self.gradient_multiplier))
        self.weights.dev_written()


class KohonenDecision(TrivialDecision):
    """Stops SOM training when the weights stop moving (``weights_min_diff``)."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.weights_mem = numpy.empty((0, 0), dtype=numpy.float32)
        self._prev_weights = numpy.empty((0, 0), dtype=numpy.float32)
        self.winners_mem = numpy.empty((0,), dtype=numpy.int32)
        self.weights_min_diff = kwargs.get("weights_min_diff", 0)
        self.demand("weights", "winners")

    @property
    def weights_diff(self):
        if self.weights_mem.size * self._prev_weights.size == 0:
            return numpy.inf
        return float(numpy.linalg.norm(self.weights_mem - self._prev_weights))

    def on_training_finished(self):
        self.weights.map_read()
        self.winners.map_write()
        self._prev_weights = self.weights_mem.copy()
        self.weights_mem = self.weights.mem.copy()
        self.winners_mem = self.winners.mem.copy()
        self.winners.mem[:] = 0
        self.winners.unmap()

    def train_improve_condition(self):
        if self.weights_diff < self.weights_min_diff:
            return True
        return super().train_improve_condition()

    def stop_condition(self):
        return self.weights_diff < self.weights_min_diff

    def fill_statistics(self, stats):
        stats.append("weights diff: %f" % self.weights_diff)


class KohonenValidator(Unit):
    """Maps winning neurons to real categories (greedy maximal assignment)."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.demand("input", "minibatch_indices", "minibatch_size", "samples_by_label",
                    "labels_mapping", "reversed_labels_mapping", "shape")
        self.accumulated_input = []
        self._fitness = 0
        self._fitness_by_label = {}
        self._fitness_by_neuron = []
        self._result = {}
        self._need_validate = False

    def init_unpickled(self):
        super().init_unpickled()
        self._lock_ = threading.Lock()

    @property
    def neurons_count(self):
        return self.shape[0] * self.shape[1]

    def initialize(self, **kwargs):
        del self.accumulated_input[:]
        self.accumulated_input.extend(set() for _ in range(self.neurons_count))
        self._fitness = 0
        self._reset_result()
        self._fitness_by_label = {label: 0 for label in self.samples_by_label}
        self._fitness_by_neuron = [0] * self.neurons_count
        self._overall = sum(len(m) for m in self.samples_by_label.values())
        if self._overall <= 0:
            raise ValueError("samples_by_label is empty")
        self._need_validate = True

    def reset(self):
        for acc in self.accumulated_input:
            acc.clear()
        self._need_validate = True

    def run(self):
        self.input.map_read()
        self.minibatch_indices.map_read()
        for i in range(int(self.minibatch_size)):
            self.accumulated_input[int(self.input.mem[i])].add(
                int(self.minibatch_indices.mem[i]))
        self._need_validate = True

    result = property(lambda self: (self._validate(), self._result)[1])
    fitness = property(lambda self: (self._validate(), self._fitness)[1])
    fitness_by_label = property(lambda self: (self._validate(), self._fitness_by_label)[1])
    fitness_by_neuron = property(lambda self: (self._validate(), self._fitness_by_neuron)[1])

    def _reset_result(self):
        self._result = {label: set() for label in self.samples_by_label}

    def _validate(self):
        with self._lock_:
            if not self._need_validate:
                return
            inter = []
            for neuron in range(self.neurons_count):
                for label, members in self.samples_by_label.items():
                    inter.append((len(self.accumulated_input[neuron].intersection(members)),
                                  neuron, label))
            inter.sort(key=lambda t: (-t[0], t[1]))
            self._reset_result()
            fitted = 0
            by_label = {label: 0 for label in self.samples_by_label}
            by_neuron = [0] * self.neurons_count
            banned = set()
            for fit, neuron, label in inter:
                if fit <= 0 or len(banned) >= self.neurons_count:
                    break
                if neuron in banned:
                    continue
                fitted += fit
                by_label[label] += fit
                by_neuron[neuron] = fit
                self._result[label].add(neuron)
                banned.add(neuron)
            self._fitness = fitted / self._overall
            for label, members in self.samples_by_label.items():
                self._fitness_by_label[label] = by_label[label] / max(len(members), 1)
            self._fitness_by_neuron = by_neuron
            self._need_validate = False
