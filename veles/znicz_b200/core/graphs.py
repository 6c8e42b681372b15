"""CUDA-graph capture of a chain of accelerated units.

The reference drives >100 tiny kernel launches per minibatch from python
(SURVEY §3.3). On H100 the python unit graph still decides *what* runs each
minibatch, but a chain of units (forwards+evaluator, or all GD units) is captured
once per gate configuration into a CUDA graph and replayed:

* ``cuda_prepare()`` of every unit runs on the host before each replay (uploads of
  runtime scalars: batch size, learning rates, RNG counters) — the kernels read
  those from HBM, so the captured graph never needs re-capturing;
* Array coherence is preserved: arrays that the captured kernels read are uploaded
  first if the host dirtied them, and arrays they wrote are marked device-owned
  after every replay.

Segments degrade to eager execution (same kernels, python-launched) for the first
``warmup`` executions and whenever capture is disabled.
"""
from __future__ import annotations

from . import memory as _memory


class _Recorder(object):
    def __init__(self):
        self.reads = []
        self.writes = []

    def read(self, arr):
        if arr not in self.reads:
            self.reads.append(arr)

    def write(self, arr):
        if arr not in self.writes:
            self.writes.append(arr)


_active_recorder = None


def recorder():
    return _active_recorder


class _Captured(object):
    __slots__ = ("graph", "reads", "writes", "n_kernels")


def _launch_counters():
    from ..kernels import api
    return api.counters


class GraphSegment(object):
    def __init__(self, name, units, key_fn=None, warmup=2, enabled=True, prelude=None):
        self.name = name
        self.units = list(units)
        # device-only callables run at the head of the segment (captured with it), e.g. the
        # loader's minibatch gather kernel: one eager launch and one graph boundary less per step
        self.prelude = list(prelude or [])
        # Train-step fusion: ``tail`` is a later segment (the backward chain) that may be run
        # together with this one as ONE graph when ``fuse_fn()`` says nothing on the host can
        # intervene between the two this iteration (steady-state TRAIN minibatch, not the last of
        # its epoch): one graph launch per training step instead of two.
        self.tail = None
        self.fuse_fn = None
        self.head = None             # set on the tail by fuse_with()
        self.iteration = 0           # executions of this segment (stamps the tail's skip mark)
        self._skip_iter = -1
        self.fused_replays = 0
        self.key_fn = key_fn or (lambda: 0)
        self.warmup = warmup
        self.enabled = enabled
        self._graphs = {}
        self._runs = {}
        self._done_for = None
        self.replays = 0
        self.eager_runs = 0
        for u in self.units:
            u.__dict__["segment_"] = self
        self.express = self._is_linear_chain()

    def _is_linear_chain(self):
        """True when the member units form a plain chain (each one's only successor is the next
        member, whose only predecessor it is). The first member executes the whole segment, so
        the scheduler may then continue at the LAST member's successors instead of walking ~12
        no-op units through queue, gates and timers (3 us each; the end-to-end CIFAR step was
        host-bound by exactly that)."""
        us = self.units
        for a, b in zip(us, us[1:]):
            if list(a.links_to) != [b] or list(b.links_from) != [a]:
                return False
        return len(us) > 1

    def detach(self):
        for u in self.units:
            u.__dict__.pop("segment_", None)

    # called from Unit._run_timed in place of unit.run()
    def run_unit(self, unit):
        if unit is self.units[0]:
            self.execute()
        # other members were executed as part of the segment this iteration

    def fuse_with(self, tail, fuse_fn):
        self.tail, self.fuse_fn = tail, fuse_fn
        tail.head = self

    def _eager(self, units=None):
        for fn in self.prelude:
            fn()
        for u in (units or self.units):
            u._backend_run_()
        self.eager_runs += 1

    def execute(self):
        global _active_recorder
        import torch
        if self.head is not None and self._skip_iter == self.head.iteration:
            self._skip_iter = -1     # already executed this iteration by the head segment
            return
        self.iteration += 1
        units = self.units
        key = self.key_fn()
        tail = self.tail
        if tail is not None and tail.enabled and self.enabled and self.fuse_fn() and \
                self._runs.get(key, 0) >= self.warmup and tail._runs.get(key, 0) >= tail.warmup:
            # both halves are past their eager warm-up: run them as one graph
            units = self.units + tail.units
            key = ("fused", key)
            tail._skip_iter = self.iteration
            self.fused_replays += 1
        for u in units:
            u.cuda_prepare()
        cap = self._graphs.get(key)
        if cap is not None:
            for a in cap.reads:
                if a._state == _memory._MAPPED_WRITE:
                    a.unmap()
            cap.graph.replay()
            for a in cap.writes:
                a._state = _memory._UNMAPPED
            self.replays += 1
            _launch_counters()["launches"] += cap.n_kernels
            return
        n = self._runs.get(key, 0)
        self._runs[key] = n + 1
        fused = units is not self.units
        if not fused and (not self.enabled or n < self.warmup):
            self._eager()
            return
        # capture
        rec = _Recorder()
        counters = _launch_counters()
        n0 = counters["launches"]
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        _active_recorder = rec
        try:
            # make every input current *before* capture (H2D copies are not captured)
            with torch.cuda.graph(g):
                for fn in self.prelude:
                    fn()
                for u in units:
                    u._backend_run_()
        finally:
            _active_recorder = None
        cap = _Captured()
        cap.graph = g
        cap.reads = rec.reads
        cap.writes = rec.writes
        cap.n_kernels = counters["launches"] - n0
        self._graphs[key] = cap
        g.replay()   # the capture pass did not execute anything
        for a in cap.writes:
            a._state = _memory._UNMAPPED
        self.replays += 1
