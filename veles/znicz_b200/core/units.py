"""Unit: the node of the dataflow/control graph.

Designed fresh for the absent Veles core (``veles.units``); the contract is what
the reference consumes (SURVEY §8 "Unit protocol"; usages
/root/reference/standard_workflow_base.py:151-158,396-452,
/root/reference/nn_units.py:380, /root/reference/all2all.py:102-104):

* control edges ``a.link_from(b)``; data aliases ``a.link_attrs(b, "x", ("mine","theirs"))``
* gates ``gate_block`` / ``gate_skip`` / ``ignores_gate`` are mutable :class:`Bool` s
* ``demand("input")`` declares attributes that must be non-None before ``initialize``
* ``initialize()`` may return True = "not ready yet, call me again" (two-stage init)
* pickle rule: attributes whose name ends with ``_`` are transient and are rebuilt
  by ``init_unpickled()``

Scheduling is a deterministic single-threaded FIFO walk owned by the Workflow
(one CUDA stream is the real executor on the H100 path; python only decides
*what* is enqueued), not the reference core's thread pool.
"""
from __future__ import annotations

import os
import time
import uuid

from .config import root
from .logger import Logger
from .mutable import Bool, LinkableAttribute
from .registry import UnitRegistry


def nothing(*args, **kwargs):
    return None


class NotInitializedError(RuntimeError):
    pass


_NVTX = []


def _nvtx():
    """torch.cuda.nvtx when CUDA is usable, else None (``root.common.trace.nvtx`` or
    ZNICZ_NVTX=1 switch the per-unit ranges on)."""
    if not _NVTX:
        mod = None
        try:
            import torch
            if torch.cuda.is_available():
                mod = torch.cuda.nvtx
        except Exception:        # pragma: no cover
            mod = None
        _NVTX.append(mod)
    return _NVTX[0]


class Unit(Logger, metaclass=UnitRegistry):
    hide_from_registry = True
    # wall-clock accounting (parity with the core's per-unit timers)
    timers = {}

    def __init__(self, workflow, **kwargs):
        self.name = kwargs.get("name") or type(self).__name__
        self.view_group = kwargs.get("view_group")
        self._links_from = {}
        self._links_to = {}
        self._gate_block = Bool(False)
        self._gate_skip = Bool(False)
        self._ignores_gate = Bool(kwargs.get("ignores_gate", False))
        self._demanded = []
        self._is_initialized = False
        self._stopped = False
        self._run_calls = 0
        self._run_time = 0.0
        self._id = str(uuid.uuid4())
        self._workflow = None
        self.init_unpickled()
        self.workflow = workflow

    # -- transient state ------------------------------------------------------
    def init_unpickled(self):
        """(Re)create every ``*_`` attribute. Called by __init__ and after unpickle."""
        pass

    def __getstate__(self):
        state = {k: v for k, v in self.__dict__.items() if not k.endswith("_")}
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)
        for name, (other, other_name, two_way) in list(
                self.__dict__.get("_linked_attrs", {}).items()):
            LinkableAttribute.install(self, name, other, other_name, two_way)
        self.init_unpickled()

    # -- identity -------------------------------------------------------------
    @property
    def id(self):
        return self._id

    def __repr__(self):
        return "<%s \"%s\">" % (type(self).__name__, self.name)

    # -- workflow membership --------------------------------------------------
    @property
    def workflow(self):
        return self._workflow

    @workflow.setter
    def workflow(self, value):
        if self._workflow is not None and self._workflow is not value:
            self._workflow.del_ref(self)
        self._workflow = value
        if value is not None and hasattr(value, "add_ref"):
            value.add_ref(self)

    @property
    def launcher(self):
        wf = self._workflow
        while wf is not None and not getattr(wf, "_is_launcher", False):
            wf = getattr(wf, "workflow", None)
        return wf

    @property
    def is_standalone(self):
        wf = self._workflow
        return True if wf is None else wf.is_standalone

    @property
    def is_master(self):
        wf = self._workflow
        return False if wf is None else wf.is_master

    @property
    def is_slave(self):
        wf = self._workflow
        return False if wf is None else wf.is_slave

    @property
    def testing(self):
        wf = self._workflow
        return False if wf is None else getattr(wf, "testing", False)

    # -- gates ----------------------------------------------------------------
    def _set_gate(self, name, value):
        if not isinstance(value, Bool):
            value = Bool(value)
        self.__dict__[name] = value

    gate_block = property(lambda self: self._gate_block,
                          lambda self, v: self._set_gate("_gate_block", v))
    gate_skip = property(lambda self: self._gate_skip,
                         lambda self, v: self._set_gate("_gate_skip", v))
    ignores_gate = property(lambda self: self._ignores_gate,
                            lambda self, v: self._set_gate("_ignores_gate", v))

    # -- control links --------------------------------------------------------
    @property
    def links_from(self):
        return self._links_from

    @property
    def links_to(self):
        return self._links_to

    def link_from(self, *units):
        for u in units:
            if u is self:
                raise ValueError("A unit may not be linked from itself")
            self._links_from[u] = False
            u._links_to[self] = False
        return self

    def unlink_from(self, *units):
        for u in units:
            self._links_from.pop(u, None)
            u._links_to.pop(self, None)
        return self

    def unlink_before(self):
        self.unlink_from(*list(self._links_from))
        return self

    def unlink_after(self):
        for dst in list(self._links_to):
            dst.unlink_from(self)
        return self

    def unlink_all(self):
        self.unlink_before()
        self.unlink_after()
        return self

    def insert_after(self, *units):
        """Re-route: everything that followed ``units`` now follows self."""
        for u in units:
            for dst in list(u._links_to):
                dst.unlink_from(u)
                dst.link_from(self)
        self.link_from(*units)
        return self

    def dependent_units(self, with_open_gate=False):
        seen = {self}
        order = [self]
        i = 0
        while i < len(order):
            for dst in order[i]._links_to:
                if dst not in seen:
                    seen.add(dst)
                    order.append(dst)
            i += 1
        return order

    # -- data links -----------------------------------------------------------
    def link_attrs(self, other, *args, **kwargs):
        two_way = kwargs.get("two_way", False)
        for arg in args:
            if isinstance(arg, (tuple, list)):
                mine, theirs = arg
            else:
                mine = theirs = arg
            if not hasattr(other, theirs):
                # allow linking to attrs created later; still forward lazily
                pass
            LinkableAttribute.install(self, mine, other, theirs, two_way)
        return self

    def unlink_attrs(self, *names):
        links = self.__dict__.get("_linked_attrs", {})
        for n in names:
            links.pop(n, None)
        return self

    def has_linked_attr(self, name):
        return name in self.__dict__.get("_linked_attrs", {})

    def demand(self, *names):
        for n in names:
            if n not in self._demanded:
                self._demanded.append(n)
            if not self.has_linked_attr(n) and n not in self.__dict__:
                try:
                    object.__getattribute__(self, n)
                except AttributeError:
                    self.__dict__[n] = None

    def undemand(self, *names):
        for n in names:
            if n in self._demanded:
                self._demanded.remove(n)

    @property
    def demanded(self):
        return list(self._demanded)

    def verify_demands(self):
        missing = []
        for n in self._demanded:
            try:
                v = getattr(self, n)
            except AttributeError:
                v = None
            if v is None:
                missing.append(n)
        return missing

    def verify_interface(self, iface):  # zope-free duck typing
        for m in getattr(iface, "__required__", ()):
            if not hasattr(self, m):
                raise NotImplementedError("%s lacks %s" % (self, m))

    # -- life cycle -----------------------------------------------------------
    @property
    def is_initialized(self):
        return self._is_initialized

    @property
    def stopped(self):
        return self._stopped

    @stopped.setter
    def stopped(self, value):
        self._stopped = bool(value)

    def initialize(self, **kwargs):
        """Override. Return True to be called again after the other units."""
        return None

    def _initialize_checked(self, **kwargs):
        missing = self.verify_demands()
        if missing:
            return missing
        self._stopped = False
        res = self.initialize(**kwargs)
        if not res:
            self._is_initialized = True
        return res

    def run(self):
        pass

    def stop(self):
        self._stopped = True

    # -- scheduling -----------------------------------------------------------
    def open_gate(self, src):
        if bool(self._ignores_gate):
            return True
        lf = self._links_from
        if src in lf:
            lf[src] = True
        if not all(lf.values()):
            return False
        for k in lf:
            lf[k] = False
        return True

    def _check_gate_and_run(self, src):
        if not self.open_gate(src):
            return
        if bool(self._gate_block):
            return
        if not bool(self._gate_skip):
            seg = self.__dict__.get("segment_")
            if seg is not None and seg.units[0] is not self and not Unit._trace_any:
                # member of a CUDA-graph segment whose first unit replayed the whole segment this
                # iteration: nothing to run, nothing to time (30 of these per training step)
                self._run_calls += 1
            else:
                self._run_timed()
                if seg is not None and seg.express and not Unit._trace_any and \
                        Unit._express_segments:
                    seg.units[-1].run_dependent()      # the chain in between has been executed
                    return
        self.run_dependent()

    # per-run tracing switches, refreshed by Workflow.run() (a Config lookup per unit run cost
    # ~10 us per training step)
    _trace_run = False
    _trace_nvtx = False
    _trace_any = False
    _express_segments = True

    @staticmethod
    def refresh_trace_flags():
        Unit._trace_run = bool(root.common.trace.run)
        Unit._trace_nvtx = bool(root.common.trace.get("nvtx", False))
        Unit._trace_any = Unit._trace_run or Unit._trace_nvtx
        Unit._express_segments = bool(root.common.engine.get("express_segments", True)) and \
            os.environ.get("ZNICZ_EXPRESS", "1") != "0"

    def _run_timed(self):
        if not self._is_initialized:
            raise NotInitializedError("%s is not initialized" % self)
        if Unit._trace_run:
            self.debug("run")
        nvtx = _nvtx() if Unit._trace_nvtx else None
        if nvtx is not None:
            nvtx.range_push(self.name)      # one range per unit run: shows up in nsys / ncu --nvtx
        t0 = time.perf_counter()
        try:
            seg = self.__dict__.get("segment_")
            if seg is not None:
                seg.run_unit(self)
            else:
                self.run()
        finally:
            if nvtx is not None:
                nvtx.range_pop()
        self._run_time += time.perf_counter() - t0
        self._run_calls += 1

    def run_dependent(self):
        wf = self._workflow
        q = wf._queue_ if wf is not None else None
        if q is None:
            for dst in list(self._links_to):
                dst._check_gate_and_run(self)
        else:
            for dst in self._links_to:
                q.append((self, dst))

    # -- timing report ----------------------------------------------------------
    @property
    def average_run_time(self):
        return self._run_time / self._run_calls if self._run_calls else 0.0

    @property
    def total_run_time(self):
        return self._run_time


class TrivialUnit(Unit):
    hide_from_registry = True


class IUnit(object):
    __required__ = ("initialize", "run")


class UnitCommandLineArgumentsRegistry(UnitRegistry):
    """Metaclass kept for API parity: per-unit CLI arguments
    (/root/reference/nn_units.py:86). Units may define ``init_parser(parser)``."""
    pass
