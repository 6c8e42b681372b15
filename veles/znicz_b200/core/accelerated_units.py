"""AcceleratedUnit: a unit with a numpy oracle path and one sm_90a path.

Fresh design for ``veles.accelerated_units`` (AcceleratedUnit, AcceleratedWorkflow,
TrivialAcceleratedUnit). The reference selects numpy/ocl/cuda per unit at run time
(/root/reference/all2all.py:52, /root/reference/conv.py:70); here ``initialize(device)``
binds ``run`` to ``numpy_run`` or ``cuda_run`` once. There is no JIT: kernels are
ahead-of-time compiled for sm_90a in ``veles.znicz_b200.kernels``.
"""
from __future__ import annotations

import numpy

from .backends import Device, NumpyDevice, get_device
from .config import root
from .memory import Array
from .units import Unit
from .workflow import Workflow


def host_dtype():
    pt = root.common.engine.get("precision_type", "float")
    return numpy.float64 if pt == "double" else numpy.float32


class AcceleratedUnit(Unit):
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        self._force_numpy = kwargs.get("force_numpy", False)
        super().__init__(workflow, **kwargs)
        self.device = None

    def init_unpickled(self):
        super().init_unpickled()
        self._backend_run_ = None
        self.ext_ = None

    @property
    def force_numpy(self):
        return self._force_numpy

    @force_numpy.setter
    def force_numpy(self, value):
        self._force_numpy = bool(value)

    @property
    def on_cuda(self):
        d = self.device
        return d is not None and d.is_cuda and not self._force_numpy

    def initialize(self, device=None, **kwargs):
        if device is None:
            device = self.device or NumpyDevice()
        elif isinstance(device, str):
            from .backends import get_device
            device = get_device(device)
        self.device = device
        if self.on_cuda:
            self.ext_ = device.ext
            self._backend_run_ = self.cuda_run
        else:
            self._backend_run_ = self.numpy_run
        return None

    def _finish_init(self):
        """Call at the end of a subclass' initialize(): backend specific setup."""
        if self.on_cuda:
            self.cuda_init()
        else:
            self.numpy_init()

    def init_vectors(self, *arrays):
        dev = self.device if self.on_cuda else None
        for a in arrays:
            if isinstance(a, Array) and a:
                a.initialize(dev)

    def unmap_vectors(self, *arrays):
        for a in arrays:
            if isinstance(a, Array) and a:
                a.unmap()

    def numpy_init(self):
        pass

    def cuda_init(self):
        pass

    def numpy_run(self):
        raise NotImplementedError("%s.numpy_run" % type(self).__name__)

    def cuda_run(self):
        raise NotImplementedError("%s.cuda_run" % type(self).__name__)

    def cuda_prepare(self):
        """Host-side, non-capturable part of a device step (scalar uploads).
        A captured graph segment calls this for every unit before replaying."""
        pass

    def run(self):
        if self._backend_run_ is None:
            raise RuntimeError("%s.run() before initialize()" % self)
        if self.ext_ is not None:
            self.cuda_prepare()
        return self._backend_run_()


class TrivialAcceleratedUnit(AcceleratedUnit):
    hide_from_registry = True

    def numpy_run(self):
        pass

    def cuda_run(self):
        pass


class AcceleratedWorkflow(Workflow):
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.device = None

    def initialize(self, device=None, **kwargs):
        if device is None or isinstance(device, str):
            device = get_device(device)
        self.device = device
        return super().initialize(device=device, **kwargs)
