"""Local response normalisation across channels.

Parity: /root/reference/normalization.py (LocalResponseNormalizer :49 with
``alpha=1e-4, beta=.75, k=2, n=5`` :56-59, LRNormalizerForward :97,
LRNormalizerBackward :184): ``y_i = x_i · (k + α·Σ_{j∈win(i)} x_j²)^(−β)`` and the
exact Jacobian-vector product (:224-261).

H100: a warp handles pixels with the channel vector held in registers (NHWC ⇒
one coalesced 16-byte load per 8 channels); forward/backward are one pass each.
"""
from __future__ import annotations

import numpy

from .nn_units import Forward, GradientDescentBase


class LocalResponseNormalizer(object):
    def _init_lrn(self, kwargs):
        self.alpha = kwargs.get("alpha", 0.0001)
        self.beta = kwargs.get("beta", 0.75)
        self.k = kwargs.get("k", 2)
        self.n = kwargs.get("n", 5)

    def _subsums(self, source_array, window_size):
        """For each channel: sum over its neighbour channels (window clipped)."""
        assert source_array.ndim == 4
        c = source_array.shape[3]
        half = int(window_size / 2)
        cs = numpy.concatenate(
            [numpy.zeros(source_array.shape[:3] + (1,), source_array.dtype),
             numpy.cumsum(source_array, axis=3)], axis=3)
        lo = numpy.maximum(numpy.arange(c) - half, 0)
        hi = numpy.minimum(numpy.arange(c) + half, c - 1) + 1
        return cs[..., hi] - cs[..., lo]

    # IDistributable: nothing to exchange
    def generate_data_for_slave(self, slave=None):
        return None

    def generate_data_for_master(self):
        return None

    def apply_data_from_master(self, data):
        pass

    def apply_data_from_slave(self, data, slave=None):
        pass

    def drop_slave(self, slave=None):
        pass


class LRNormalizerForward(LocalResponseNormalizer, Forward):
    MAPPING = {"norm"}

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._init_lrn(kwargs)
        self.exports.extend(("alpha", "beta", "k", "n"))

    def initialize(self, device=None, **kwargs):
        if not self.input:
            return True
        super().initialize(device=device, **kwargs)
        if len(self.input.shape) != 4:
            raise ValueError("LRN needs NHWC input")
        self.make_output(self.input.shape, self.input.dtype)
        self.output.dev_dtype = self.input.dev_dtype
        self.init_vectors(self.input, self.output)
        return None

    def numpy_run(self):
        self.output.map_invalidate()
        self.input.map_read()
        x = self.input.mem
        s = self._subsums(numpy.square(x), self.n) * self.alpha + self.k
        self.output.mem[...] = x / s ** self.beta

    def cuda_run(self):
        from ..kernels import api
        api.lrn_forward(self)


class LRNormalizerBackward(LocalResponseNormalizer, GradientDescentBase):
    MAPPING = {"norm"}

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._init_lrn(kwargs)

    def initialize(self, device=None, **kwargs):
        if not self.input or not self.err_output:
            return True
        return super().initialize(device=device, **kwargs)

    def numpy_run(self):
        self.err_input.map_invalidate()
        self.err_output.map_read()
        self.input.map_read()
        x = self.input.mem.astype(numpy.float64)
        ey = self.err_output.mem.reshape(x.shape).astype(numpy.float64)
        s = self._subsums(numpy.square(x), self.n) * self.alpha + self.k
        # dL/dx_i = ey_i·s_i^-β − 2αβ·x_i·Σ_{j: i∈win(j)} ey_j·x_j·s_j^(-β-1)
        t = ey * x * s ** (-self.beta - 1.0)
        tsum = self._subsums(t, self.n)       # window is symmetric ⇒ same index set
        eh = ey * s ** (-self.beta) - 2.0 * self.alpha * self.beta * x * tsum
        self.err_input.mem[...] = eh.reshape(self.err_input.shape)

    def cuda_run(self):
        from ..kernels import api
        api.lrn_backward(self)
