"""Per-minibatch learning-rate schedules.

Parity: /root/reference/lr_adjust.py (LearningRateAdjust :61, policies ``exp`` :183,
``fixed`` :201, ``step_exp`` :217, ``inv`` :236, ``arbitrary_step`` :252). The unit
rewrites ``learning_rate(_bias)`` of every registered GD unit each minibatch; on
H100 the GD units mirror those scalars into a device vector (``sync_hyper``), so
captured CUDA graphs keep replaying while the schedule moves.
"""
from __future__ import annotations

from math import floor

import numpy

from ..core.registry import make_registry
from ..core.units import Unit
from ..ops.nn_units import GradientDescentBase

LRAdjustPolicyRegistry = make_registry("lradjustpolicy")
LRAdjustPolicyRegistry.lradjustpolicy = LRAdjustPolicyRegistry.registry


class PolicyBase(object, metaclass=LRAdjustPolicyRegistry):
    MAPPING = None

    def __init__(self, lr_to_adjust, **kwargs):
        self.base_lr = kwargs.get("base_lr", lr_to_adjust)


class ExpPolicy(PolicyBase):
    """LR = LR_base · γ^(a·iter)."""
    MAPPING = "exp"

    def __init__(self, lr_to_adjust, **kwargs):
        super().__init__(lr_to_adjust, **kwargs)
        self.gamma = kwargs["gamma"]
        self.a_ratio = kwargs["a_ratio"]

    def __call__(self, itr):
        return self.base_lr * (self.gamma ** (self.a_ratio * itr))


class FixedAjustPolicy(PolicyBase):
    """LR = LR_base."""
    MAPPING = "fixed"

    def __call__(self, itr):
        return self.base_lr


class StepExpPolicy(PolicyBase):
    """LR = LR_base · γ^floor(iter/step)."""
    MAPPING = "step_exp"

    def __init__(self, lr_to_adjust, **kwargs):
        super().__init__(lr_to_adjust, **kwargs)
        self.gamma = kwargs["gamma"]
        self.step = kwargs["step"]

    def __call__(self, itr):
        return self.base_lr * (self.gamma ** floor(float(itr) / float(self.step)))


class InvAdjustPolicy(PolicyBase):
    """LR = LR_base · (1 + γ·iter)^(−pow)."""
    MAPPING = "inv"

    def __init__(self, lr_to_adjust, **kwargs):
        super().__init__(lr_to_adjust, **kwargs)
        self.gamma = kwargs["gamma"]
        self.pow_ratio = kwargs["pow_ratio"]

    def __call__(self, itr):
        return self.base_lr * (1.0 + self.gamma * itr) ** (-self.pow_ratio)


class ArbitraryStepPolicy(PolicyBase):
    """Piecewise-constant: ``lrs_with_lengths = [(coeff, n_iters), ...]``; 0 after."""
    MAPPING = "arbitrary_step"

    def __init__(self, lr_to_adjust, **kwargs):
        super().__init__(lr_to_adjust, **kwargs)
        lrs_with_lengths = kwargs["lrs_with_lengths"]
        if not lrs_with_lengths:
            raise ValueError("lrs_with_lengths must not be empty")
        self.bounds = []
        self.values = []
        cur = 0
        for coeff, length in lrs_with_lengths:
            if coeff * self.base_lr < 0 or length <= 0:
                raise ValueError("invalid (coeff, length) = (%s, %s)" % (coeff, length))
            cur += length
            self.bounds.append(cur)
            self.values.append(coeff * self.base_lr)

    def __call__(self, itr):
        for b, v in zip(self.bounds, self.values):
            if itr < b:
                return v
        return 0.0


class LearningRateAdjust(Unit):
    """Link it so that it runs every TRAIN minibatch (after the GD units)."""

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self._gd_units = []
        self._minibatches_count = 0
        self.lr_policy_name = kwargs.get("lr_policy_name", None)
        self.bias_lr_policy_name = kwargs.get("bias_lr_policy_name", None)
        self.lr_parameters = dict(kwargs.get("lr_parameters", {}) or {})
        self.bias_lr_parameters = dict(kwargs.get("bias_lr_parameters", {}) or {})
        self.already_get_base_lr = False
        self.base_lr = {}
        self.base_lr_bias = {}
        self._policies = {}

    def add_gd_unit(self, gd_unit):
        if not isinstance(gd_unit, GradientDescentBase):
            raise TypeError("gd_unit must be a GradientDescentBase")
        self.gate_skip = gd_unit.gate_skip
        self._gd_units.append(gd_unit)

    def _policy(self, key, name, base, params):
        pol = self._policies.get(key)
        if pol is None:
            try:
                cls = LRAdjustPolicyRegistry.registry[name]
            except KeyError:
                raise ValueError("Unknown LR policy %r" % name)
            pol = self._policies[key] = cls(base, **params)
        return pol

    def adjust_learning_rate(self, key, lr_to_adjust, name, params):
        if name is None:
            return None
        return float(self._policy(key, name, lr_to_adjust, params)(
            self._minibatches_count))

    def initialize(self, **kwargs):
        pass

    def run(self):
        if self.is_slave:
            return
        if not self.already_get_base_lr:
            for i, gd in enumerate(self._gd_units):
                self.base_lr[i] = gd.learning_rate
                self.base_lr_bias[i] = gd.learning_rate_bias
            self.already_get_base_lr = True
        # layers that share a base rate share the schedule value: evaluate each distinct
        # (policy, base) once per minibatch instead of once per layer (this unit runs on the
        # host between two graph launches every step)
        memo = {}
        wname, bname = self.lr_policy_name, self.bias_lr_policy_name
        for i, gd in enumerate(self._gd_units):
            if wname is not None:
                base = self.base_lr[i]
                lr = memo.get((0, base))
                if lr is None:
                    lr = memo[(0, base)] = self.adjust_learning_rate(
                        ("w", base), base, wname, self.lr_parameters)
                gd.learning_rate = lr
            if bname is not None:
                base = self.base_lr_bias[i]
                lrb = memo.get((1, base))
                if lrb is None:
                    lrb = memo[(1, base)] = self.adjust_learning_rate(
                        ("b", base), base, bname, self.bias_lr_parameters)
                gd.learning_rate_bias = lrb
        self._minibatches_count += 1

    # IDistributable
    def generate_data_for_slave(self, slave=None):
        return None

    def generate_data_for_master(self):
        return True

    def apply_data_from_master(self, data):
        pass

    def apply_data_from_slave(self, data, slave=None):
        if not bool(self.gate_block) and not bool(self.gate_skip):
            self.run()

    def drop_slave(self, slave=None):
        pass
