"""Graph-level activation fusion for the CUDA backend.

The reference configs spell activations as separate layers (``conv`` → ``activation_str``,
``max_pooling`` → ``activation_str`` in cifar_caffe_config.py:86-144); the reference then
runs one elementwise kernel per activation in each direction. On H100 these kernels are
pure HBM round trips, so before the units are initialised this pass folds every
*stand-alone* tanh / softplus / strict-ReLU / sigmoid activation into its producer:

  forward   the producer (conv / fully connected with linear activation, max / maxabs / avg
            pooling) applies f in its kernel epilogue; the activation unit aliases its
            ``output`` to its ``input`` and launches nothing;
  backward  the producer's GD unit multiplies the incoming error by f'(y) in the kernel it
            runs anyway (``err_act_colsum`` for conv/FC, the pooling backward gather); the
            activation's GD unit aliases ``err_input`` to ``err_output``.

All four functions have derivatives expressible through the output y alone, so aliasing
input and output loses nothing.

A second pass (:func:`fuse_backward_derivatives`) moves the ``err_output *= f'(y)`` multiply of a
convolutional layer into the backward kernel of the pooling layer above it (which writes that
very ``err_output`` and has y as its own input), and lets the wgmma weight-gradient kernel
deliver the bias gradient as an extra product row: the conv layer's separate pass over
``err_output`` (one launch per layer per step in the reference, gd_conv.py:645-750) disappears. The unit graph, the layer DSL, snapshots and
``package_export`` are unchanged — only launches disappear. ``root.common.engine.
fuse_activations = False`` switches the pass off.
"""
from __future__ import annotations

from ..core.config import root
from ..ops.activation import ActivationBackward, ActivationForward
from ..ops.all2all import All2All, All2AllSoftmax
from ..ops.conv import Conv
from ..ops.pooling import AvgPooling, MaxAbsPooling, MaxPooling

FUSABLE_CODES = (1, 2, 3, 4)       # tanh, softplus, strict relu, sigmoid


def _producer_ok(p):
    if isinstance(p, All2AllSoftmax):
        return False
    if isinstance(p, (Conv, All2All)):
        return p.ACT == 0 and not getattr(p, "weights_transposed", False)
    return type(p) in (MaxPooling, MaxAbsPooling, AvgPooling)


def clear(workflow):
    for u in list(workflow.forwards) + [g for g in workflow.gds if g is not None]:
        u.__dict__.pop("in_deriv_act_", None)
        u.__dict__.pop("deriv_upstream_", None)
        if "fused_act_" in u.__dict__:
            u.__dict__["fused_act_"] = 0
        if getattr(u, "fused_into_", None) is not None:
            u.fused_into_ = None


def fuse_activations(workflow, device):
    """Returns the number of activation layers folded away."""
    clear(workflow)
    if device is None or not device.is_cuda or \
            not root.common.engine.get("fuse_activations", True):
        return 0
    fwds = list(workflow.forwards)
    gds = [g for g in workflow.gds if g is not None]
    # GD units are matched through ``forward_unit`` (layers without a GD, e.g. zero_filter,
    # make the two lists differ in length)
    gd_of = {id(g.forward_unit): g for g in gds if getattr(g, "forward_unit", None) is not None}
    n = 0
    for i in range(1, len(fwds)):
        a, p = fwds[i], fwds[i - 1]
        if not isinstance(a, ActivationForward) or a.CODE not in FUSABLE_CODES:
            continue
        if not _producer_ok(p) or getattr(a, "force_numpy", False) or \
                getattr(p, "force_numpy", False):
            continue
        if gds:
            ga, gp = gd_of.get(id(a)), gd_of.get(id(p))
            if not isinstance(ga, ActivationBackward) or gp is None or \
                    getattr(gp, "force_numpy", False) or getattr(ga, "force_numpy", False):
                continue
            gp.__dict__["fused_act_"] = a.CODE
            ga.fused_into_ = gp
        p.__dict__["fused_act_"] = a.CODE
        a.fused_into_ = p
        n += 1
    return n


def fuse_backward_derivatives(workflow, device):
    """conv (activation f, own or fused) → [fused activation unit] → pooling, LRN or another conv:
    that layer's GD multiplies its err_input by f'(its input) in the kernel it runs anyway (pooling /
    LRN backward, the dgrad epilogue); the conv GD skips its derivative pass.
    Must run after :func:`fuse_activations`. Returns the number of conv layers relieved."""
    if device is None or not device.is_cuda or \
            not root.common.engine.get("fuse_activations", True):
        return 0
    from ..ops.gd_conv import GradientDescentConv
    from ..ops.gd_pooling import GDPooling
    from ..ops.normalization import LRNormalizerBackward
    fwds = list(workflow.forwards)
    gds = [g for g in workflow.gds if g is not None]
    gd_of = {id(g.forward_unit): g for g in gds if getattr(g, "forward_unit", None) is not None}
    n = 0
    for i, p in enumerate(fwds):
        if not isinstance(p, Conv) or getattr(p, "force_numpy", False):
            continue
        gp = gd_of.get(id(p))
        if not isinstance(gp, GradientDescentConv) or getattr(gp, "force_numpy", False):
            continue
        act = int(gp.__dict__.get("fused_act_", 0) or 0) or int(getattr(gp, "ACT", 0) or 0)
        if act not in FUSABLE_CODES:
            continue
        from ..ops.weights_zerofilling import ZeroFiller
        j = i + 1
        while j < len(fwds) and (getattr(fwds[j], "fused_into_", None) is p or
                                 isinstance(fwds[j], ZeroFiller)):
            j += 1      # activation units folded into the conv; weight-mask units carry no data
        if j >= len(fwds):
            continue
        c = fwds[j]
        gc = gd_of.get(id(c))
        conv_ok = isinstance(gc, GradientDescentConv) and not gc.err_input_beta and \
            not getattr(c, "weights_transposed", False)      # dgrad epilogue folds it (bf16 path)
        if not (isinstance(gc, (GDPooling, LRNormalizerBackward)) or conv_ok) or \
                getattr(gc, "force_numpy", False) or \
                getattr(c, "force_numpy", False) or not gc.need_err_input:
            continue
        gc.__dict__["in_deriv_act_"] = act
        gp.__dict__["deriv_upstream_"] = True
        n += 1
    return n


def fuse_evaluator(workflow, device):
    """softmax layer served by the few-output FC kernel → EvaluatorSoftmax: the evaluator's work
    rides in the FC launch (kernels/api.py::fc_forward checks the remaining run-time conditions
    and falls back to the stand-alone kernel when they do not hold). Returns 1 if armed."""
    for f in workflow.forwards:
        f.__dict__.pop("fused_eval_", None)
    if device is None or not device.is_cuda or \
            not root.common.engine.get("fuse_activations", True) or not workflow.forwards:
        return 0
    from .evaluator import EvaluatorSoftmax
    last = workflow.forwards[-1]
    ev = getattr(workflow, "evaluator", None)
    if not isinstance(last, All2AllSoftmax) or type(ev) is not EvaluatorSoftmax or \
            getattr(last, "force_numpy", False) or getattr(ev, "force_numpy", False):
        return 0
    last.__dict__["fused_eval_"] = ev
    return 1
