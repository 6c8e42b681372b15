"""Sequence classification with the whole-sequence LSTM unit (north-star config 5:
"LSTM unit sequence workflow").

The reference builds sequences by chaining single-step ``LSTM`` sub-workflows and sharing their
weights (/root/reference/lstm.py:52-143, BPTT through ``GDLSTM.err_prev_output/err_prev_memory``
:263,304); here the ``lstm_seq`` layer (ops/lstm_seq.py) runs all time steps of a minibatch
[batch][T][features] inside one unit - one wgmma GEMM + one fused cell kernel per step, a single
weight-gradient GEMM over the whole sequence - followed by a softmax classifier on the last
hidden state.
"""
from __future__ import annotations

from ..core.workflow import DummyLauncher
from ..workflow.standard_workflow import StandardWorkflow


def layers(hidden=256, n_classes=10, lr=0.05):
    gd = {"learning_rate": lr, "learning_rate_bias": lr, "gradient_moment": 0.9,
          "gradient_moment_bias": 0.9, "weights_decay": 0.0}
    return [
        {"name": "lstm", "type": "lstm_seq",
         "->": {"output_sample_shape": hidden, "weights_stddev": 0.08}, "<-": dict(gd)},
        {"name": "out", "type": "softmax",
         "->": {"output_sample_shape": n_classes, "weights_stddev": 0.05}, "<-": dict(gd)}]


def build(launcher=None, seq_len=32, features=128, hidden=256, n_classes=10,
          loader_name="synthetic_image", loader_config=None, decision_config=None,
          snapshotter_config=None, **kwargs):
    cfg = {"minibatch_size": 128, "shape": (seq_len, features), "n_classes": n_classes,
           "n_train": 4096, "n_valid": 512, "normalization_type": "none", "noise": 0.5}
    cfg.update(loader_config or {})
    return StandardWorkflow(
        launcher or DummyLauncher(), loader_name=loader_name, loader_config=cfg,
        layers=kwargs.pop("layers", None) or layers(hidden, n_classes),
        loss_function="softmax",
        decision_config=decision_config or {"max_epochs": 10, "fail_iterations": 20},
        snapshotter_config=snapshotter_config or {"prefix": "lstm_seq", "interval": 1000,
                                                  "time_interval": 1e9},
        **kwargs)
