"""Device-timed ms per training step with each solver on every layer.

Builds the flagship workflows of bench.py (CIFAR caffe net, AlexNet), puts momentum plus the
chosen solver on every GD unit, runs the graph-capture and warm-up steps, then times K steps
between CUDA events. The card's name and power limit are printed with the numbers.

usage: python tests/bench_solvers.py [--models cifar_caffe,alexnet] [--steps 50] [--warmup 10]
prints one JSON line per (model, solver).
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

SOLVERS = {"momentum": set(), "adagrad": {"adagrad"}, "adadelta": {"adadelta"},
           "fast": {"fast"}, "adagrad+fast": {"adagrad", "fast"}}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def time_steps(model, solver, steps, warmup, n_train):
    import torch
    import bench
    from veles.znicz_b200.core.config import root
    wf = bench.build_workflow(False, "bf16", True, n_train, model)
    for u in wf.gds:
        if u is not None and hasattr(u, "solvers"):
            u.solvers = {"momentum"} | SOLVERS[solver]
    wf.initialize(device="cuda")
    gds = [u for u in wf.gds if u is not None and getattr(u, "weights", None)]
    on_cuda = all(u.on_cuda for u in gds)
    wf.run(iterations=bench.GRAPH_CAPTURE_STEPS + warmup)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    wf.run(iterations=steps)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res = {"model": model, "solver": solver, "ms_per_step": round(ms, 4), "steps": steps,
           "all_gd_on_cuda": on_cuda, "fused_step": wf.fused_step_ is not None,
           "compute": root.common.engine.compute_type}
    del wf
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="cifar_caffe,alexnet")
    ap.add_argument("--solvers", default=",".join(SOLVERS))
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--n-train", type=int, default=50000)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_solvers.py needs a CUDA device")
    gpu = card()
    for model in args.models.split(","):
        for solver in args.solvers.split(","):
            r = time_steps(model, solver, args.steps, args.warmup, args.n_train)
            r["gpu"] = gpu
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
