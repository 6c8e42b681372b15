"""Per-kernel device-time profile of the flagship training step (bench.py's timed loop).

Builds the workflow exactly as ``bench.py`` does (CIFAR caffe-conv, bf16, CUDA graphs, the
50000-sample dataset resident on the device), runs the graph-capture steps and a warm-up, then
records ``--steps`` steady-state steps under ``torch.profiler`` with CUDA activities and prints
one row per kernel (name + grid): calls per step, mean duration and share of the kernel time of
the step. Run it on its own: tracing slows the host, so its timings are not step times.

Usage (GPU): ``python tools/step_profile.py [--steps 200] [--warmup 50] [--model cifar_caffe]
[--trace OUT.json]``
"""
import argparse
import collections
import gzip
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], stdout=subprocess.PIPE,
                              stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except Exception as exc:
        return "unknown (%s)" % type(exc).__name__


def kernel_events(trace_path):
    opener = gzip.open if trace_path.endswith(".gz") else open
    with opener(trace_path, "rt") as f:
        trace = json.load(f)
    for ev in trace.get("traceEvents", []):
        if ev.get("ph") == "X" and ev.get("cat") == "kernel":
            args = ev.get("args", {})
            yield ev["name"], tuple(args.get("grid", ())), float(ev["ts"]), float(ev["dur"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--model", default="cifar_caffe")
    ap.add_argument("--top", type=int, default=40)
    ap.add_argument("--trace", default=None, help="also keep the chrome trace at this path")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench

    if not torch.cuda.is_available():
        raise SystemExit("step_profile.py needs a GPU")
    wf = bench.build_workflow(False, "bf16", True, 50000, args.model)
    wf.initialize(device="cuda")
    wf.run(iterations=bench.GRAPH_CAPTURE_STEPS)
    wf.run(iterations=args.warmup)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        n = wf.run(iterations=args.steps)
        torch.cuda.synchronize()
    if n != args.steps:
        raise RuntimeError("ran %d steps, not %d" % (n, args.steps))
    with tempfile.TemporaryDirectory() as tmp:
        path = args.trace or os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        evs = list(kernel_events(path))
    if not evs:
        raise RuntimeError("the trace holds no kernel records")

    rows = collections.OrderedDict()
    for name, grid, _, dur in evs:
        cnt, tot = rows.get((name, grid), (0, 0.0))
        rows[(name, grid)] = (cnt + 1, tot + dur)
    busy = sum(d for _, _, _, d in evs)
    span = max(t + d for _, _, t, d in evs) - min(t for _, _, t, _ in evs)
    print("card: %s" % card())
    print("model %s, %d steps traced: %d kernel launches, kernel time %.2f us/step, "
          "first-to-last-kernel span %.2f us/step (traced; not a step time)"
          % (args.model, args.steps, len(evs), busy / args.steps, span / args.steps))
    print("| kernel | grid | calls/step | mean us | us/step | share |")
    print("|---|---|---|---|---|---|")
    ranked = sorted(rows.items(), key=lambda kv: -kv[1][1])
    for (name, grid), (cnt, tot) in ranked[:args.top]:
        print("| `%s` | %s | %.2f | %.2f | %.2f | %.1f %% |" % (
            name[:110], "x".join(str(g) for g in grid), cnt / args.steps, tot / cnt,
            tot / args.steps, 100.0 * tot / busy))
    del wf
    return 0


if __name__ == "__main__":
    sys.exit(main())
