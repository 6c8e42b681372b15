"""CD-k step time of the mnist_rbm workflow with its RBM units on the device and on the host.

The host path sets ``force_numpy`` on the Binarization, BatchWeights, GradientsCalculator and
WeightsUpdater units before ``initialize`` (``run`` is bound there): sampling, batch statistics and
the update then run in numpy with the samples and weights mapped across every step, while the
All2AllSigmoid GEMMs stay on the GPU. The two paths alternate in one process, each timed with CUDA
events around ``run(iterations=steps)`` after a warm-up; the median over the rounds is reported.

    python tools/bench_rbm.py [--steps 20] [--warmup 3] [--rounds 3] [--compute bf16]

Shapes: mnist_rbm's own (196 visibles, 1000 hidden, batch 128, CD-1) and a larger one (784
visibles, 4096 hidden, batch 512, CD-1 and CD-5). Samples are random binary patterns written to a
temporary .mat file; nothing is written to the source tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIGS = [  # (visibles, hidden, batch, cd_k)
    (196, 1000, 128, 1),
    (784, 4096, 512, 1),
    (784, 4096, 512, 5),
]


def card():
    """(name, power limit) of GPU 0, read in this run."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:                 # pragma: no cover - no nvidia-smi
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def build(tmp, v, h, batch, cd_k, host, compute):
    import scipy.io
    from veles.znicz_b200.core import prng
    from veles.znicz_b200.core.config import root
    from veles.znicz_b200.models import mnist_rbm
    from veles.znicz_b200.ops import rbm_units
    root.common.engine.compute_type = compute
    rs = numpy.random.RandomState(v + h)
    n = 4 * batch
    patterns = (rs.rand(16, v) > 0.5).astype(numpy.float32)
    path = os.path.join(tmp, "patches_%d.mat" % v)
    scipy.io.savemat(path, {"patches": patterns[rs.randint(0, 16, n)]})
    root.mnist_rbm.loader.data_path = path
    root.mnist_rbm.cd_k = cd_k
    prng.get(1).seed(1234)
    prng.get(2).seed(5678)
    wf = mnist_rbm.build(minibatch_size=batch, n_samples=n, v_size=v, h_size=h,
                         max_epochs=10 ** 9, learning_rate=0.001)
    if host:
        units = list(rbm_units._all_units(wf))
        for u in units:
            if isinstance(u, (rbm_units.Binarization, rbm_units.BatchWeights,
                              rbm_units.GradientsCalculator, rbm_units.WeightsUpdater)):
                u.force_numpy = True
    wf.initialize(device="cuda")
    return wf


def time_steps(wf, steps):
    import torch
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    wf.run(iterations=steps)
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--compute", default="bf16", choices=("bf16", "fp32"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_rbm.py needs a CUDA device")
    name, limit = card()
    print("card: %s, power limit %s, compute_type %s, %d steps x %d rounds after %d warm-up steps"
          % (name, limit, args.compute, args.steps, args.rounds, args.warmup), flush=True)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for v, h, batch, cd_k in CONFIGS:
            wfs = {p: build(tmp, v, h, batch, cd_k, p == "host", args.compute)
                   for p in ("device", "host")}
            for wf in wfs.values():
                wf.run(iterations=args.warmup)
            times = {p: [] for p in wfs}
            for _ in range(args.rounds):
                for p, wf in wfs.items():
                    times[p].append(time_steps(wf, args.steps))
            dev, host = (statistics.median(times[p]) for p in ("device", "host"))
            row = {"visible": v, "hidden": h, "batch": batch, "cd_k": cd_k,
                   "device_ms_per_step": round(dev, 4), "host_ms_per_step": round(host, 4),
                   "speedup": round(host / dev, 2), "device_runs": [round(t, 4) for t in times["device"]],
                   "host_runs": [round(t, 4) for t in times["host"]]}
            rows.append(row)
            print("V %4d H %4d batch %3d CD-%d: device %.3f ms/step, host %.3f ms/step (x%.1f)"
                  % (v, h, batch, cd_k, dev, host, host / dev), flush=True)
            del wfs
    print(json.dumps({"card": name, "power_limit": limit, "compute_type": args.compute,
                      "results": rows}))


if __name__ == "__main__":
    main()
