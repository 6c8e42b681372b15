"""Real-data AlexNet training throughput with the ImageNet loader's three input paths.

Generates a seeded uint8 dataset in the AlexNet config's format (256x256x3 samples, 1000
classes, a mean file), then trains ``alexnet_layers(1000)`` in bf16 with CUDA graphs, crop 227
and mirror, at each ``--batches`` size, on three arms run in the same process:

  streamed   device augmentation, rows streamed through the pinned slot (the default)
  resident   device augmentation, the sample file resident in HBM (``on_device=True``)
  host       the host path: numpy crop / mirror / mean in ``fill_minibatch``, fp32 staging,
             H2D copy and ``cast_copy`` (a subclass that overrides ``fill_minibatch``)

Every run is one epoch of ``--warmup`` + timed steps; the timed window is the last steps of the
epoch, so each arm has the same single epoch end in it. The arm order rotates over ``--repeats``.
Per arm: images/s (host clock, synchronised at both ends), the loader's host ms per minibatch
(assembly + enqueue, and the wait for a free slot) and ``h2d_bytes_per_step``. The augmentation
kernel alone is timed with CUDA events over ``--kernel-launches`` launches and set against the
HBM lower bound (uint8 samples read + minibatch written, at 3.35 TB/s).

Usage (GPU): ``python tools/bench_imagenet_loader.py --out DIR [--batches 256,128]``
"""
import argparse
import json
import os
import pickle
import subprocess
import sys
import tempfile
import time

import numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
SY = SX = 256
C = 3
CROP = 227


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], stdout=subprocess.PIPE,
                              stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except Exception as exc:
        return "unknown (%s)" % type(exc).__name__


def make_dataset(path, n, seed=2024):
    rs = numpy.random.RandomState(seed)
    with open(os.path.join(path, "samples.dat"), "wb") as f:
        for a in range(0, n, 256):
            f.write(rs.randint(0, 256, (min(256, n - a), SY, SX, C)).astype(numpy.uint8).tobytes())
    labels = rs.randint(0, 1000, n)
    labels[:min(n, 1000)] = numpy.arange(min(n, 1000))   # every class present
    with open(os.path.join(path, "labels.pickle"), "wb") as f:
        pickle.dump([("n%08d" % l, int(l)) for l in labels], f)
    with open(os.path.join(path, "count.json"), "w") as f:
        json.dump({"test": 0, "val": 0, "train": n}, f)
    mean = rs.uniform(90, 130, (SY, SX, C))
    with open(os.path.join(path, "matrixes.pickle"), "wb") as f:
        pickle.dump([mean, numpy.full((SY, SX, C), 1 / 64.0)], f)
    return {"sx": SX, "sy": SY, "channels": C, "crop_size_sx": CROP, "crop_size_sy": CROP,
            "mirror": True, "normalization_type": "none",
            "original_labels_filename": os.path.join(path, "labels.pickle"),
            "samples_filename": os.path.join(path, "samples.dat"),
            "matrixes_filename": os.path.join(path, "matrixes.pickle"),
            "count_samples_filename": os.path.join(path, "count.json")}


_HOST_PATH = []


def host_path_loader():
    """Registers (once) a loader that overrides fill_minibatch, so the generic host staging path
    serves it; returns its registry name."""
    if not _HOST_PATH:
        from veles.znicz_b200.loader.imagenet_loader import ImagenetLoader

        class HostPathImagenetLoader(ImagenetLoader):
            MAPPING = "bench_imagenet_host_path"

            def fill_minibatch(self):
                super().fill_minibatch()
        _HOST_PATH.append(HostPathImagenetLoader.MAPPING)
    return _HOST_PATH[0]


def run_arm(arm, loader_cfg, batch, n_train, warmup):
    import torch
    from veles.znicz_b200.core import prng
    from veles.znicz_b200.models import alexnet
    prng.get(1).seed(1234)
    prng.get(2).seed(5678)
    cfg = dict(loader_cfg, minibatch_size=batch, prng=prng.RandomGenerator(seed=99))
    name = "imagenet_pickle_loader"
    if arm == "resident":
        cfg["on_device"] = True
    elif arm == "host":
        name = host_path_loader()
    wf = alexnet.build(loader_name=name, loader_config=cfg, layers=alexnet.alexnet_layers(1000),
                       use_graphs=True,
                       decision_config={"max_epochs": 1, "fail_iterations": 1000},
                       snapshotter_config={"prefix": "bench_inet", "interval": 10 ** 9,
                                           "time_interval": 1e12})
    wf.initialize(device="cuda")
    ld = getattr(wf, "real_loader", None) or wf.loader
    if (ld._aug_ is None) != (arm == "host"):
        raise RuntimeError("arm %s did not get its loader path" % arm)
    mark = {}
    orig = ld.run

    def run():
        if ld.samples_served == warmup * batch:
            torch.cuda.synchronize()
            mark["t0"] = time.perf_counter()
            ld.__dict__["prof_"] = [0.0, 0.0, 0.0, 0]
        orig()
    ld.run = run
    wf.run()
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    if not bool(wf.decision.complete) or ld.samples_served != n_train:
        raise RuntimeError("arm %s: the run did not end after one epoch" % arm)
    prof = ld.__dict__["prof_"]
    steps = n_train // batch - warmup
    res = {"arm": arm, "batch": batch, "timed_steps": steps,
           "images_per_s": steps * batch / (t1 - mark["t0"]),
           "loader_host_ms_per_minibatch": 1e3 * (prof[1] + prof[2]) / max(prof[3], 1),
           "loader_wait_ms_per_minibatch": 1e3 * prof[0] / max(prof[3], 1),
           "h2d_bytes_per_step": int(ld.h2d_bytes_per_step)}
    kernel = None
    if arm != "host" and batch == max(BATCHES):
        kernel = time_kernel(ld, batch)
    ld.stop()
    del wf, ld
    torch.cuda.empty_cache()
    return res, kernel


def time_kernel(ld, batch, launches=None):
    import torch
    launches = launches or KERNEL_LAUNCHES
    for _ in range(10):
        ld._device_augment()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(launches):
        ld._device_augment()
    end.record()
    torch.cuda.synchronize()
    sec = start.elapsed_time(end) / 1e3 / launches
    md = ld.minibatch_data.devmem
    nbytes = batch * SY * SX * C + md.numel() * md.element_size()
    pad = ld.minibatch_data.__dict__.get("padded_dev_")
    if pad is not None:
        nbytes += pad.numel() * pad.element_size()
    bound = nbytes / HBM_BYTES_PER_S
    return {"arm": "kernel_" + ("resident" if ld.on_device else "streamed"), "batch": batch,
            "launches": launches, "us_per_launch": sec * 1e6, "bytes": int(nbytes),
            "padded_copy": pad is not None, "achieved_GB_per_s": nbytes / sec / 1e9,
            "hbm_bound_us": bound * 1e6, "share_of_bound": bound / sec}


BATCHES = (256, 128)
KERNEL_LAUNCHES = 200


def main():
    global BATCHES, KERNEL_LAUNCHES
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--batches", default="256,128")
    ap.add_argument("--epoch-steps", type=int, default=24,
                    help="steps per epoch at the largest batch (the dataset size follows)")
    ap.add_argument("--warmup", type=int, default=8,
                    help="untimed steps per run at the largest batch (graph capture included)")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--kernel-launches", type=int, default=200)
    args = ap.parse_args()
    BATCHES = tuple(int(b) for b in args.batches.split(","))
    KERNEL_LAUNCHES = args.kernel_launches
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_imagenet_loader needs a GPU")
    from veles.znicz_b200.core.config import root
    root.common.engine.compute_type = "bf16"
    os.makedirs(args.out, exist_ok=True)
    gpu = card()
    print("card: %s" % gpu, flush=True)
    bmax = max(BATCHES)
    n_train = args.epoch_steps * bmax
    results = []
    with tempfile.TemporaryDirectory() as tmp:
        loader_cfg = make_dataset(tmp, n_train)
        arms = ["streamed", "resident", "host"]
        for rep in range(args.repeats):
            order = arms[rep % 3:] + arms[:rep % 3]
            for batch in BATCHES:
                warmup = args.warmup * bmax // batch
                for arm in order:
                    res, kernel = run_arm(arm, loader_cfg, batch, n_train, warmup)
                    res["repeat"] = rep
                    results.append(res)
                    print(json.dumps(res), flush=True)
                    if kernel is not None:
                        kernel["repeat"] = rep
                        results.append(kernel)
                        print(json.dumps(kernel), flush=True)
    summary = {}
    for r in results:
        if "images_per_s" in r:
            summary.setdefault("%s@%d" % (r["arm"], r["batch"]), []).append(
                round(r["images_per_s"], 1))
    out = {"card": gpu, "dataset_samples": n_train, "results": results,
           "images_per_s": summary}
    print(json.dumps({"card": gpu, "images_per_s": summary}))
    with open(os.path.join(args.out, "bench_imagenet_loader.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
