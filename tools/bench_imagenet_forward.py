"""Merge stage of the localisation pipeline (models/imagenet_forward) with host and device shots.

Synthetic uint8 375 x 500 x 3 pictures with random candidate boxes (plus the 7 relative probes
per picture) go through ``ImagenetForward``'s merge stage: one angle, both mirrors, so each box
gives 2 shots of 227 x 227 x 3, and AlexNet's forward chain in bf16 classifies them. Pictures are
held in memory: decoding is not part of the measurement. Two arms, alternated over ``--repeats``
in one process:

  device   ``render_shots_k`` renders the shots from the uint8 pictures (the cuda path)
  host     ``render_shot`` in numpy, then the fp32 minibatch is uploaded (the host path)

Per arm: shots/s over the stage after ``--warmup`` minibatches (host clock, synchronised at both
ends), the loader's host ms per minibatch and the host-to-device bytes per minibatch. The kernel
alone is timed with CUDA events over ``--kernel-launches`` launches on a full minibatch and set
against the HBM lower bound of the bytes it must move (the minibatch and its channel-padded copy
written, the fp32 mean and the parameter table read; the pictures, a few hundred KB read through
L2 by many shots, are left out) at 3.35 TB/s.

Usage (GPU): ``python tools/bench_imagenet_forward.py --out DIR``
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
H, W, C = 375, 500, 3
A = 227


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], stdout=subprocess.PIPE,
                              stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except Exception as exc:
        return "unknown (%s)" % type(exc).__name__


def make_pictures(n, boxes, seed=7):
    """{key: uint8 [H][W][C]} (smooth random pictures) and their candidate boxes."""
    rs = numpy.random.RandomState(seed)
    pics, cands = {}, {}
    yy, xx = numpy.mgrid[0:H, 0:W]
    for i in range(n):
        key = "pic%03d" % i
        f = rs.uniform(0.005, 0.05, (3, 2))
        img = numpy.stack([128 + 90 * numpy.sin(f[c, 0] * xx + f[c, 1] * yy + c) for c in range(C)], -1)
        pics[key] = numpy.clip(img + rs.normal(0, 12, img.shape), 0, 255).astype(numpy.uint8)
        bw, bh = rs.randint(40, 300, boxes), rs.randint(40, 250, boxes)
        x, y = rs.randint(bw // 2 + 1, W - bw // 2 - 1), rs.randint(bh // 2 + 1, H - bh // 2 - 1)
        cands[key] = {"path": key, "width": W, "height": H, "bbxs": [
            {"x": float(x[j]), "y": float(y[j]), "width": float(bw[j]), "height": float(bh[j])}
            for j in range(boxes)]}     # inside the picture
    return pics, cands


def alexnet_forwards():
    """AlexNet's forward chain, taken out of an (uninitialised) training workflow (without the
    units that mask the grouped layers' weights: they are not part of the data chain)."""
    from veles.znicz_b200.models import alexnet
    train = alexnet.build(loader_name="synthetic_image",
                          loader_config={"shape": (A, A, C), "n_classes": 1000, "n_train": 8,
                                         "n_valid": 0, "minibatch_size": 8},
                          layers=alexnet.alexnet_layers(1000))
    forwards = [f for f in train.forwards if type(f).__name__ != "ZeroFiller"]
    for u in list(train):
        if u not in forwards:
            u.unlink_all()
            train.del_ref(u)
    return forwards


def _host_rendering(self):
    self.numpy_run()
    self.minibatch_data.unmap()


def run_arm(arm, pics, cands, batch, warmup, out_dir):
    import torch
    from veles.znicz_b200.core.workflow import DummyLauncher
    from veles.znicz_b200.models.imagenet_forward.loader import ForwardLoaderBbox
    from veles.znicz_b200.models.imagenet_forward.workflow import ImagenetForward
    saved = ForwardLoaderBbox.cuda_run
    if arm == "host":
        ForwardLoaderBbox.cuda_run = _host_rendering
    try:
        mean = numpy.random.RandomState(3).uniform(90, 130, (A, A, C)).astype(numpy.float32)
        wf = ImagenetForward(
            DummyLauncher(testing=True), forwards=alexnet_forwards(), entry_shape=(batch, A, A, C),
            mean=mean, bboxes=cands, image_reader=lambda p: pics[p],
            result_path=os.path.join(out_dir, "result_%s.json" % arm),
            labels_mapping={i: "n%08d" % i for i in range(1000)},
            loader_config={"minibatch_size": batch, "raw_bboxes_min_area": 0,
                           "raw_bboxes_min_size": 0, "raw_bboxes_min_area_ratio": 0,
                           "raw_bboxes_min_size_ratio": 0},
            merge_config={"use_compatibility": False})
        wf.initialize(device="cuda")
    finally:
        ForwardLoaderBbox.cuda_run = saved
    ld = wf.loader
    ext = wf.device.ext
    launches0 = ext.render_shots_launches()
    mark = {"k": 0, "host": 0.0}
    orig = ld.run

    def run():
        if mark["k"] == warmup:
            torch.cuda.synchronize()
            mark["t0"] = time.perf_counter()
            mark["shots0"] = ld.processed
            mark["h2d0"] = ld.h2d_bytes
        t = time.perf_counter()
        orig()
        if mark["k"] >= warmup:
            mark["host"] += time.perf_counter() - t
        mark["k"] += 1
    ld.run = run
    wf.run_stage()
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    timed = mark["k"] - warmup
    launched = ext.render_shots_launches() - launches0
    if launched != (mark["k"] if arm == "device" else 0):
        raise RuntimeError("arm %s: %d kernel launches for %d minibatches" % (arm, launched, mark["k"]))
    md = ld.minibatch_data
    h2d = (ld.h2d_bytes - mark["h2d0"]) / timed if arm == "device" else md.mem.nbytes
    res = {"arm": arm, "batch": batch, "shots": ld.processed, "timed_minibatches": timed,
           "shots_per_s": (ld.processed - mark["shots0"]) / (t1 - mark["t0"]),
           "loader_host_ms_per_minibatch": 1e3 * mark["host"] / timed,
           "h2d_bytes_per_minibatch": int(h2d), "input_dtype": str(md.devmem.dtype),
           "pictures_uploaded": ld.pictures_uploaded}
    kernel = None
    if arm == "device":
        ld.reset()          # the stage's last run may be ragged or empty: time its first minibatch
        ld.run()
        kernel = time_kernel(ld, batch)
    del wf, ld
    torch.cuda.empty_cache()
    return res, kernel


def time_kernel(ld, batch, launches=None):
    import torch
    from veles.znicz_b200.loader.base import channel_pad_target
    launches = launches or KERNEL_LAUNCHES
    rs = ld.render_
    md = ld.minibatch_data
    pad = channel_pad_target(md)
    dv = rs["dv"]

    def launch():
        ld.device.ext.render_shots(rs["arena"], dv["hdr"], dv["shots"], dv["pics"], rs["mean"],
                                   md.devmem, pad)
    resident = len(rs["resident"])
    rendered = int((dv["pics"][:, 1] > 0).sum().item())
    for _ in range(10):
        launch()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(launches):
        launch()
    end.record()
    torch.cuda.synchronize()
    sec = start.elapsed_time(end) / 1e3 / launches
    nbytes = md.devmem.numel() * md.devmem.element_size() + A * A * C * 4 + rs["tab"]
    if pad is not None:
        nbytes += pad.numel() * pad.element_size()
    bound = nbytes / HBM_BYTES_PER_S
    return {"arm": "kernel", "batch": batch, "rendered_rows": rendered, "resident_pictures": resident,
            "launches": launches, "us_per_launch": sec * 1e6, "bytes": int(nbytes),
            "padded_copy": pad is not None, "achieved_GB_per_s": nbytes / sec / 1e9,
            "hbm_bound_us": bound * 1e6, "share_of_bound": bound / sec}


KERNEL_LAUNCHES = 200


def main():
    global KERNEL_LAUNCHES
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--pictures", type=int, default=16)
    ap.add_argument("--boxes", type=int, default=25, help="candidate boxes per picture")
    ap.add_argument("--warmup", type=int, default=2, help="untimed minibatches per run")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--kernel-launches", type=int, default=200)
    args = ap.parse_args()
    KERNEL_LAUNCHES = args.kernel_launches
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_imagenet_forward needs a GPU")
    from veles.znicz_b200.core.config import root
    root.common.engine.compute_type = "bf16"
    os.makedirs(args.out, exist_ok=True)
    gpu = card()
    print("card: %s" % gpu, flush=True)
    pics, cands = make_pictures(args.pictures, args.boxes)
    results, written = [], {}
    arms = ["device", "host"]
    with tempfile.TemporaryDirectory() as tmp:
        for rep in range(args.repeats):
            for arm in arms[rep % 2:] + arms[:rep % 2]:
                res, kernel = run_arm(arm, pics, cands, args.batch, args.warmup, tmp)
                res["repeat"] = rep
                results.append(res)
                print(json.dumps(res), flush=True)
                with open(os.path.join(tmp, "result_%s.json" % arm)) as f:
                    written.setdefault(arm, []).append(json.load(f))
                if kernel is not None:
                    kernel["repeat"] = rep
                    results.append(kernel)
                    print(json.dumps(kernel), flush=True)
    same = all(w == written["device"][0] for ws in written.values() for w in ws)
    summary = {}
    for r in results:
        if "shots_per_s" in r:
            summary.setdefault(r["arm"], []).append(round(r["shots_per_s"], 1))
    out = {"card": gpu, "pictures": args.pictures, "boxes_per_picture": args.boxes,
           "results": results, "shots_per_s": summary, "same_json_both_arms": same}
    print(json.dumps({"card": gpu, "shots_per_s": summary, "same_json_both_arms": same}))
    with open(os.path.join(args.out, "bench_imagenet_forward.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
