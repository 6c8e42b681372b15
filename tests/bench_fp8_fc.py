"""bf16 vs fp8 fully connected layers on AlexNet's FC shapes (batch 128), then the AlexNet training
step through the public API in both compute types. Run on an H100:  python tests/bench_fp8_fc.py

Part 1 times each product with the kernels it needs (CUDA events, L2 flushed before every launch
group): forward = [x quantiser +] GEMM, dgrad = [err quantiser (both forms) +] GEMM,
wgrad = [x^T quantiser +] GEMM, and the per-step fp8 weight re-quantisation.
Part 2 alternates bf16 and fp8 AlexNet training runs (synthetic 227x227 data, batch 128, CUDA
graphs) and reports ms per step from CUDA events around ``wf.run(iterations=...)``.
"""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from veles.znicz_b200.kernels import load_extension  # noqa: E402

ext = load_extension(required=True)
dev = torch.device("cuda")
flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)
BATCH = 128
SHAPES = (("fc6", 9216, 4096), ("fc7", 4096, 4096), ("fc8", 4096, 1000))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], stdout=subprocess.PIPE, text=True,
                              timeout=30).stdout.strip()
    except Exception as exc:          # pragma: no cover
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(), exc)


def timeit(fn, iters=30):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        flush.fill_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters * 1000.0


def r16(n):
    return (n + 15) // 16 * 16


def quant_bufs(rows, cols):
    kr, kc = -(-rows // 128), -(-cols // 128)
    return (torch.empty((rows, r16(cols)), dtype=torch.uint8, device=dev),
            torch.empty((kc, kr * 128), device=dev),
            torch.empty((cols, r16(rows)), dtype=torch.uint8, device=dev),
            torch.empty((kr, kc * 128), device=dev))


def check(r):
    if r != 0:
        raise RuntimeError("launch refused (code %d)" % r)


def bench_layer(name, n_in, n_out):
    x = torch.randn(BATCH, n_in, device=dev).bfloat16()
    err = (torch.randn(BATCH, n_out, device=dev) * 0.01).bfloat16()
    w = torch.randn(n_out, n_in, device=dev) * 0.01
    w_lp = w.bfloat16()
    bias = torch.zeros(n_out, device=dev)
    y = torch.empty(BATCH, n_out, device=dev, dtype=torch.bfloat16)
    ei = torch.empty(BATCH, n_in, device=dev, dtype=torch.bfloat16)
    g = torch.empty(n_out, n_in, device=dev)
    wq, ws, wqt, wst = quant_bufs(n_out, n_in)
    check(ext.fp8_quant(w, n_out, n_in, 1, wq, ws, wqt, wst))
    xq, xs, _, _ = quant_bufs(BATCH, n_in)
    _, _, xqt, xst = quant_bufs(BATCH, n_in)
    eq, es, eqt, est = quant_bufs(BATCH, n_out)

    def bf_fwd():
        check(ext.gemm(x, n_in, False, w_lp, n_in, True, y, n_out, False, BATCH, n_out, n_in, bias,
                       1, 1.0, 0.0, 1, 0, 1))

    def bf_dgrad():
        check(ext.gemm(err, n_out, False, w_lp, n_in, False, ei, n_in, False, BATCH, n_in, n_out,
                       None, 0, 1.0, 0.0, 1, 0, 1))

    def bf_wgrad():
        check(int(ext.fc_wgrad_pair(err, x, g)))

    def f8_fwd():
        check(ext.fp8_quant(x, BATCH, n_in, 0, xq, xs, None, None))
        check(ext.fp8_gemm(xq, xs, wq, ws, y, BATCH, n_out, n_in, bias, 1, 1.0))

    def f8_dgrad():
        check(ext.fp8_quant(err, BATCH, n_out, 0, eq, es, eqt, est))
        check(ext.fp8_gemm(eq, es, wqt, wst, ei, BATCH, n_in, n_out, None, 0, 1.0))

    def f8_wgrad():
        check(ext.fp8_quant(x, BATCH, n_in, 0, None, None, xqt, xst))
        check(ext.fp8_gemm(eqt, est, xqt, xst, g, n_out, n_in, BATCH, None, 0, 1.0))

    def f8_requant():
        check(ext.fp8_quant(w, n_out, n_in, 1, wq, ws, wqt, wst))

    def f8_gemm_only():
        check(ext.fp8_gemm(xq, xs, wq, ws, y, BATCH, n_out, n_in, bias, 1, 1.0))

    res = {}
    for k, fn in (("bf16 forward", bf_fwd), ("fp8 forward", f8_fwd), ("fp8 forward GEMM only",
                  f8_gemm_only), ("bf16 dgrad", bf_dgrad), ("fp8 dgrad", f8_dgrad),
                  ("bf16 wgrad", bf_wgrad), ("fp8 wgrad", f8_wgrad),
                  ("fp8 weight re-quantisation", f8_requant)):
        res[k] = timeit(fn)
    tiles = -(-BATCH // 128) * -(-n_out // 128)
    print("%s (batch %d, %d -> %d; forward GEMM: %d output tiles on %d SMs)" % (
        name, BATCH, n_in, n_out, tiles, torch.cuda.get_device_properties(dev).multi_processor_count))
    for k, v in res.items():
        print("  %-28s %8.1f us" % (k, v))
    return res


def alexnet_step_ms(compute, steps, warmup):
    from veles.znicz_b200.core.config import root
    from veles.znicz_b200.models import alexnet
    root.common.engine.compute_type = compute
    root.common.disable.snapshotting = True
    wf = alexnet.build(
        loader_name="synthetic_imagenet", layers=alexnet.alexnet_layers(1000), use_graphs=True,
        loader_config={"minibatch_size": BATCH, "n_train": 128 * 40, "n_valid": 0, "n_test": 0,
                       "n_classes": 1000, "normalization_type": "internal_mean",
                       "on_device": True, "shuffle_limit": 2000000000},
        decision_config={"max_epochs": 1000000000, "fail_iterations": 1000000},
        snapshotter_config={"prefix": "bench_f8", "interval": 1000000, "time_interval": 1e9})
    wf.initialize(device="cuda")
    wf.run(iterations=6 + warmup)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    n = wf.run(iterations=steps)
    e1.record()
    torch.cuda.synchronize()
    assert n == steps, n
    fc = [f.name for f in wf.forwards if getattr(f, "weights_q_", None) is not None]
    del wf
    torch.cuda.empty_cache()
    return e0.elapsed_time(e1) / steps, fc


def main():
    print("GPU: %s" % gpu_info())
    for name, n_in, n_out in SHAPES:
        bench_layer(name, n_in, n_out)
    print("AlexNet training step, batch %d, CUDA graphs (alternating runs):" % BATCH)
    for rnd in range(2):
        for compute in ("bf16", "fp8"):
            ms, fc = alexnet_step_ms(compute, 20, 4)
            print("  round %d %-5s %7.2f ms/step  (%.0f images/s)%s" % (
                rnd, compute, ms, BATCH / ms * 1000.0,
                "  fp8 layers: " + ",".join(fc) if fc else ""))
    print("GPU: %s" % gpu_info())


if __name__ == "__main__":
    main()
