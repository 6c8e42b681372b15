"""Single-GPU fake-peer harness for ``multi_update_k`` (SURVEY §4: "a single-process fake-peer
mode where the fused all-reduce kernel is pointed at N buffers on one GPU").

N "ranks" = N sets of tensors on ONE device; rank r's launch goes to its own stream with the
same flag / slot / sum pointer tables a real N-GPU run has (all pointing into this GPU's
memory). The N launches must be co-resident (each waits for its peers' flags), hence the
``max_blocks`` cap. Gradients are small dyadic rationals, so every summation order is exact and
the result can be compared BIT FOR BIT with the single-GPU kernel fed the summed gradient.

usage: fake_peer_worker.py N ALGO   (ALGO: 0 one-shot peer loads, 1 two-shot peer stores)
prints one JSON line.
"""
import json
import os
import sys

import numpy
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from veles.znicz_b200.kernels import load_extension  # noqa: E402
from veles.znicz_b200.kernels.api import UpdateDesc  # noqa: E402

MAX_BLOCKS = 592


def hyper(dev):
    # lr wd l1 moment acc_a acc_b gd_a gd_b ortho lr_b wd_b l1_b moment_b + 3 reserved
    return torch.tensor([0.01, 0.0005, 0.25, 0.9, 0, 0, 0, 1, 0.001, 0.02, 0.0, 0.0, 0.9, 0, 0, 0],
                        dtype=torch.float32, device=dev)


def main():
    N, algo = int(sys.argv[1]), int(sys.argv[2])
    ext = load_extension(required=True)
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(5)
    # (rows, cols, is_bias, nparts, lanes): a bias, a small split-K conv weight (lane groups),
    # a mid-size FC weight with the ortho regulariser, a > 1 M tensor (float4 tile path)
    shapes = [(1, 10, 1, 1, 1), (32, 800, 0, 4, 4), (64, 1024, 0, 1, 1), (1200, 1024, 0, 2, 1)]
    w0 = [torch.randn(r, c, generator=g).to(dev) for r, c, *_ in shapes]
    v0 = [torch.randn(r, c, generator=g).to(dev) * 0.01 for r, c, *_ in shapes]
    grads = []          # [rank][tensor] -> [nparts, rows, cols], values k / 64
    for r in range(N):
        grads.append([(torch.randint(-8, 9, (sh[3], sh[0], sh[1]), generator=g).float() / 64).to(dev)
                      for sh in shapes])
    hyp = hyper(dev)

    def build(rank_grads, nranks_parts=1):
        ws = [t.clone() for t in w0]
        vs = [t.clone() for t in v0]
        cs = [torch.zeros(sh[1], device=dev) if (not sh[2] and i == 2) else None
              for i, sh in enumerate(shapes)]
        descs = []
        for i, sh in enumerate(shapes):
            flags = 1 | 2 | (8 if cs[i] is not None else 0)
            gr = rank_grads[i]
            descs.append(UpdateDesc(w=ws[i], grad=gr, hyper=hyp, nparts=gr.shape[0],
                                    part_stride=sh[0] * sh[1], flags=flags, rows=sh[0], cols=sh[1],
                                    is_bias=sh[2], lanes=sh[4], vel=vs[i], col_sums=cs[i]))
        table, tiles, red, _ = ext.multi_update_table(descs, [True] * len(descs), 0)
        return ws, vs, cs, table.to(dev), int(tiles), int(red)

    # ---- oracle: single-GPU kernel fed the (exact) cross-rank sum of the gradients
    summed = [sum(grads[r][i] for r in range(N)) for i in range(len(shapes))]
    ws_ref, vs_ref, _cs, table, tiles, red = build(summed)
    gs = torch.zeros(2, dtype=torch.int32, device=dev)
    for _step in range(3):
        ext.multi_update(table, len(shapes), tiles, True, [], 0, 0, gs, [], 0, 1, [], 0, 0, 0, 0)
    torch.cuda.synchronize()

    # ---- N fake ranks
    ranks = [build(grads[r]) for r in range(N)]
    red_bufs = [torch.zeros(2 * red, device=dev) for _ in range(N)]
    sum_bufs = [torch.full((2 * red,), float("nan"), device=dev) for _ in range(N)]
    flag_bufs = [torch.zeros(MAX_BLOCKS * 8, dtype=torch.int32, device=dev) for _ in range(N)]
    epochs = [torch.zeros(MAX_BLOCKS, dtype=torch.int32, device=dev) for _ in range(N)]
    gss = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in range(N)]
    streams = [torch.cuda.Stream() for _ in range(N)]
    torch.cuda.synchronize()
    # all N launches must be co-resident: 4 CTAs per SM between them
    cap = min(MAX_BLOCKS, 4 * torch.cuda.get_device_properties(dev).multi_processor_count) // N
    for _step in range(3):
        for r in range(N):
            with torch.cuda.stream(streams[r]):
                ext.multi_update(ranks[r][3], len(shapes), ranks[r][4], True,
                                 [int(f.data_ptr()) for f in flag_bufs], int(epochs[r].data_ptr()), r,
                                 gss[r], [int(b.data_ptr()) for b in red_bufs], red, 1,
                                 [int(b.data_ptr()) for b in sum_bufs] if algo == 1 else [], 0, 0,
                                 algo, cap)
    torch.cuda.synchronize()
    out = {"n": N, "algo": algo, "tiles": tiles, "equal_w": True, "equal_v": True,
           "ranks_identical": True, "max_abs_diff": 0.0}
    for r in range(N):
        for i in range(len(shapes)):
            dw = (ranks[r][0][i] - ws_ref[i]).abs().max().item()
            out["max_abs_diff"] = max(out["max_abs_diff"], dw)
            out["equal_w"] &= bool(torch.equal(ranks[r][0][i], ws_ref[i]))
            out["equal_v"] &= bool(torch.equal(ranks[r][1][i], vs_ref[i]))
            out["ranks_identical"] &= bool(torch.equal(ranks[r][0][i], ranks[0][0][i]))
    # the oracle itself against plain PyTorch fp32 for the tensor without ortho (3 steps)
    i = 1
    w, v = w0[i].clone(), v0[i].clone()
    lr, wd, l1, mom = 0.01, 0.0005, 0.25, 0.9
    for _ in range(3):
        gd = -lr * (summed[i].sum(0) + wd * ((1 - l1) * w + 0.5 * l1 * torch.sign(w)))
        gd = gd + v * mom
        v = gd
        w = w + gd
    out["oracle_vs_torch"] = (w - ws_ref[i]).abs().max().item()
    out["finite"] = all(bool(torch.isfinite(t).all()) for rk in ranks for t in rk[0])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
