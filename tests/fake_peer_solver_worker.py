"""Single-GPU fake-peer harness for the solver bits of ``multi_update_k`` (adagrad, adadelta, fast,
RProp), modelled on fake_peer_worker.py: N "ranks" = N sets of tensors on ONE device, each launch
on its own stream with the flag / slot / sum pointer tables of a real N-GPU run. Gradients are
small dyadic rationals, so every summation order is exact and the result is compared BIT FOR BIT
with the single-GPU kernel fed the summed gradient: weights, velocities, the gradient written back
(RProp's previous gradient) and the solver state, for the whole-network kernel (multi_update_k)
and for the per-tensor kernel (fused_update_k).

usage: fake_peer_solver_worker.py N ALGO   (ALGO: 0 one-shot peer loads, 1 two-shot peer stores)
prints one JSON line.
"""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from veles.znicz_b200.kernels import load_extension  # noqa: E402
from veles.znicz_b200.kernels.api import UpdateDesc  # noqa: E402

MAX_BLOCKS = 592
ADAGRAD, ADADELTA, FAST, RPROP = 32, 64, 128, 256


def hyper(dev):
    # GradientDescentBase.HYPER_FIELDS: 13 SGD slots, then adagrad eps, adadelta rho / eps,
    # fast lr, RProp increase / decrease / min / max, 3 reserved
    return torch.tensor([0.01, 0.0005, 0.25, 0.9, 0, 0, 0, 1, 0.001, 0.02, 0.0, 0.0, 0.9,
                         1e-8, 0.9, 1e-6, 0.02, 1.2, 0.5, 1e-5, 0.05, 0, 0, 0],
                        dtype=torch.float32, device=dev)


def desc(w, gout, vel, hyp, colsums, grad, flags, sh, states):
    return UpdateDesc(w=w, grad=grad, hyper=hyp, nparts=grad.shape[0], part_stride=sh[0] * sh[1],
                      flags=flags, rows=sh[0], cols=sh[1], is_bias=sh[2], lanes=sh[4],
                      grad_out=gout, vel=vel, col_sums=colsums, s0=states[0], s1=states[1],
                      s2=states[2])


def main():
    N, algo = int(sys.argv[1]), int(sys.argv[2])
    ext = load_extension(required=True)
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(7)
    # (rows, cols, is_bias, nparts, lanes, solver bits): every solver on a bias, on a split-K conv
    # weight (lane groups), on an FC weight with ortho, and on > 1 M tensors (4 elements per
    # thread, scalar path)
    shapes = [(1, 10, 1, 1, 1, RPROP), (32, 800, 0, 4, 4, ADADELTA | FAST),
              (64, 1024, 0, 1, 1, ADAGRAD | FAST), (1200, 1024, 0, 2, 1, ADAGRAD),
              (1, 64, 1, 3, 2, ADADELTA), (1100, 1024, 0, 1, 1, RPROP)]
    w0 = [torch.randn(r, c, generator=g).to(dev) for r, c, *_ in shapes]
    v0 = [torch.randn(r, c, generator=g).to(dev) * 0.01 for r, c, *_ in shapes]
    grads = []          # [rank][tensor] -> [nparts, rows, cols], values k / 64
    for r in range(N):
        grads.append([(torch.randint(-8, 9, (sh[3], sh[0], sh[1]), generator=g).float() / 64).to(dev)
                      for sh in shapes])
    hyp = hyper(dev)
    ortho_i = 2

    def build(rank_grads):
        # every tensor the table points at is kept in ``out``: a freed buffer would be reused by
        # the next allocation (e.g. the grid-barrier counter) while the kernel still writes it
        out = {"w": [], "v": [], "gout": [], "state": []}
        descs = []
        for i, sh in enumerate(shapes):
            bits = sh[5]
            w, v = w0[i].clone(), v0[i].clone()
            gout = torch.zeros_like(w)
            cs = torch.zeros(sh[1], device=dev) if i == ortho_i else None
            st = [(torch.full_like(w, 0.01) if bits & RPROP else torch.zeros_like(w))
                  if bits & (ADAGRAD | ADADELTA | RPROP) else None,
                  torch.zeros_like(w) if bits & ADADELTA else None,
                  torch.zeros_like(w) if bits & FAST else None]
            flags = 1 | bits | (0 if bits & RPROP else 2) | (8 if cs is not None else 0)
            gr = rank_grads[i]
            descs.append(desc(w, gout, v, hyp, cs, gr, flags, sh, st))
            out["w"].append(w)
            out["v"].append(v)
            out["gout"].append(gout)
            out["state"].append(st + [cs])
        table, tiles, red, _ = ext.multi_update_table(descs, [True] * len(descs), 0)
        out["table"], out["tiles"], out["red"] = table.to(dev), int(tiles), int(red)
        return out

    # ---- oracle: single-GPU kernel fed the (exact) cross-rank sum of the gradients
    summed = [sum(grads[r][i] for r in range(N)) for i in range(len(shapes))]
    ref = build(summed)
    gs = torch.zeros(2, dtype=torch.int32, device=dev)
    for _step in range(3):
        ext.multi_update(ref["table"], len(shapes), ref["tiles"], True, [], 0, 0, gs, [], 0,
                         1, [], 0, 0, 0, 0)
    torch.cuda.synchronize()

    # ---- N fake ranks
    ranks = [build(grads[r]) for r in range(N)]
    red = ref["red"]
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
                ext.multi_update(ranks[r]["table"], len(shapes), ranks[r]["tiles"], True,
                                 [int(f.data_ptr()) for f in flag_bufs], int(epochs[r].data_ptr()), r,
                                 gss[r], [int(b.data_ptr()) for b in red_bufs], red, 1,
                                 [int(b.data_ptr()) for b in sum_bufs] if algo == 1 else [], 0, 0,
                                 algo, cap)
    torch.cuda.synchronize()
    out = {"n": N, "algo": algo, "tiles": ref["tiles"], "equal_w": True, "equal_v": True,
           "equal_gout": True, "equal_state": True, "ranks_identical": True, "max_abs_diff": 0.0}
    for rk in ranks:
        for i in range(len(shapes)):
            out["max_abs_diff"] = max(out["max_abs_diff"],
                                      (rk["w"][i] - ref["w"][i]).abs().max().item())
            out["equal_w"] &= bool(torch.equal(rk["w"][i], ref["w"][i]))
            out["equal_v"] &= bool(torch.equal(rk["v"][i], ref["v"][i]))
            out["equal_gout"] &= bool(torch.equal(rk["gout"][i], ref["gout"][i]))
            for a, b in zip(rk["state"][i], ref["state"][i]):
                if a is not None:
                    out["equal_state"] &= bool(torch.equal(a, b))
            out["ranks_identical"] &= bool(torch.equal(rk["w"][i], ranks[0]["w"][i]))
    # ---- the per-tensor kernel (fused_update_k, used for tied weights and without the fused
    # step): every rank reads every rank's split-K partials over the peer pointers
    blocks = 8                      # N launches of this size are co-resident whatever N is
    pt_ref = build(summed)
    pt_ranks = [build(grads[r]) for r in range(N)]

    def per_tensor(bufs, i, grad, grad_ptrs, peer_flags, epoch_ptr, rank):
        sh = shapes[i]
        flags = 1 | sh[5] | (0 if sh[5] & RPROP else 2)          # (no ortho: needs col sums)
        ext.fused_update(desc(bufs["w"][i], bufs["gout"][i], bufs["v"][i], hyp, None, grad, flags,
                              sh, bufs["state"][i]),
                         grad_ptrs, peer_flags, epoch_ptr, rank, blocks)
    pt_flags = [[torch.zeros(MAX_BLOCKS * 8, dtype=torch.int32, device=dev) for _ in range(N)]
                for _ in shapes]
    pt_epochs = [[torch.zeros(MAX_BLOCKS, dtype=torch.int32, device=dev) for _ in range(N)]
                 for _ in shapes]
    torch.cuda.synchronize()
    for _step in range(3):
        for i in range(len(shapes)):
            per_tensor(pt_ref, i, summed[i], [], [], 0, 0)
            for r in range(N):
                with torch.cuda.stream(streams[r]):
                    per_tensor(pt_ranks[r], i, grads[r][i],
                               [int(grads[q][i].data_ptr()) for q in range(N)],
                               [int(f.data_ptr()) for f in pt_flags[i]],
                               int(pt_epochs[i][r].data_ptr()), r)
    torch.cuda.synchronize()
    out["per_tensor_equal"] = all(
        all(torch.equal(rk[k][i], pt_ref[k][i]) for k in ("w", "v", "gout")) and
        all(a is None or torch.equal(a, b) for a, b in zip(rk["state"][i], pt_ref["state"][i]))
        for rk in pt_ranks for i in range(len(shapes)))
    # every solver actually moved its state
    out["state_moved"] = all(
        bool((st[0] != 0.01).any()) if sh[5] & RPROP else
        all(t is None or bool((t != 0).any()) for t in st[:3])
        for sh, st in zip(shapes, ref["state"]))
    out["finite"] = all(bool(torch.isfinite(t).all()) for rk in ranks for t in rk["w"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
