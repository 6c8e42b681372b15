"""Small workloads for ``compute-sanitizer --tool {memcheck,racecheck,synccheck}``: every
hand-rolled synchronisation protocol of the repo on sizes a sanitizer run can finish -
gemm_umma_k (mbarrier ring, TMA + LDGSTS producers, wgmma), gemm_pair_k (producer / MMA
warpgroups, TMA-store epilogue), lstm kernels (barrier.cluster), multi_update_k (grid barrier;
fake-peer flag protocol with 2 ranks sharing the GPU), fc_small, pooling / LRN / evaluator,
rbm_sample_k / rbm_apply_k (ragged shapes: partial batch, partial transpose tiles),
render_shots_k (1 x N and N x 1 pictures, boxes over the edges, rows past n, padded copy)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from veles.znicz_b200.kernels import load_extension  # noqa: E402

ext = load_extension(required=True)
dev = torch.device("cuda:0")
torch.manual_seed(0)


def gemm_single():
    m, n, k = 256, 96, 192
    a = torch.randn(m, k, device=dev).bfloat16()
    b = torch.randn(n, k, device=dev).bfloat16()
    o = torch.empty(m, n, device=dev, dtype=torch.bfloat16)
    assert ext.gemm(a, k, False, b, k, True, o, n, False, m, n, k, None, 0, 1.0, 0.0, 1, 0, 1) == 0
    torch.cuda.synchronize()
    assert ((o.float() - a.float() @ b.float().t()).abs().max() < 0.5)


def conv_umma():
    n, h, w, c, f = 4, 12, 12, 16, 32
    x = torch.randn(n, h, w, c, device=dev).bfloat16()
    wt = torch.randn(f, 3 * 3 * c, device=dev).bfloat16().contiguous()
    out = torch.empty(n, h, w, f, device=dev, dtype=torch.bfloat16)
    g = [n, h, w, c, h, w, f, 3, 3, 1, 1, 1, 1]
    assert ext.conv_fprop(x, wt, wt.shape[1], False, None, out, g, 0, 1) == 0
    torch.cuda.synchronize()


def gemm_pair():
    m, n, k = 512, 256, 128
    a = torch.randn(m, k, device=dev).bfloat16()
    b = torch.randn(n, k, device=dev).bfloat16()
    o = torch.empty(m, n, device=dev, dtype=torch.bfloat16)
    assert ext.gemm_pair(a, b, o, None, 0, 1.0) == 0
    torch.cuda.synchronize()
    assert ((o.float() - a.float() @ b.float().t()).abs().max() < 0.5)


def multi_update():
    sys.argv = ["fake_peer_worker.py", "2", "1"]
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import fake_peer_worker
    fake_peer_worker.main()


def rbm_sample():
    rows, n, bs = 9, 70, 5
    rng = torch.tensor([12345, 7], dtype=torch.int32, device=dev)
    for dt in (torch.float32, torch.bfloat16):
        p = torch.rand(rows, n, device=dev).to(dt)
        out = torch.empty_like(p)
        ext.rbm_sample(p, out, bs, rng)
        torch.cuda.synchronize()
        assert torch.equal(out[bs:], p[bs:]) and bool(((out[:bs] == 0) | (out[:bs] == 1)).all())


def rbm_apply():
    h, v = 45, 37
    w = torch.randn(h, v, device=dev)
    g = torch.randn(v, h, device=dev)
    hb, hg, vb, vg = (torch.randn(k, device=dev) for k in (h, h, v, v))
    want = (w + 0.5 * g.t(), hb + 0.5 * hg, vb + 0.5 * vg)
    ext.rbm_apply(w, g, hb, hg, vb, vg, 0.5)
    torch.cuda.synchronize()
    assert all(torch.allclose(a, b) for a, b in zip((w, hb, vb), want))


def render_shots():
    import numpy
    from veles.znicz_b200.models.imagenet_forward.loader import shot_table_row
    a, c, rows = 13, 3, 7
    pics = [(1, 30), (25, 1), (17, 22)]               # h, w: 1 x N, N x 1 and a plain picture
    arena = torch.randint(0, 256, (sum(h * w * c for h, w in pics) + 5,), dtype=torch.uint8,
                          device=dev)
    table = numpy.zeros((rows, 8))
    geo = numpy.zeros((rows, 4), numpy.int64)
    at = 5
    for r, (h, w) in enumerate(pics * 2):
        if r < len(pics):
            geo[r] = (at, h, w, r % 2)
            at += h * w * c
        else:
            geo[r] = geo[r - len(pics)]
        box = {"x": w - 1.0, "y": 0.0, "width": 9.0 + r, "height": 8.0}
        table[r] = shot_table_row(box, 0.7 * r - 2.0, a)
    hdr = torch.tensor([rows - 2, 0, 0, 0], dtype=torch.int32, device=dev)
    mean = torch.rand(a, a, c, device=dev)
    for dt in (torch.float32, torch.bfloat16):
        out = torch.empty(rows, a, a, c, device=dev, dtype=dt)
        pad = torch.empty(rows, a, a, 8, device=dev, dtype=dt)
        ext.render_shots(arena, hdr, torch.from_numpy(table).to(dev), torch.from_numpy(geo).to(dev),
                         mean, out, pad)
        torch.cuda.synchronize()
        assert not out[rows - 2:].any() and torch.equal(pad[..., :c], out) and not pad[..., c:].any()


if __name__ == "__main__":
    which = sys.argv[1:] or ["gemm_single", "conv_umma", "gemm_pair", "multi_update", "rbm_sample",
                             "rbm_apply", "render_shots"]
    for name in which:
        globals()[name]()
        print("ok", name, flush=True)
