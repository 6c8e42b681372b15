"""Localisation shots rendered on the GPU (csrc/render.cu, models/imagenet_forward/loader.py):
the kernel contract stated in numpy against ``render_shot`` (CPU), then the kernel, the loader and
the whole two-stage pipeline on the device against the host renderer, bit for bit."""
import json
import pickle

import numpy
import pytest

from veles.znicz_b200.core.config import root
from veles.znicz_b200.core.workflow import DummyLauncher
from veles.znicz_b200.models.imagenet_forward.loader import (ForwardLoaderBbox, render_shot,
                                                             shot_table_row)
from veles.znicz_b200.models.imagenet_forward.workflow import ImagenetForward

PI = numpy.pi
ANGLES = (0.0, PI / 2, -PI / 2, PI, -PI, PI / 4)


def _sweep_pictures():
    rs = numpy.random.RandomState(21)
    return {3: [rs.randint(0, 256, (37, 52, 3)).astype(numpy.uint8),
                rs.randint(0, 256, (1, 40, 3)).astype(numpy.uint8),     # 1 x N
                rs.randint(0, 256, (33, 1, 3)).astype(numpy.uint8)],    # N x 1
            1: [rs.randint(0, 256, (29, 44, 1)).astype(numpy.uint8),
                rs.randint(0, 256, (1, 25, 1)).astype(numpy.uint8),
                rs.randint(0, 256, (21, 1, 1)).astype(numpy.uint8)]}


def _sweep_boxes(h, w, aperture):
    """Inside, hanging over each edge, fully outside; the last two are the aperture's own size,
    odd or even, centred so that their sample points fall exactly on pixel centres."""
    a = float(aperture)
    centre = (a - 1) / 2.0 % 1.0           # 0 for odd, 0.5 for even apertures
    return [{"x": w / 2.0, "y": h / 2.0, "width": 0.6 * w + 1, "height": 0.7 * h + 1},
            {"x": 1.0, "y": h / 2.0, "width": 9.0, "height": 6.0},            # left edge
            {"x": w - 2.0, "y": h / 2.0, "width": 8.0, "height": 7.0},        # right edge
            {"x": w / 2.0, "y": 0.0, "width": 7.0, "height": 9.0},            # top edge
            {"x": w / 2.0, "y": h - 1.0, "width": 6.0, "height": 8.0},        # bottom edge
            {"x": -30.0, "y": -40.0, "width": 10.0, "height": 12.0},          # fully outside
            {"x": w + 25.0, "y": h / 2.0, "width": 8.0, "height": 8.0},       # fully outside
            {"x": w // 2 + centre, "y": h // 2 + centre, "width": a, "height": a},
            {"x": w // 2 + centre, "y": h // 2 + centre, "width": a + 1, "height": a - 1}]


def _sweep(channels, aperture):
    """[(picture, bbox, angle, flip)] over every picture, box, angle and mirror of one C."""
    out = []
    for img in _sweep_pictures()[channels]:
        for box in _sweep_boxes(img.shape[0], img.shape[1], aperture):
            for angle in ANGLES:
                for flip in (False, True):
                    out.append((img, box, angle, flip))
    return out


def _tables(shots, aperture, rows):
    """The picture arena (pictures at odd byte offsets) and the kernel's parameter tables, from the
    loader's own ``shot_table_row``."""
    arena, where = [numpy.zeros(3, numpy.uint8)], {}
    at = 3
    for img, _box, _angle, _flip in shots:
        if id(img) not in where:
            where[id(img)] = at
            arena.append(img.reshape(-1))
            at += img.size
    table = numpy.zeros((rows, 8), numpy.float64)
    pics = numpy.zeros((rows, 4), numpy.int64)
    for r, (img, box, angle, flip) in enumerate(shots):
        table[r] = shot_table_row(box, angle, aperture)
        pics[r] = (where[id(img)], img.shape[0], img.shape[1], int(flip))
    return numpy.concatenate(arena), table, pics


def _contract(arena, n, table, pics, mean, aperture, channels):
    """The kernel contract of render_shots_k in numpy, one float64 operation at a time."""
    A, C = aperture, channels
    out = numpy.zeros((len(table), A, A, C), numpy.float32)
    m = numpy.zeros((A, A, C), numpy.float32) if mean is None else mean
    a2 = (A - 1) / 2.0
    u = numpy.arange(A, dtype=numpy.float64) - a2
    for r in range(n):
        ca, sa, scale, hbw, hbh, cx, cy, _ = table[r]
        off, h, w, flip = (int(x) for x in pics[r])
        img = arena[off:off + h * w * C].reshape(h, w, C)
        ux = numpy.broadcast_to(-u if flip else u, (A, A))
        uy = numpy.broadcast_to(u[:, None], (A, A))
        bx = numpy.add(numpy.multiply(ux, ca), numpy.multiply(uy, sa)) / scale
        by = numpy.add(numpy.multiply(-ux, sa), numpy.multiply(uy, ca)) / scale
        px, py = bx + cx, by + cy
        inside = ((numpy.abs(bx) <= hbw) & (numpy.abs(by) <= hbh) & (px >= 0) & (px <= w - 1) &
                  (py >= 0) & (py <= h - 1))
        x0 = numpy.minimum(numpy.maximum(numpy.floor(px), 0.0), w - 2 if w > 1 else 0).astype(int)
        y0 = numpy.minimum(numpy.maximum(numpy.floor(py), 0.0), h - 2 if h > 1 else 0).astype(int)
        x1, y1 = numpy.minimum(x0 + 1, w - 1), numpy.minimum(y0 + 1, h - 1)
        fx = numpy.minimum(numpy.maximum(px - x0.astype(numpy.float64), 0.0), 1.0)[..., None]
        fy = numpy.minimum(numpy.maximum(py - y0.astype(numpy.float64), 0.0), 1.0)[..., None]
        gx, gy = 1.0 - fx, 1.0 - fy
        s = img.astype(numpy.float64)
        val = (s[y0, x0] * gx) * gy
        val = val + (s[y0, x1] * fx) * gy
        val = val + (s[y1, x0] * gx) * fy
        val = val + (s[y1, x1] * fx) * fy
        a = inside[..., None].astype(numpy.float32)
        blend = (m * (numpy.float32(1.0) - a)).astype(numpy.float64) + val * a.astype(numpy.float64)
        out[r] = blend.astype(numpy.float32)
    return out


def _means(aperture, channels):
    rs = numpy.random.RandomState(5)
    return (None, (rs.rand(aperture, aperture, channels) * 255 - 60).astype(numpy.float32))


def _reference(shots, aperture, channels, mean):
    m = numpy.zeros((aperture, aperture, channels), numpy.float32) if mean is None else mean
    return numpy.stack([render_shot(img, box, angle, flip, aperture, m)
                        for img, box, angle, flip in shots])


@pytest.mark.parametrize("channels,aperture", [(3, 15), (3, 16), (1, 15), (1, 16)])
def test_contract_of_the_kernel_equals_render_shot(channels, aperture):
    """Fed the loader's parameter table, the numpy statement of the kernel contract gives
    render_shot's bits: angles 0, +-pi/2, +-pi and pi/4, both mirrors, boxes over every edge and
    outside, pixel-centred odd and even boxes, 1 x N and N x 1 pictures, with and without a mean."""
    shots = _sweep(channels, aperture)
    arena, table, pics = _tables(shots, aperture, len(shots))
    for mean in _means(aperture, channels):
        got = _contract(arena, len(shots), table, pics, mean, aperture, channels)
        want = _reference(shots, aperture, channels, mean)
        assert got.view(numpy.uint32).tobytes() == want.view(numpy.uint32).tobytes()


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
def _ext():
    from veles.znicz_b200.kernels import load_extension
    return load_extension(required=True)


def _bits(t):
    import torch
    return t.detach().cpu().contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("channels,aperture", [(3, 15), (3, 16), (1, 15), (1, 16)])
def test_kernel_equals_render_shot(channels, aperture):
    """fp32 output = render_shot bit for bit, bf16 = its round-to-nearest-even, rows past n zero,
    the channel-padded copy = the output padded to 8 channels."""
    import torch
    ext = _ext()
    dev = torch.device("cuda:0")
    shots = _sweep(channels, aperture)
    rows = len(shots) + 5
    arena, table, pics = _tables(shots, aperture, rows)
    hdr = torch.tensor([len(shots), 0, 0, 0], dtype=torch.int32, device=dev)
    targs = (torch.from_numpy(arena).to(dev), hdr, torch.from_numpy(table).to(dev),
             torch.from_numpy(pics).to(dev))
    for mean in _means(aperture, channels):
        want = torch.from_numpy(_reference(shots, aperture, channels, mean))
        md = None if mean is None else torch.from_numpy(mean).to(dev)
        for dt in (torch.float32, torch.bfloat16):
            out = torch.full((rows, aperture, aperture, channels), 3.0, dtype=dt, device=dev)
            pad = torch.full((rows, aperture, aperture, 8), 3.0, dtype=dt, device=dev)
            before = ext.render_shots_launches()
            ext.render_shots(*targs, md, out, pad)
            torch.cuda.synchronize()
            assert ext.render_shots_launches() == before + 1
            ref = want if dt == torch.float32 else want.to(torch.bfloat16)
            assert torch.equal(_bits(out[:len(shots)]), _bits(ref))
            assert not out[len(shots):].any()
            padded = torch.zeros((rows, aperture, aperture, 8), dtype=dt, device=dev)
            padded[..., :channels] = out
            assert torch.equal(_bits(pad), _bits(padded))


def _loader_pictures():
    rs = numpy.random.RandomState(8)
    pics = {"p0.npy": rs.randint(0, 256, (41, 57, 3)).astype(numpy.uint8),
            "p1.npy": rs.randint(0, 256, (60, 38, 3)).astype(numpy.uint8),
            "p2.npy": rs.randint(0, 256, (35, 35, 3)).astype(numpy.uint8)}
    boxes = {"p0.npy": [{"x": 28.0, "y": 20.0, "width": 30.0, "height": 24.0},
                        {"x": 5.0, "y": 36.0, "width": 16.0, "height": 19.0},
                        {"x": 40.0, "y": 10.0, "width": 21.0, "height": 21.0}],
             "p1.npy": [{"x": 19.0, "y": 30.0, "width": 25.0, "height": 40.0},
                        {"x": 30.5, "y": 55.0, "width": 14.0, "height": 12.0}],
             "p2.npy": [{"x": 17.0, "y": 17.0, "width": 35.0, "height": 35.0},
                        {"x": 0.0, "y": 34.0, "width": 20.0, "height": 10.0}]}
    return pics, {k: {"path": k, "bbxs": v} for k, v in boxes.items()}


def _loader(pics, bboxes, device, **kw):
    ld = ForwardLoaderBbox(DummyLauncher(), bboxes=bboxes, minibatch_size=8,
                           angle_step=PI / 12, min_angle=-PI / 12, max_angle=PI / 12,
                           add_relative_bboxes=False, image_reader=lambda p: pics[p],
                           entry_shape=(8, 16, 16, 3),
                           mean=numpy.random.RandomState(3).rand(16, 16, 3).astype(numpy.float32) * 200,
                           **kw)
    ld.initialize(device=device)
    return ld


def _run_side_by_side(pics, bboxes, feeds_first_layer=False, padded=False):
    """Both loaders minibatch by minibatch; returns the cuda loader and the number of minibatches
    it rendered on the device. ``padded``: a first conv layer has asked for the channel-padded
    copy, which must equal the minibatch padded to 8 channels after every run, whichever path
    rendered it."""
    import torch
    ext = _ext()
    host = _loader(pics, bboxes, None)
    cuda = _loader(pics, bboxes, "cuda", feeds_first_layer=feeds_first_layer)
    if padded:
        cuda.minibatch_data.__dict__["pad_request_"] = 8
    device_batches = 0
    while not host.ended:
        before = ext.render_shots_launches()
        host.run()
        cuda.run()
        n = host.minibatch_size
        assert cuda.minibatch_size == n and cuda.processed == host.processed
        assert cuda.minibatch_bboxes[:n] == host.minibatch_bboxes[:n]
        assert cuda.minibatch_images[:n] == host.minibatch_images[:n]
        assert bool(cuda.ended) == bool(host.ended)
        launched = ext.render_shots_launches() - before
        assert launched in (0, 1)
        device_batches += launched
        got = cuda.minibatch_data.devmem[:n]
        want = torch.from_numpy(host.minibatch_data.mem[:n]).to(got.device).to(got.dtype)
        assert torch.equal(_bits(got), _bits(want))
        if padded:
            md = cuda.minibatch_data.devmem
            pad = cuda.minibatch_data.__dict__["padded_dev_"]
            want = torch.zeros(tuple(md.shape[:3]) + (8,), dtype=md.dtype, device=md.device)
            want[..., :md.shape[3]] = md
            assert torch.equal(_bits(pad), _bits(want))
    return cuda, device_batches


@pytest.mark.gpu
@pytest.mark.parametrize("compute", ["fp32", "bf16"])
def test_loader_on_cuda_serves_the_numpy_minibatches(compute):
    """3 pictures, 42 shots in minibatches of 8 (the last one ragged): the same boxes, pictures,
    ``processed`` and rows as the numpy loader, one launch per minibatch, each picture uploaded
    once per stage."""
    import torch
    root.common.engine.compute_type = compute
    pics, bboxes = _loader_pictures()
    cuda, launched = _run_side_by_side(pics, bboxes, feeds_first_layer=True)
    assert cuda.processed == cuda.total == 42 and launched == 6
    assert cuda.minibatch_data.devmem.dtype == (torch.bfloat16 if compute == "bf16" else torch.float32)
    assert cuda.pictures_uploaded == 3
    # the next stage starts over: every picture goes up once more
    cuda.reset()
    assert cuda.pictures_uploaded == 0
    while not cuda.ended:
        cuda.run()
    torch.cuda.synchronize()
    assert cuda.pictures_uploaded == 3


@pytest.mark.gpu
def test_loader_renders_other_pictures_on_the_host():
    """A minibatch holding a float picture (or one of another channel count) is rendered on the
    host and uploaded: the rows still equal the numpy loader's, and only the minibatches of uint8
    pictures launch the kernel."""
    pics, bboxes = _loader_pictures()
    pics["p1.npy"] = pics["p1.npy"].astype(numpy.float32)
    pics["p3.npy"] = numpy.random.RandomState(9).randint(0, 256, (30, 30, 1)).astype(numpy.uint8)
    bboxes["p3.npy"] = {"path": "p3.npy", "bbxs": [{"x": 15.0, "y": 15.0, "width": 20.0,
                                                    "height": 20.0}]}
    cuda, launched = _run_side_by_side(pics, bboxes)
    # shots 0-17 p0, 18-29 p1 (float), 30-41 p2, 42-47 p3 (C = 1): minibatches 0, 1 and 4 on the
    # device, and the empty seventh run that ends the stage (its rows are zero)
    assert cuda.processed == 48 and launched == 4
    assert cuda.pictures_uploaded == 2


@pytest.mark.gpu
def test_host_minibatches_keep_the_padded_copy_current():
    """A first conv layer with C < 8 reads the loader's channel-padded copy as current: after a
    device minibatch the host path must refresh it too (device, device, host, host, device, host,
    device in bf16)."""
    root.common.engine.compute_type = "bf16"
    pics, bboxes = _loader_pictures()
    pics["p1.npy"] = pics["p1.npy"].astype(numpy.float32)
    pics["p3.npy"] = pics["p0.npy"].astype(numpy.float64)
    bboxes["p3.npy"] = {"path": "p3.npy", "bbxs": bboxes["p0.npy"]["bbxs"][:1]}
    cuda, launched = _run_side_by_side(pics, bboxes, feeds_first_layer=True, padded=True)
    assert cuda.processed == 48 and launched == 4


# ---------------------------------------------------------------------------------------------
# the two-stage pipeline
# ---------------------------------------------------------------------------------------------
def _pictures():
    """The picture set of test_imagenet_forward: a grey picture with a bright and a dark square,
    and a plain one."""
    a = numpy.full((100, 120, 1), 110, numpy.uint8)
    a[20:60, 30:70] = 255
    a[60:90, 80:110] = 0
    b = numpy.full((80, 80, 1), 110, numpy.uint8)
    return {"pic_a.npy": a, "pic_b.npy": b}


def _candidates():
    return {
        "pic_a.npy": {"path": "pic_a.npy", "bbxs": [
            {"x": 50.0, "y": 40.0, "width": 40.0, "height": 40.0},
            {"x": 52.0, "y": 41.0, "width": 36.0, "height": 36.0},
            {"x": 48.0, "y": 38.0, "width": 30.0, "height": 30.0},
            {"x": 95.0, "y": 75.0, "width": 28.0, "height": 28.0},
            {"x": 94.0, "y": 74.0, "width": 24.0, "height": 24.0},
            {"x": 20.0, "y": 85.0, "width": 24.0, "height": 24.0},
            {"x": 3.0, "y": 3.0, "width": 4.0, "height": 4.0}]},
        "pic_b.npy": {"path": "pic_b.npy", "bbxs": [
            {"x": 40.0, "y": 40.0, "width": 30.0, "height": 30.0}]}}


def _pipeline(tmp_path, tag, normalized, device="cuda"):
    """test_two_stage_pipeline_localises_objects' hand-set 3-class softmax on cuda: returns the
    workflow, the final results and both stages' JSON."""
    from veles.znicz_b200.kernels import api
    from veles.znicz_b200.ops import all2all
    from veles.znicz_b200.utils.mean_disp_normalizer import MeanDispNormalizer
    pics = _pictures()
    out = tmp_path / tag
    out.mkdir()
    stream = out / "raw.pickle"
    with open(stream, "wb") as fout:
        for i, (k, meta) in enumerate(sorted(_candidates().items())):
            pickle.dump((i, meta), fout)
    launcher = DummyLauncher(testing=True)
    fc = all2all.All2AllSoftmax(launcher, output_sample_shape=3, weights_stddev=0.01)
    mean = numpy.full((8, 8, 1), 110.0, numpy.float32)
    norm = None
    if normalized:
        norm = MeanDispNormalizer(launcher)
        norm.mean, norm.rdisp = mean, numpy.full((8, 8, 1), 1.0 / 64, numpy.float32)
    wf = ImagenetForward(
        launcher, forwards=[fc], normalizer=norm, entry_shape=(4, 8, 8, 1), mean=mean,
        image_reader=lambda p: pics[p], result_path=str(out / "result.json"),
        labels_mapping={0: "nothing", 1: "bright", 2: "dark"},
        loader_config={"path_to_bboxes": str(stream), "minibatch_size": 4, "raw_bboxes_min_size": 8,
                       "raw_bboxes_min_area": 64, "add_relative_bboxes": False},
        merge_config={"ignore_negative": False, "use_compatibility": False,
                      "probability_threshold": 0.45, "last_chance_probability_threshold": 0.39})
    wf.initialize(device=device)
    fc.weights.map_write()
    fc.bias.map_write()
    fc.weights.mem[...] = 0
    if normalized:        # input (x - 110) / 64: the same logits as below
        fc.weights.mem[1], fc.weights.mem[2] = 0.1, -0.1
        fc.bias.mem[...] = [0.0, -5.0, -5.0]
    else:
        fc.weights.mem[1] = 0.1 / 64                                # logit = (mean - 160) / 10
        fc.weights.mem[2] = -0.1 / 64                               # logit = (60 - mean) / 10
        fc.bias.mem[...] = [0.0, -16.0, 6.0]
    if device == "cuda":
        fc.weights.unmap()
        fc.bias.unmap()
        api.refresh_weight_shadows(fc)
    final = wf.run_pipeline()
    raw = json.load(open(out / "result.json.raw"))
    return wf, final, raw, json.load(open(out / "result.json"))


def _host_rendering(self):
    self.numpy_run()
    self.minibatch_data.unmap()


@pytest.mark.gpu
@pytest.mark.parametrize("normalized", [False, True])
def test_pipeline_on_cuda_matches_host_rendering(tmp_path, monkeypatch, normalized):
    """run_pipeline in bf16 with device rendering writes the same JSON, both stages, as the same
    workflow with the shots rendered on the host, and localises both objects. Without a
    normaliser the first layer takes bf16 input; with one, the minibatch stays fp32."""
    import torch
    root.common.engine.compute_type = "bf16"
    ext = _ext()
    before = ext.render_shots_launches()
    wf, final, raw, written = _pipeline(tmp_path, "device", normalized)
    assert ext.render_shots_launches() > before
    assert wf.loader.minibatch_data.devmem.dtype == (torch.float32 if normalized else torch.bfloat16)
    with monkeypatch.context() as mp:
        mp.setattr(ForwardLoaderBbox, "cuda_run", _host_rendering)
        before = ext.render_shots_launches()
        _, h_final, h_raw, h_written = _pipeline(tmp_path, "host", normalized)
        assert ext.render_shots_launches() == before
    assert raw == h_raw and written == h_written and final == h_final
    assert {b["label"] for b in raw["pic_a.npy"]["bbxs"]} == {"bright", "dark"}
    assert wf.loader.mode == "final"
    dets = {b["label"]: b for b in final["pic_a.npy"]["bbxs"]}
    assert set(dets) == {"bright", "dark"}
    assert abs(dets["bright"]["x"] - 50) <= 4 and abs(dets["bright"]["y"] - 40) <= 4
    assert abs(dets["dark"]["x"] - 95) <= 4 and abs(dets["dark"]["y"] - 75) <= 4
    assert dets["bright"]["conf"] > 0.9
    assert "pic_b.npy" not in final or final["pic_b.npy"]["bbxs"] == []
    assert raw["pic_b.npy"]["bbxs"] == []
    assert written == final


def _conv_pipeline(tmp_path, tag):
    """Both stages with a 3x3 stride-1 conv (C = 1, so it reads the channel-padded input) under
    a softmax, over a uint8, a float and another uint8 picture: minibatches rendered on the host
    follow ones rendered on the device. Returns both stages' JSON and every minibatch's
    probabilities."""
    from veles.znicz_b200.kernels import api
    from veles.znicz_b200.ops import all2all, conv
    pics = _pictures()
    pics["pic_b.npy"] = pics["pic_b.npy"].astype(numpy.float32)
    pics["pic_c.npy"] = pics["pic_a.npy"].copy()
    cands = _candidates()
    cands["pic_c.npy"] = dict(cands["pic_a.npy"], path="pic_c.npy")
    out = tmp_path / tag
    out.mkdir()
    stream = out / "raw.pickle"
    with open(stream, "wb") as fout:
        for i, (k, meta) in enumerate(sorted(cands.items())):
            pickle.dump((i, meta), fout)
    launcher = DummyLauncher(testing=True)
    cv = conv.Conv(launcher, n_kernels=8, kx=3, ky=3, padding=(1, 1, 1, 1))
    fc = all2all.All2AllSoftmax(launcher, output_sample_shape=3)
    wf = ImagenetForward(
        launcher, forwards=[cv, fc], entry_shape=(4, 8, 8, 1),
        mean=numpy.full((8, 8, 1), 110.0, numpy.float32), image_reader=lambda p: pics[p],
        result_path=str(out / "result.json"), labels_mapping={0: "nothing", 1: "one", 2: "two"},
        loader_config={"path_to_bboxes": str(stream), "minibatch_size": 4, "raw_bboxes_min_size": 8,
                       "raw_bboxes_min_area": 64, "add_relative_bboxes": False},
        merge_config={"ignore_negative": False, "use_compatibility": False,
                      "probability_threshold": 0.0, "last_chance_probability_threshold": 0.0})
    wf.initialize(device="cuda")
    rs = numpy.random.RandomState(12)
    for unit, scale in ((cv, 0.01), (fc, 0.05)):
        for arr in (unit.weights, unit.bias):
            arr.map_write()
            arr.mem[...] = rs.normal(0, scale, arr.mem.shape)
            arr.unmap()
        api.refresh_weight_shadows(unit)
    probs = []
    merge, merge_run = wf.mergebboxes, wf.mergebboxes.run

    def record():
        n = merge.minibatch_size
        probs.append(merge.probabilities.map_read().mem[:n].copy())
        merge_run()
    merge.run = record
    wf.run_pipeline()
    return (json.load(open(out / "result.json.raw")), json.load(open(out / "result.json")),
            probs, wf)


@pytest.mark.gpu
def test_conv_first_layer_sees_every_minibatch(tmp_path, monkeypatch):
    """A bf16 conv first layer that reads the loader's channel-padded copy gets, minibatch by
    minibatch, the same probabilities out of mixed device / host rendering as out of host
    rendering alone, and both stages write the same JSON."""
    import torch
    root.common.engine.compute_type = "bf16"
    ext = _ext()
    before = ext.render_shots_launches()
    raw, final, probs, wf = _conv_pipeline(tmp_path, "device")
    assert ext.render_shots_launches() > before
    assert wf.loader.minibatch_data.__dict__.get("padded_dev_") is not None
    assert wf.loader.minibatch_data.devmem.dtype == torch.bfloat16
    with monkeypatch.context() as mp:
        mp.setattr(ForwardLoaderBbox, "cuda_run", _host_rendering)
        h_raw, h_final, h_probs, _ = _conv_pipeline(tmp_path, "host")
    assert len(probs) == len(h_probs) > 8
    for got, want in zip(probs, h_probs):
        assert got.tobytes() == want.tobytes()
    assert raw == h_raw and final == h_final
