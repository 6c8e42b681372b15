"""ImageNet loaders on the GPU: crop, mirror and mean subtraction of uint8 samples in one kernel
(csrc/augment.cu), streamed through a pinned slot or gathered from HBM, against the numpy path."""
import json
import pickle

import numpy
import pytest

from veles.znicz_b200.core.config import root
from veles.znicz_b200.core.prng import RandomGenerator
from veles.znicz_b200.core.workflow import DummyWorkflow
from veles.znicz_b200.loader.base import TEST, VALID, TRAIN
from veles.znicz_b200.loader.imagenet_loader import ImagenetLoaderBase, ImagenetLoader


def _write_dataset(path, counts, sy, sx, c, mean=True, seed=11):
    """samples.dat / labels.pickle / count.json (/ matrixes.pickle) as utils/preparation_imagenet
    writes them; returns the loader kwargs and the samples."""
    rs = numpy.random.RandomState(seed)
    n = sum(counts)
    samples = rs.randint(0, 256, (n, sy, sx, c)).astype(numpy.uint8)
    samples.tofile(str(path / "samples.dat"))
    with open(path / "labels.pickle", "wb") as f:
        pickle.dump([("n%04d" % (i % 7), i % 7) for i in range(n)], f)
    with open(path / "count.json", "w") as f:
        json.dump({"test": counts[0], "val": counts[1], "train": counts[2]}, f)
    kw = dict(sy=sy, sx=sx, channels=c, original_labels_filename=str(path / "labels.pickle"),
              count_samples_filename=str(path / "count.json"),
              samples_filename=str(path / "samples.dat"))
    if mean:
        m = samples[counts[0] + counts[1]:].mean(axis=0)        # float64, as the tools write it
        with open(path / "matrixes.pickle", "wb") as f:
            pickle.dump([m, 1.0 / (samples.std(axis=0) + 1.0)], f)
        kw["matrixes_filename"] = str(path / "matrixes.pickle")
    return kw, samples


class _OldTransform(ImagenetLoader):
    """The numpy transform_batch as it was before augment_params existed, recording its draws."""
    hide_from_registry = True

    def transform_batch(self, raw):
        n = raw.shape[0]
        x = raw.astype(numpy.float32)
        if self.has_mean_file:
            x -= self.mean.mem.astype(x.dtype)
        cy, cx = self.final_sy, self.final_sx
        hs = numpy.full(n, (self.sy - cy) // 2)
        ws = numpy.full(n, (self.sx - cx) // 2)
        flip = numpy.zeros(n, bool)
        if (cy, cx) != (self.sy, self.sx):
            if self.minibatch_class == TRAIN:
                st = self.prng.state if hasattr(self.prng, "state") else numpy.random
                hs = st.randint(0, self.sy - cy + 1, n)
                ws = st.randint(0, self.sx - cx + 1, n)
            rows = hs[:, None] + numpy.arange(cy)[None, :]
            cols = ws[:, None] + numpy.arange(cx)[None, :]
            x = x[numpy.arange(n)[:, None, None], rows[:, :, None], cols[:, None, :]]
        if self.mirror and self.minibatch_class == TRAIN:
            st = self.prng.state if hasattr(self.prng, "state") else numpy.random
            flip = st.randint(0, 2, n).astype(bool)
            x[flip] = x[flip][:, :, ::-1]
        self.draws = numpy.stack([hs, ws, flip.astype(numpy.int64)], axis=1).astype(numpy.int32)
        return x


class _Recording(ImagenetLoader):
    hide_from_registry = True

    def augment_params(self, n):
        self.draws = super().augment_params(n)
        return self.draws


def _kernel_model(samples, idx, params, mean, cy, cx, max_rows):
    """numpy statement of the augment_minibatch_k contract (fp32 output)."""
    n = len(idx)
    out = numpy.zeros((max_rows, cy, cx, samples.shape[3]), numpy.float32)
    for r in range(n):
        y0, x0, f = params[r]
        for x in range(cx):
            xs = x0 + (cx - 1 - x if f else x)
            v = samples[idx[r], y0:y0 + cy, xs].astype(numpy.float32)
            if mean is not None:
                v = v - mean[y0:y0 + cy, xs]
            out[r, :, x] = v
    return out


@pytest.mark.parametrize("crop,mirror", [((9, 11), True), ((9, 11), False), ((12, 14), True)])
@pytest.mark.parametrize("counts", [(3, 6, 20), (0, 0, 13)])
def test_augment_params_reproduce_old_transform_draws(tmp_path, crop, mirror, counts):
    kw, samples = _write_dataset(tmp_path, counts, 12, 14, 3)
    common = dict(kw, minibatch_size=4, crop_size_sy=crop[0], crop_size_sx=crop[1], mirror=mirror)
    old = _OldTransform(DummyWorkflow(), prng=RandomGenerator(seed=21), **common)
    new = _Recording(DummyWorkflow(), prng=RandomGenerator(seed=21), **common)
    old.initialize(device="numpy")
    new.initialize(device="numpy")
    classes = set()
    mean = new.mean.mem.astype(numpy.float32) if new.has_mean_file else None
    for _ in range(3 * 9):                     # three epochs
        old.run()
        new.run()
        classes.add(new.minibatch_class)
        n = int(new.minibatch_size)
        assert old.minibatch_class == new.minibatch_class and n == int(old.minibatch_size)
        numpy.testing.assert_array_equal(new.draws, old.draws)
        assert new.draws.dtype == numpy.int32 and new.draws.shape == (n, 3)
        numpy.testing.assert_array_equal(new.minibatch_data.mem, old.minibatch_data.mem)
        numpy.testing.assert_array_equal(new.minibatch_labels.mem, old.minibatch_labels.mem)
        idx = new.minibatch_indices.mem[:n]
        want = _kernel_model(samples, idx, new.draws, mean, crop[0], crop[1], 4)
        numpy.testing.assert_array_equal(new.minibatch_data.mem, want)
    assert old.prng.state.randint(1 << 30) == new.prng.state.randint(1 << 30)
    assert classes == {c for c, k in zip((TEST, VALID, TRAIN), counts) if k}


def test_raw_loader_params_are_zero(tmp_path):
    kw, samples = _write_dataset(tmp_path, (0, 2, 5), 6, 5, 1, mean=False)
    ld = ImagenetLoaderBase(DummyWorkflow(), minibatch_size=3, **kw)
    ld.initialize(device="numpy")
    assert not ld.augment_params(3).any()
    ld.run()
    numpy.testing.assert_array_equal(
        ld.minibatch_data.mem[:2], _kernel_model(samples, ld.minibatch_indices.mem[:2],
                                                 ld.augment_params(2), None, 6, 5, 3)[:2])


@pytest.mark.parametrize("shape", [(7, 5, 3), (4, 4, 4), (1, 1, 1)])
def test_native_raw_row_gather_and_prefetch(shape):
    import torch
    from veles.znicz_b200.kernels import load_extension
    ext = load_extension(required=True)
    rs = numpy.random.RandomState(5)
    data = rs.randint(0, 256, (37,) + shape).astype(numpy.uint8)
    src = torch.from_numpy(data)
    for n, cap in ((9, 12), (12, 12), (0, 3)):
        idx = rs.randint(0, 37, cap).astype(numpy.int32)
        idx[:2] = (-5, 99)                     # clamped, as in the fp32 gather
        want = numpy.zeros((cap,) + shape, numpy.uint8)
        numpy.take(data, idx[:n], axis=0, out=want[:n], mode="clip")
        dst = torch.full((cap,) + shape, 0xAB, dtype=torch.uint8)
        ext.host_gather_rows(src, torch.from_numpy(idx), dst, n)
        numpy.testing.assert_array_equal(dst.numpy(), want)
        dst.fill_(0xCD)
        ticket = ext.host_prefetch_submit(src, torch.from_numpy(idx), dst, n)
        ext.host_prefetch_wait(ticket)
        numpy.testing.assert_array_equal(dst.numpy(), want)
    with pytest.raises(RuntimeError):
        ext.host_gather_rows(src, torch.zeros(3, dtype=torch.int32),
                             torch.zeros((3,) + shape, dtype=torch.float32), 3)


# ------------------------------------------------------------------------------------- GPU
_COUNTS = (0, 8, 26)      # 8 VALID + 26 TRAIN, minibatch 6: both classes end on a short minibatch


def _twins(tmp_path, cls=ImagenetLoader, c=3, mean=True, on_device=False, seed=33, **extra):
    kw, samples = _write_dataset(tmp_path, _COUNTS, 40, 36, c, mean=mean)
    kw.update(minibatch_size=6, **extra)
    ref = cls(DummyWorkflow(), prng=RandomGenerator(seed=seed), **kw)
    dut = cls(DummyWorkflow(), prng=RandomGenerator(seed=seed), on_device=on_device, **kw)
    ref.initialize(device="numpy")
    dut.initialize(device="cuda")
    return ref, dut, samples


_CASES = [  # (loader, crop, C, mean)
    ("aug", (27, 23), 3, True), ("aug", (27, 23), 3, False), ("base", None, 3, True),
    ("aug", (40, 36), 3, True), ("aug", (27, 23), 1, True), ("base", None, 1, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", _CASES, ids=lambda c: "%s-%s-c%d-%s" % (
    c[0], "x".join(map(str, c[1])) if c[1] else "full", c[2], "mean" if c[3] else "nomean"))
@pytest.mark.parametrize("resident", [False, True], ids=["streamed", "resident"])
@pytest.mark.parametrize("compute", ["bf16", "fp32"])
def test_cuda_loader_matches_numpy_bit_for_bit(tmp_path, case, resident, compute):
    import torch
    root.common.engine.compute_type = compute
    kind, crop, c, mean = case
    extra = {} if kind == "base" else dict(crop_size_sy=crop[0], crop_size_sx=crop[1], mirror=True)
    cls = ImagenetLoaderBase if kind == "base" else ImagenetLoader
    ref, dut, _ = _twins(tmp_path, cls, c, mean, resident, **extra)
    assert dut._aug_ is not None
    ext = dut.device.ext
    dtype = torch.bfloat16 if compute == "bf16" else torch.float32
    assert dut.minibatch_data.devmem.dtype == dtype
    mb = 6
    if resident:
        assert dut.h2d_bytes_per_step < 1024
    else:
        assert dut.h2d_bytes_per_step >= mb * 40 * 36 * c
    ragged = 0
    for step in range(2 * 7):
        before = ext.augment_launches()
        ref.run()
        dut.run()
        assert ext.augment_launches() == before + 1
        assert (dut.minibatch_class, dut.minibatch_size) == (ref.minibatch_class, ref.minibatch_size)
        ragged += int(ref.minibatch_size) < mb
        want = torch.from_numpy(ref.minibatch_data.mem).to(dtype).cuda()
        got = dut.minibatch_data.devmem
        assert got.shape == want.shape and torch.equal(got, want), step
        assert torch.equal(dut.minibatch_labels.devmem.cpu(),
                           torch.from_numpy(ref.minibatch_labels.mem)), step
        dut.minibatch_data.map_read()          # a host reader sees the augmented batch
        assert numpy.array_equal(dut.minibatch_data.mem,
                                 want.float().cpu().numpy()), step
    assert ragged == 4
    dut.stop()


def _tiny_layers():
    return [
        {"name": "conv1", "type": "conv",
         "->": {"n_kernels": 8, "kx": 5, "ky": 5, "sliding": (1, 1), "padding": (0, 0, 0, 0),
                "weights_filling": "gaussian", "weights_stddev": 0.05},
         "<-": {"learning_rate": 0.01, "gradient_moment": 0.9}},
        {"name": "pool1", "type": "max_pooling", "->": {"kx": 3, "ky": 3, "sliding": (2, 2)}},
        {"name": "fc", "type": "softmax",
         "->": {"output_sample_shape": 7, "weights_filling": "gaussian", "weights_stddev": 0.05},
         "<-": {"learning_rate": 0.01, "gradient_moment": 0.9}}]


def _tiny_workflow(kw, graphs, seed, max_epochs=2):
    from veles.znicz_b200.core import prng
    from veles.znicz_b200.models import alexnet
    prng.get(1).seed(1234)
    prng.get(2).seed(5678)
    return alexnet.build(
        loader_name="imagenet_pickle_loader", layers=_tiny_layers(), use_graphs=graphs,
        loader_config=dict(kw, prng=RandomGenerator(seed=seed)),
        decision_config={"max_epochs": max_epochs, "fail_iterations": 100},
        snapshotter_config={"prefix": "inet_aug", "interval": 1000, "time_interval": 1e9})


@pytest.mark.gpu
def test_graph_replay_serves_the_twin_minibatch_and_trains_like_eager(tmp_path):
    """The augmentation runs as the prelude of the captured forward graph: after the run the
    device minibatch (and the first conv's channel-padded copy) is the numpy twin's last one, and
    the weights equal those of the same run without graphs, bit for bit."""
    import torch
    root.common.engine.compute_type = "bf16"
    kw, _ = _write_dataset(tmp_path, _COUNTS, 40, 36, 3)
    kw.update(minibatch_size=6, crop_size_sy=27, crop_size_sx=23, mirror=True)
    weights = {}
    for graphs in (True, False):
        wf = _tiny_workflow(kw, graphs, seed=44)
        wf.initialize(device="cuda")
        ld = getattr(wf, "real_loader", None) or wf.loader
        assert ld._aug_ is not None
        wf.run()
        torch.cuda.synchronize()
        assert bool(wf.decision.complete)
        if graphs:
            assert ld.__dict__.get("augment_in_graph_")
            assert all(s.replays > 0 for s in wf.segments_), [
                (s.name, s.replays, s.eager_runs) for s in wf.segments_]
            twin = ImagenetLoader(DummyWorkflow(), prng=RandomGenerator(seed=44), **kw)
            twin.initialize(device="numpy")
            while twin.samples_served < ld.samples_served:
                twin.run()
            assert (twin.epoch_number, twin.global_offset) == (ld.epoch_number, ld.global_offset)
            md = ld.minibatch_data
            want = torch.from_numpy(twin.minibatch_data.mem).to(torch.bfloat16).cuda()
            assert torch.equal(md.devmem, want)
            pad = md.__dict__.get("padded_dev_")
            assert pad is not None and tuple(pad.shape) == (6, 27, 23, 8)
            assert torch.equal(pad[..., :3], want) and not pad[..., 3:].any()
        weights[graphs] = []
        for f in wf.forwards:
            if getattr(f, "weights", None):
                f.weights.map_read()
                weights[graphs].append(f.weights.mem.copy())
        ld.stop()
    for a, b in zip(weights[True], weights[False]):
        assert numpy.array_equal(a, b)


@pytest.mark.gpu
def test_resident_dataset_past_two_gigabytes(tmp_path):
    """Sample offsets are 64-bit: a sparse 256x256x3 file of 11000 samples (2.16e9 bytes), random
    bytes only in the rows read, the last one included."""
    import torch
    root.common.engine.compute_type = "fp32"
    n, sy, sx, c = 11000, 256, 256, 3
    row = sy * sx * c
    assert n * row > 2 ** 31
    rows = [0, 10922, 10923, n - 1]
    rs = numpy.random.RandomState(8)
    content = {}
    with open(tmp_path / "samples.dat", "wb") as f:
        f.truncate(n * row)
        for r in rows:
            content[r] = rs.randint(0, 256, (sy, sx, c)).astype(numpy.uint8)
            f.seek(r * row)
            f.write(content[r].tobytes())
    with open(tmp_path / "labels.pickle", "wb") as f:
        pickle.dump([("n%d" % (i % 3), i % 3) for i in range(n)], f)
    with open(tmp_path / "count.json", "w") as f:
        json.dump({"test": 0, "val": n, "train": 0}, f)
    ld = ImagenetLoader(DummyWorkflow(), minibatch_size=4, shuffle_limit=0, on_device=True,
                        sy=sy, sx=sx, channels=c, crop_size_sy=227, crop_size_sx=227,
                        original_labels_filename=str(tmp_path / "labels.pickle"),
                        count_samples_filename=str(tmp_path / "count.json"),
                        samples_filename=str(tmp_path / "samples.dat"))
    ld.initialize(device="cuda")
    assert ld._aug_ is not None and ld._aug_["src"].numel() == n * row
    ld.shuffled_indices.mem[:4] = rows
    ld.run()
    want = numpy.stack([content[r][14:241, 14:241] for r in rows]).astype(numpy.float32)
    assert torch.equal(ld.minibatch_data.devmem.cpu(), torch.from_numpy(want))
    assert ld.minibatch_labels.devmem.cpu().tolist() == [r % 3 for r in rows]


@pytest.mark.gpu
def test_snapshot_of_device_path_workflow_restores(tmp_path):
    import torch
    from veles.znicz_b200.core.workflow import DummyLauncher
    root.common.engine.compute_type = "bf16"
    kw, _ = _write_dataset(tmp_path, _COUNTS, 40, 36, 3)
    kw.update(minibatch_size=6, crop_size_sy=27, crop_size_sx=23, mirror=True)
    # without graphs: the loader's run() then launches the augmentation itself
    wf = _tiny_workflow(kw, False, seed=55)
    wf.initialize(device="cuda")
    assert wf.loader._aug_ is not None
    wf2 = pickle.loads(pickle.dumps(wf))
    wf2.workflow = DummyLauncher()
    wf2.initialize(device="cuda", snapshot=True)
    ld = getattr(wf2, "real_loader", None) or wf2.loader
    assert ld._aug_ is not None
    twin = ImagenetLoader(DummyWorkflow(), prng=RandomGenerator(seed=55), **kw)
    twin.initialize(device="numpy")
    before = ld.device.ext.augment_launches()
    for _ in range(3):
        ld.run()
        twin.run()
        want = torch.from_numpy(twin.minibatch_data.mem).to(torch.bfloat16).cuda()
        assert torch.equal(ld.minibatch_data.devmem, want)
    assert ld.device.ext.augment_launches() == before + 3
    ld.stop()
