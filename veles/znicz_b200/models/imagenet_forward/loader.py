"""Candidate-box loader of the localisation pipeline
(/root/reference/tests/research/ImagenetAE/imagenet_forward/forward_loader.py:59-477).

For every picture and every candidate box the network sees the box content rotated by each angle
of ``[min_angle, max_angle]`` (step ``angle_step``), plain and mirrored, scaled so that the rotated
rectangle exactly fits the ``aperture x aperture`` input and alpha-blended over the training mean
image (pixels outside the box show the mean, i.e. "nothing" after normalisation).

The reference builds each shot with a chain of OpenCV calls (crop, enlarge canvas, warpAffine,
flip, crop, blend). Here ONE inverse mapping does it: for every output pixel of the aperture the
source position inside the picture is computed (undo the mirror, the scale and the rotation about
the box centre) and sampled bilinearly; coverage (inside the box AND inside the picture) is the
alpha of the blend. No OpenCV dependency, no intermediate canvases, exact centring.

On ``cuda`` the shots are rendered on the device by ``render_shots_k`` (kernels/csrc/render.cu),
bit-identical to ``render_shot``, when every picture of the minibatch is a uint8 ``[h][w][C]``
array with the network's channel count (C <= 8); any other minibatch is rendered on the host and
uploaded. Only the pictures cross PCIe, each once per stage: the pictures of the current minibatch
stay resident in a device arena, so the picture that continues from the previous minibatch is not
sent again. Each minibatch's parameter table and new pictures go through one of ``SLOTS`` pinned
slots, reused once the copies out of it have completed.
"""
from __future__ import annotations

import json
import os
import pickle

import numpy

from ...core.accelerated_units import AcceleratedUnit
from ...core.memory import Array
from ...core.mutable import Bool
from ...loader.base import channel_pad_target

# relative (x_center, y_center, width, height) boxes every picture is probed with on top of its own
# candidates in the merge stage (forward_loader.py:71-77: typical object placements)
DEFAULT_RELATIVE_BBOXES = ((0.479, 0.598, 0.319, 0.213), (0.454, 0.556, 0.501, 0.457),
                           (0.499, 0.606, 0.394, 0.3854), (0.489, 0.518, 0.672, 0.717),
                           (0.465, 0.502, 0.294, 0.708), (0.492, 0.489, 0.711, 0.447),
                           (0.503, 0.631, 0.4, 0.302))


class NoMoreShots(Exception):
    pass


def default_image_reader(path):
    """uint8 [H, W, C]; ``.npy`` arrays are taken as they are."""
    if path.endswith(".npy"):
        img = numpy.load(path)
        return img[:, :, None] if img.ndim == 2 else img
    from ...loader.image import read_image
    return read_image(path, "RGB")


def shot_geometry(bbox, angle, aperture):
    """``(ca, sa, scale, bw, bh, cx, cy)`` of one shot: cosine and sine of ``angle``, the scale
    that makes the rotated box fit ``aperture`` exactly, the box size and its centre. Both the host
    renderer and the device kernel's parameter table take them from here."""
    bw, bh = float(bbox["width"]), float(bbox["height"])
    cx, cy = float(bbox["x"]), float(bbox["y"])
    ca, sa = numpy.cos(angle), numpy.sin(angle)
    # extent of the rotated rectangle -> scale that makes it fit the aperture exactly
    ext = max(abs(bw * ca) + abs(bh * sa), abs(bw * sa) + abs(bh * ca))
    scale = aperture / max(ext, 1e-6)
    return ca, sa, scale, bw, bh, cx, cy


def shot_table_row(bbox, angle, aperture):
    """float64 ``(ca, sa, scale, bw/2, bh/2, cx, cy, 0)``: one row of ``render_shots_k``'s table."""
    ca, sa, scale, bw, bh, cx, cy = shot_geometry(bbox, angle, aperture)
    return (ca, sa, scale, bw / 2.0, bh / 2.0, cx, cy, 0.0)


def render_shot(img, bbox, angle, flip, aperture, mean):
    """One network input: the content of ``bbox`` ({x, y, width, height}, centre view) of ``img``
    [H, W, C], rotated by ``angle`` (radians, about the box centre), optionally mirrored, scaled
    to fit ``aperture`` and blended over ``mean`` [aperture, aperture, C] (float32 out)."""
    h, w = img.shape[:2]
    ca, sa, scale, bw, bh, cx, cy = shot_geometry(bbox, angle, aperture)
    u = numpy.arange(aperture, dtype=numpy.float64) - (aperture - 1) / 2.0
    ux, uy = numpy.meshgrid(-u if flip else u, u)
    # output -> box frame (undo scale, undo rotation), box frame -> picture
    bx = (ux * ca + uy * sa) / scale
    by = (-ux * sa + uy * ca) / scale
    inside = (numpy.abs(bx) <= bw / 2.0) & (numpy.abs(by) <= bh / 2.0)
    px, py = bx + cx, by + cy
    inside &= (px >= 0) & (px <= w - 1) & (py >= 0) & (py <= h - 1)
    x0 = numpy.clip(numpy.floor(px), 0, w - 2 if w > 1 else 0).astype(numpy.int64)
    y0 = numpy.clip(numpy.floor(py), 0, h - 2 if h > 1 else 0).astype(numpy.int64)
    x1, y1 = numpy.minimum(x0 + 1, w - 1), numpy.minimum(y0 + 1, h - 1)
    fx = numpy.clip(px - x0, 0.0, 1.0)[..., None]
    fy = numpy.clip(py - y0, 0.0, 1.0)[..., None]
    src = img.astype(numpy.float32)
    val = (src[y0, x0] * (1 - fx) * (1 - fy) + src[y0, x1] * fx * (1 - fy) +
           src[y1, x0] * (1 - fx) * fy + src[y1, x1] * fx * fy)
    alpha = inside[..., None].astype(numpy.float32)
    return (mean * (1.0 - alpha) + val * alpha).astype(numpy.float32)


def _align(nbytes):
    return (nbytes + 255) // 256 * 256


class ForwardLoaderBbox(AcceleratedUnit):
    """Defines ``minibatch_data``, ``minibatch_bboxes`` [(bbox, angle, flip)], ``minibatch_images``
    [(key, (height, width))], ``minibatch_size``, ``ended``, ``mode`` ("merge" for a pickled
    candidate stream, "final" for the json the merge stage wrote), ``total``.

    ``feeds_first_layer``: the minibatch goes straight into the first forward unit, so on the
    device it takes the activation dtype (bf16 under the bf16 and fp8 compute types); otherwise
    (a normaliser in between) it stays fp32. ``pictures_uploaded`` and ``h2d_bytes`` count what
    the device path sent since the last ``reset()``."""
    hide_from_registry = True
    SLOTS = 3           # pinned slots: one is filled while the copies out of the others run

    def __init__(self, workflow, bboxes_file_name=None, **kwargs):
        kwargs["view_group"] = kwargs.get("view_group", "LOADER")
        super().__init__(workflow, **kwargs)
        self.bboxes_file_name = bboxes_file_name
        self.bboxes = dict(kwargs.get("bboxes", {}))          # direct input (tests, small jobs)
        self.mode = kwargs.get("mode", "merge" if self.bboxes else "")
        self.angle_step = float(kwargs.get("angle_step", numpy.pi / 4))
        if self.angle_step <= 0:
            raise ValueError("angle_step must be positive")
        self.min_angle = float(kwargs.get("min_angle", -numpy.pi))
        self.max_angle = float(kwargs.get("max_angle", numpy.pi))
        self.min_index = int(kwargs.get("min_index", 0))
        self.max_index = int(kwargs.get("max_index", 0))
        self.only_this_file = kwargs.get("only_this_file", "")
        self.raw_bboxes_min_area = kwargs.get("raw_bboxes_min_area", 0)
        self.raw_bboxes_min_size = kwargs.get("raw_bboxes_min_size", 0)
        self.raw_bboxes_min_area_ratio = kwargs.get("raw_bboxes_min_area_ratio", 0)
        self.raw_bboxes_min_size_ratio = kwargs.get("raw_bboxes_min_size_ratio", 0)
        self.path_to_empty_images = kwargs.get("path_to_empty_images")
        self.add_relative_bboxes = kwargs.get("add_relative_bboxes", True)
        self.max_minibatch_size = int(kwargs.get("minibatch_size", 32))
        self.image_reader = kwargs.get("image_reader", default_image_reader)
        self.minibatch_data = Array()
        self.minibatch_size = 0
        self.minibatch_bboxes = []
        self.minibatch_images = []
        self.ended = Bool(False)
        self.current_image = ""
        self.total = 0
        self.processed = 0
        self.entry_shape = kwargs.get("entry_shape")
        self.mean = kwargs.get("mean")        # None: pixels outside the box are 0
        self.feeds_first_layer = kwargs.get("feeds_first_layer", False)
        self.pictures_uploaded = 0
        self.h2d_bytes = 0
        self.demand("entry_shape")

    def init_unpickled(self):
        super().init_unpickled()
        self.shots_ = None
        self.image_cache_ = (None, None)
        self.render_ = None         # device rendering state, made on the first device minibatch
                                    # and kept across stages

    # -- candidates -----------------------------------------------------------------------
    @property
    def angles(self):
        n = int(numpy.floor((self.max_angle - self.min_angle + 1e-4) / self.angle_step)) + 1
        return [self.min_angle + k * self.angle_step for k in range(max(n, 1))]

    def image_size(self, key):
        meta = self.bboxes[key]
        if meta.get("height", -1) > 0 and meta.get("width", -1) > 0:
            return int(meta["height"]), int(meta["width"])
        return tuple(self._image(key).shape[:2])

    def _image(self, key):
        if self.image_cache_[0] != key:
            self.image_cache_ = (key, self.image_reader(self.bboxes[key]["path"]))
        return self.image_cache_[1]

    def bbox_is_small(self, bbox, size):
        width, height = bbox["width"], bbox["height"]
        if width * height < max(self.raw_bboxes_min_area,
                                size[0] * size[1] * self.raw_bboxes_min_area_ratio):
            return True
        return min(width, height) < max(self.raw_bboxes_min_size,
                                        min(size) * self.raw_bboxes_min_size_ratio)

    def load_bboxes(self):
        """(Re)read the candidate file: a stream of pickled (key, {"path", "bbxs"}) pairs = merge
        stage, or the json of a previous stage = final stage."""
        if self.bboxes_file_name:
            ext = os.path.splitext(self.bboxes_file_name)[1]
            self.bboxes = {}
            if ext == ".pickle":
                self.mode = "merge"
                empty = None
                if self.path_to_empty_images and os.path.exists(self.path_to_empty_images):
                    with open(self.path_to_empty_images) as fin:
                        empty = set(line.strip() for line in fin)
                index = 0
                with open(self.bboxes_file_name, "rb") as fin:
                    while not (self.max_index > 0 and index >= self.max_index):
                        try:
                            meta = pickle.load(fin)[1]
                        except EOFError:
                            break
                        index += 1
                        if index <= self.min_index:
                            continue
                        path = meta["path"]
                        if self.only_this_file and path.find(self.only_this_file) < 0:
                            continue
                        if empty is not None and os.path.basename(path) not in empty:
                            continue
                        self.bboxes[path] = dict(meta, bbxs=list(meta["bbxs"]))
            elif ext == ".json":
                self.mode = "final"
                with open(self.bboxes_file_name) as fin:
                    self.bboxes = {val["path"]: val for val in json.load(fin).values()}
            else:
                raise ValueError("%s: expected .pickle (merge stage) or .json (final stage)" %
                                 self.bboxes_file_name)
        if self.mode == "merge" and self.add_relative_bboxes:
            for key, meta in self.bboxes.items():
                if meta.get("relative_added_"):
                    continue
                h, w = self.image_size(key)
                meta["bbxs"] = list(meta["bbxs"]) + [
                    {"x": float(numpy.round(rx * w)), "y": float(numpy.round(ry * h)),
                     "width": float(numpy.round(rw * w)), "height": float(numpy.round(rh * h))}
                    for rx, ry, rw, rh in DEFAULT_RELATIVE_BBOXES]
                meta["relative_added_"] = True
        self.total = sum(len(m["bbxs"]) for m in self.bboxes.values()) * 2 * len(self.angles)

    def _shots(self):
        for key in sorted(self.bboxes):
            size = self.image_size(key)
            for bbox in self.bboxes[key]["bbxs"]:
                if self.bbox_is_small(bbox, size):
                    self.processed += 2 * len(self.angles)
                    continue
                for flip in (False, True):
                    for angle in self.angles:
                        yield key, size, bbox, angle, flip

    def reset(self):
        self.processed = 0
        self.load_bboxes()
        self.shots_ = self._shots()
        self.ended <<= False
        if self.render_ is not None:
            # a new stage: the mean, the table and the pinned slots stay, every picture goes up
            # again when its shots come
            self.render_["resident"] = {}
        self.pictures_uploaded = 0
        self.h2d_bytes = 0

    # -- unit life cycle --------------------------------------------------------------------
    def initialize(self, device=None, **kwargs):
        super().initialize(device=device, **kwargs)
        shape = list(self.entry_shape)
        shape[0] = self.max_minibatch_size
        self.aperture, self.channels = int(shape[1]), int(shape[3])
        if shape[1] != shape[2]:
            raise ValueError("square network input expected, got %s" % (shape,))
        if not self.minibatch_data or tuple(self.minibatch_data.shape) != tuple(shape):
            self.minibatch_data.reset(numpy.zeros(shape, dtype=numpy.float32))
        if self.on_cuda:
            from ...ops.nn_units import torch_act_dtype
            dt = torch_act_dtype() if self.feeds_first_layer else None
            if self.minibatch_data.dev_dtype != dt:
                self.minibatch_data.reset(self.minibatch_data.mem)    # reallocated in that dtype
                self.minibatch_data.dev_dtype = dt
        self.init_vectors(self.minibatch_data)
        self.minibatch_bboxes = [None] * self.max_minibatch_size
        self.minibatch_images = [None] * self.max_minibatch_size
        self.render_ = None         # sized for this minibatch, made on the first device minibatch
        self.reset()

    def _mean_image(self):
        m = self.mean.mem if hasattr(self.mean, "mem") else self.mean
        if m is None:
            return numpy.zeros((self.aperture, self.aperture, self.channels), numpy.float32)
        return numpy.asarray(m, dtype=numpy.float32).reshape(self.aperture, self.aperture,
                                                             self.channels)

    def take_shots(self):
        """The next minibatch's shots ``[(key, picture, bbox, angle, flip)]``; fills
        ``minibatch_bboxes``, ``minibatch_images``, ``minibatch_size`` and advances ``processed``
        and ``ended``. The pictures are read in the same order as the shots are taken."""
        if self.ended:
            raise NoMoreShots()
        shots = []
        while len(shots) < self.max_minibatch_size:
            try:
                key, size, bbox, angle, flip = next(self.shots_)
            except StopIteration:
                self.ended <<= True
                break
            self.current_image = key
            n = len(shots)
            shots.append((key, self._image(key), bbox, angle, flip))
            self.minibatch_bboxes[n] = (bbox, angle, flip)
            self.minibatch_images[n] = (key, size)
            self.processed += 1
        self.minibatch_size = len(shots)
        if self.ended:
            self.image_cache_ = (None, None)
        return shots

    def render_host(self, shots):
        """``render_shot`` of each shot into the host ``minibatch_data`` (rows past the shots
        keep what they held)."""
        self.minibatch_data.map_invalidate()
        mean = self._mean_image()
        for n, (_key, img, bbox, angle, flip) in enumerate(shots):
            self.minibatch_data.mem[n] = render_shot(img, bbox, angle, flip, self.aperture, mean)

    def numpy_run(self):
        self.render_host(self.take_shots())

    def cuda_run(self):
        shots = self.take_shots()
        if self.device_renders(shots):
            self.render_device(shots)
        else:
            self.render_host(shots)
            md = self.minibatch_data
            md.unmap()
            # the first conv layer takes the channel-padded copy as current once the loader has
            # made one (the device path writes it with the minibatch), so keep it current here too
            pad = channel_pad_target(md)
            if pad is not None:
                self.device.ext.pad_channels(md.devmem, pad, self.channels, pad.shape[3])

    # -- cuda: shots rendered on the device --------------------------------------------------
    def device_renders(self, shots):
        """Whether ``render_shots_k`` renders these shots: every picture uint8 ``[h][w][C]``
        with the network's C (at most 8) and a fp32 or bf16 device minibatch."""
        import torch
        md = self.minibatch_data
        if md.devmem is None or md.devmem.dtype not in (torch.float32, torch.bfloat16) or \
                self.channels > 8:
            return False
        return all(isinstance(img, numpy.ndarray) and img.dtype == numpy.uint8 and img.ndim == 3
                   and img.shape[2] == self.channels and img.size > 0
                   for _key, img, _bbox, _angle, _flip in shots)

    def _render_setup(self):
        import torch
        dev = self.device.torch_device
        mb = self.max_minibatch_size
        off = {"shots": 256}                         # header: 16 bytes of int32, n first
        off["pics"] = _align(off["shots"] + 64 * mb)
        tab = _align(off["pics"] + 32 * mb)

        def views(buf):
            return {"hdr": buf[:16].view(torch.int32),
                    "shots": buf[off["shots"]:off["shots"] + 64 * mb].view(torch.float64).view(mb, 8),
                    "pics": buf[off["pics"]:off["pics"] + 32 * mb].view(torch.int64).view(mb, 4)}
        rs = {"tab": tab, "dev": torch.zeros(tab, dtype=torch.uint8, device=dev),
              "arena": torch.zeros(0, dtype=torch.uint8, device=dev),
              "resident": {},                      # key -> byte offset in the arena
              "mean": torch.from_numpy(self._mean_image()).to(dev),
              "slots": [None] * self.SLOTS, "i": 0, "views": views}
        rs["dv"] = views(rs["dev"])
        self.render_ = rs
        return rs

    def _render_slot(self, rs, nbytes):
        """The next pinned slot, its copies done, holding at least ``nbytes``."""
        import torch
        i = rs["i"]
        rs["i"] = (i + 1) % self.SLOTS
        sl = rs["slots"][i]
        if sl is not None:
            sl["event"].synchronize()
        if sl is None or sl["pin"].numel() < nbytes:
            pin = torch.zeros(_align(nbytes), dtype=torch.uint8).pin_memory()
            v = rs["views"](pin)
            sl = {"pin": pin, "buf": pin.numpy(), "event": torch.cuda.Event(),
                  "hdr": v["hdr"].numpy(), "shots": v["shots"].numpy(), "pics": v["pics"].numpy()}
            rs["slots"][i] = sl
        return sl

    def render_device(self, shots):
        import torch
        rs = self.render_ or self._render_setup()
        tab = rs["tab"]
        pictures = {}
        for key, img, _bbox, _angle, _flip in shots:
            pictures.setdefault(key, img)
        # pictures resident since the previous minibatch stay where they are; the new ones are
        # packed before or after them
        kept = {k: rs["resident"][k] for k in pictures if k in rs["resident"]}
        new = [k for k in pictures if k not in kept]
        total = sum(pictures[k].nbytes for k in new)
        lo = min(kept.values(), default=0)
        hi = max((o + pictures[k].nbytes for k, o in kept.items()), default=0)
        base = 0 if total <= lo else hi
        arena = rs["arena"]
        if base + total > arena.numel():
            grown = torch.empty(max(base + total, 2 * arena.numel()), dtype=torch.uint8,
                                device=arena.device)
            if hi > lo:
                grown[lo:hi].copy_(arena[lo:hi])
            arena = rs["arena"] = grown
        sl = self._render_slot(rs, tab + total)
        resident = dict(kept)
        at = base
        for k in new:
            img = pictures[k]
            sl["buf"][tab + at - base:tab + at - base + img.nbytes] = img.reshape(-1)
            resident[k] = at
            at += img.nbytes
        n = len(shots)
        sl["hdr"][0] = n
        for r, (key, img, bbox, angle, flip) in enumerate(shots):
            sl["shots"][r] = shot_table_row(bbox, angle, self.aperture)
            sl["pics"][r] = (resident[key], img.shape[0], img.shape[1], int(bool(flip)))
        sl["shots"][n:] = 0
        sl["pics"][n:] = 0
        rs["dev"].copy_(sl["pin"][:tab], non_blocking=True)
        if total:
            arena[base:base + total].copy_(sl["pin"][tab:tab + total], non_blocking=True)
        sl["event"].record()
        rs["resident"] = resident
        self.pictures_uploaded += len(new)
        self.h2d_bytes += tab + total
        md = self.minibatch_data
        dv = rs["dv"]
        self.device.ext.render_shots(arena, dv["hdr"], dv["shots"], dv["pics"], rs["mean"],
                                     md.devmem, channel_pad_target(md))
        md.dev_written()
