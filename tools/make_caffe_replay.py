"""Converts ONE iteration of the reference's Caffe CIFAR export
(/root/reference/tests/functional/data/cifar_export.tar.xz: text dumps of every layer's blobs
before/after its forward and backward pass, batch 3) into the fixtures of
tests/test_caffe_replay.py under ``tests/golden/caffe_replay/`` (the tarball is 65 MB of text and
only exists where the reference is mounted). Only the blobs the replay compares are kept; a blob
that Caffe dumps identically under several names (in-place layers, a layer's top = the next
layer's bottom) is stored once and the other names are listed in ``__aliases__``
("name=stored name"). The arrays are split over one file per group of layers so that every file
stays below 1 MB. Arrays are NHWC float32; weights keep Caffe's [F][C][ky][kx] order."""
import os
import sys
import tarfile

import numpy

SRC = "/root/reference/tests/functional/data/cifar_export.tar.xz"
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "caffe_replay")
GROUPS = {"a": ("conv1",), "b": ("pool1", "relu1", "norm1"), "c": ("conv2", "pool2", "relu2", "norm2"),
          "d": ("conv3", "pool3", "relu3", "ip1", "loss")}


def used_keys():
    keys = []
    for g in GROUPS.values():
        for n in g:
            if n in ("ip1", "loss"):
                continue
            keys += [n + "/forward/bottom_0", n + "/forward/top_0", n + "/backward/top_err_0",
                     n + "/backward/bottom_err_0"]
            if n.startswith("conv"):
                keys += [n + "/forward/blob_0", n + "/forward/blob_1"]
    return keys + ["ip1/forward/bottom_0", "ip1/forward/blob_0", "ip1/forward/blob_1",
                   "loss/forward/top_0", "ip1/backward/top_err_0", "ip1/backward/bottom_err_0"]


def parse(text):
    blobs = {}
    lines = text.split("\n")
    i = 0
    while i < len(lines):
        parts = lines[i].rstrip().split("\t")
        if len(parts) >= 5 and parts[1].startswith("num:"):
            name = parts[0]
            d = dict(p.split(":") for p in parts[1:])
            n, c, h, w = int(d["num"]), int(d["channels"]), int(d["height"]), int(d["width"])
            arr = numpy.zeros((n, c, h, w), numpy.float32)
            i += 1
            for a in range(n):
                assert lines[i].strip() == "num:%d" % a, lines[i]
                i += 1
                for b in range(c):
                    assert lines[i].strip() == "channels:%d" % b, lines[i]
                    i += 1
                    for y in range(h):
                        arr[a, b, y] = numpy.array(lines[i].split(), dtype=numpy.float64)
                        i += 1
            blobs[name] = arr
        else:
            i += 1
    return blobs


def main(iteration=0):
    out = {}
    with tarfile.open(SRC, "r:xz") as tar:
        for m in tar.getmembers():
            parts = m.name.split("/")
            if len(parts) != 3 or parts[1] != str(iteration):
                continue
            kind, layer, direction, when, _ts = parts[2].split(".")
            if when != "after":
                continue
            blobs = parse(tar.extractfile(m).read().decode())
            for name, arr in blobs.items():
                if name.startswith("blob_"):
                    if direction != "forward":
                        continue
                    val = arr                                   # weights: Caffe order
                else:
                    val = numpy.ascontiguousarray(arr.transpose(0, 2, 3, 1))   # NCHW -> NHWC
                out["%s/%s/%s" % (layer, direction, name)] = val.astype(numpy.float32)
    stored, aliases = {}, []
    for k in used_keys():
        a = out[k]
        same = [k2 for k2, a2 in stored.items() if a2.shape == a.shape and numpy.array_equal(a, a2)]
        if same:
            aliases.append("%s=%s" % (k, same[0]))
        else:
            stored[k] = a
    os.makedirs(OUT, exist_ok=True)
    for g, layers in GROUPS.items():
        part = {k: a for k, a in stored.items() if k.split("/")[0] in layers}
        if g == "a":
            part["__aliases__"] = numpy.array(aliases)
        path = os.path.join(OUT, "iter%d_%s.npz" % (iteration, g))
        numpy.savez_compressed(path, **part)
        print(path, os.path.getsize(path), len(part))


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 0)
