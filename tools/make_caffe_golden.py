"""Converts the Caffe blob dumps and golden conv3 arrays that ship with the reference's test suite
(tests/functional/data/*.txt and tests/data/gd_conv_data/gd_conv3.*.npz there) into the fixtures
of tests/test_caffe_golden.py: ``tests/golden/caffe/<dump>.npz``, every blob a float32 NHWC array
(all images, nothing sampled). The text dumps carry 6 decimals, which float32 holds exactly
enough; the conv3 arrays come from a Caffe fp32 run.

usage: python tools/make_caffe_golden.py [reference tree]"""
import os
import sys

import numpy

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import install_reference  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else install_reference.SRC
DATA = os.path.join(REF, "tests", "functional", "data")
CONV3 = os.path.join(REF, "tests", "data", "gd_conv_data", "gd_conv3.")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "caffe")


def _lines(name):
    with open(os.path.join(DATA, name)) as f:
        return [l.replace("\t\n", "\n") for l in f.readlines()]


def read_blob(lines, name, shape):
    """``<name>[\\tnum:N\\tchannels:C\\theight:H\\twidth:W]`` followed by ``num:i`` / ``channels:c``
    headers and H tab-separated rows per channel plane -> [num, height, width, channels]; blobs
    named ``*_flat`` hold the whole NCHW tensor in one row."""
    start = [i for i, l in enumerate(lines) if l.rstrip("\n").split("\t")[0].strip() == name][0] + 1
    n, h, w, c = shape
    if name.endswith("_flat"):
        vals = [float(v) for v in lines[start + 2].split()]
        return numpy.array(vals).reshape(n, c, h, w).transpose(0, 2, 3, 1)
    out = numpy.zeros(shape)
    cur = start
    for pic in range(n):
        assert lines[cur].strip() == "num:%d" % pic, lines[cur]
        cur += 1
        for ch in range(c):
            assert lines[cur].strip() == "channels:%d" % ch, lines[cur]
            cur += 1
            for y in range(h):
                out[pic, y, :, ch] = [float(v) for v in lines[cur].split()]
                cur += 1
    return out


def read_vec(lines, name, width):
    """Softmax dump: per image ``num:i``, then per channel ``channels:c`` and one value."""
    start = [i for i, l in enumerate(lines) if l.strip() == name][0] + 1
    out = numpy.zeros((2, width))
    cur = start
    for pic in range(2):
        assert lines[cur].strip() == "num:%d" % pic
        cur += 1
        for ch in range(width):
            assert lines[cur].strip() == "channels:%d" % ch
            out[pic, ch] = float(lines[cur + 1].split()[0])
            cur += 2
    return out


def blobs(dump, spec):
    lines = _lines(dump + ".txt")
    return {name: read_blob(lines, name, shape) for name, shape in spec}


def main():
    x3, w3, y2, x2 = (2, 32, 32, 3), (2, 5, 5, 3), (2, 32, 32, 2), (2, 16, 16, 2)
    sets = {
        "conv": blobs("conv", [("bottom", x3), ("weights", w3), ("top", y2)]),
        "conv_grad": blobs("conv_grad", [("bottom", x3), ("weights", w3), ("top", y2),
                                         ("top_diff", y2), ("bottom_diff", x3)]),
        "pool": blobs("pool", [("bottom", y2), ("top", x2)]),
        "pool_grad": blobs("pool_grad", [("bottom", y2), ("top", x2), ("top_diff", x2),
                                         ("bottom_diff", y2)]),
        "norm_gd": blobs("norm_gd", [(n, x2) for n in ("bottom", "top", "top_diff", "bottom_diff")]),
        "conv_relu": blobs("conv_relu", [("conv_bottom", x3), ("conv_weights", w3),
                                         ("relu_top_flat", y2)]),
        "conv_relu_grad": blobs("conv_relu_grad", [
            ("relu_bottom", y2), ("relu_top_diff", y2), ("relu_bottom_diff", y2),
            ("conv_weights", w3), ("conv_bottom", x3), ("conv_bottom_diff", x3),
            ("conv_weight_delta", w3), ("relu_top_flat", y2)]),
    }
    lines = _lines("softmax.txt")
    sets["softmax"] = {"labels": read_vec(lines, "labels", 1)[:, 0],
                       "sm_bottom": read_vec(lines, "sm_bottom", 10),
                       "sm_top": read_vec(lines, "sm_top", 10),
                       "sm_bottom_diff": read_vec(lines, "sm_bottom_diff", 10)}
    sets["gd_conv3"] = {n: numpy.load(CONV3 + n + ".npz")["arr_0"]
                        for n in ("input", "weights", "bias", "output", "err_output", "err_input")}
    os.makedirs(OUT, exist_ok=True)
    for dump, d in sets.items():
        path = os.path.join(OUT, dump + ".npz")
        numpy.savez_compressed(path, **{k: numpy.asarray(a, numpy.float32) for k, a in d.items()})
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
