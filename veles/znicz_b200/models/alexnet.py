"""ImageNet models: AlexNet (with 2-group ``zero_filter`` grouping), Network-in-Network and
the 13-conv VGG variant, plus the ImageNet workflow.

Parity: /root/reference/tests/research/AlexNet/imagenet_workflow.py:168-208 (workflow:
snapshotter → plotters → GDs → LR adjuster → loop) and the three layer configs
imagenet_workflow_config.py:94-250, imagenet_workflow_nin_config.py,
imagenet_workflow_vgga_config.py, and the LMDB variant imagenet_workflow_lmdb_config.py.
The layer lists are generated from compact tables instead of being spelled out.

H100: on the CUDA backend all conv/FC layers run on the wgmma implicit-GEMM kernels in
bf16 with fp32 accumulation; FC6 (9216x4096) is the tensor the two-shot fused reduce+update
exists for in data-parallel runs.
"""
from __future__ import annotations

import os

from ..core.config import root
from ..workflow.standard_workflow import StandardWorkflow

BASE_LR, WD = 0.01, 0.0005


def _gd(lr=BASE_LR, wd=WD, ortho=0.001, bias_wd=0.0):
    return {"learning_rate": lr, "learning_rate_bias": lr * 2, "weights_decay": wd,
            "weights_decay_bias": bias_wd, "factor_ortho": ortho, "gradient_moment": 0.9,
            "gradient_moment_bias": 0.9}


def _conv(name, tpe, n, k, stride=1, pad=0, std=0.01, bias=0.0, filling="gaussian", gd=None):
    return {"name": name, "type": tpe,
            "->": {"n_kernels": n, "kx": k, "ky": k, "padding": (pad,) * 4,
                   "sliding": (stride, stride), "weights_filling": filling,
                   "weights_stddev": std, "bias_filling": "constant", "bias_stddev": bias},
            "<-": dict(gd or _gd())}


def _pool(name, k, stride, tpe="max_pooling"):
    return {"name": name, "type": tpe, "->": {"kx": k, "ky": k, "sliding": (stride, stride)}}


def _fc(name, n, std, bias, tpe="all2all", gd=None):
    return {"name": name, "type": tpe,
            "->": {"output_sample_shape": n, "weights_filling": "gaussian",
                   "weights_stddev": std, "bias_filling": "constant", "bias_stddev": bias},
            "<-": dict(gd or _gd())}


def alexnet_layers(n_classes=1000):
    norm = {"n": 5, "alpha": 0.0001, "beta": 0.75}
    return [
        _conv("conv_str1", "conv_str", 96, 11, 4, 0, 0.01, 0),
        _pool("max_pool1", 3, 2), dict(name="norm1", type="norm", **norm),
        {"name": "grouping1", "type": "zero_filter", "grouping": 2},
        _conv("conv_str2", "conv_str", 256, 5, 1, 2, 0.01, 0.1),
        _pool("max_pool2", 3, 2), dict(name="norm2", type="norm", **norm),
        {"name": "grouping2", "type": "zero_filter", "grouping": 2},
        _conv("conv_str3", "conv_str", 384, 3, 1, 1, 0.01, 0),
        _conv("conv_str4", "conv_str", 384, 3, 1, 1, 0.01, 0.1),
        {"name": "grouping4", "type": "zero_filter", "grouping": 2},
        _conv("conv_str5", "conv_str", 256, 3, 1, 1, 0.01, 0.1),
        _pool("max_pool5", 3, 2),
        {"name": "grouping5", "type": "zero_filter", "grouping": 2},
        _fc("fc_linear6", 4096, 0.005, 0.1), {"name": "relu6", "type": "activation_str"},
        {"name": "drop6", "type": "dropout", "dropout_ratio": 0.5},
        _fc("fc_linear7", 4096, 0.005, 0.1), {"name": "relu7", "type": "activation_str"},
        {"name": "drop7", "type": "dropout", "dropout_ratio": 0.5},
        _fc("fc_softmax8", n_classes, 0.01, 0, "softmax", _gd(ortho=0.0))]


def nin_layers(n_classes=1000, filling="gaussian", lr=0.01):
    g = _gd(lr, ortho=0.0)
    layers = []
    spec = [  # (n, k, stride, pad, std) ... "P" = max-pool 3/2, "D" = dropout
        (96, 11, 4, 0, 0.01), (96, 1, 1, 0, 0.05), (96, 1, 1, 0, 0.05), "P",
        (256, 5, 1, 2, 0.05), (256, 1, 1, 0, 0.05), (256, 1, 1, 0, 0.05), "P",
        (384, 3, 1, 1, 0.01), (384, 1, 1, 0, 0.05), (384, 1, 1, 0, 0.05), "P", "D",
        (1024, 3, 1, 1, 0.05), (1024, 1, 1, 0, 0.05), (n_classes, 1, 1, 0, 0.01)]
    i = 0
    for item in spec:
        if item == "P":
            layers.append(_pool("pool%d" % i, 3, 2))
        elif item == "D":
            layers.append({"name": "drop%d" % i, "type": "dropout", "dropout_ratio": 0.5})
        else:
            i += 1
            n, k, s, p, std = item
            layers.append(_conv("conv%d" % i, "conv", n, k, s, p, std, 0, filling, g))
            layers.append({"name": "relu%d" % i, "type": "activation_str"})
    layers.append(_pool("pool%d" % i, 6, 1, "avg_pooling"))
    layers.append(_fc("fc_softmax%d" % (i + 1), n_classes, 0.01, 0, "softmax", g))
    return layers


def vgga_layers(n_classes=1000):
    g = {"learning_rate": 0.01, "learning_rate_bias": 0.02}
    g2 = {"learning_rate": 0.001, "learning_rate_bias": 0.002}
    layers, i = [], 0
    for n, reps in ((64, 2), (128, 2), (256, 3), (512, 3), (512, 3)):
        for _ in range(reps):
            i += 1
            layers.append(_conv("conv_str%d" % i, "conv_str", n, 3, 1, 1, 0.01, 0, gd=g))
        layers.append(_pool("max_pool%d" % i, 2, 2))
    for j, gd_ in ((i + 1, g), (i + 2, g2)):
        layers.append(_fc("fc_linear%d" % j, 4096, 0.005, 0, gd=gd_))
        layers.append({"name": "relu%d" % j, "type": "activation_str"})
        layers.append({"name": "drop%d" % j, "type": "dropout", "dropout_ratio": 0.5})
    layers.append(_fc("fc_softmax%d" % (i + 3), n_classes, 0.01, 0, "softmax", g2))
    return layers


_root_path = os.path.join(str(root.common.dirs.datasets), "AlexNet", "imagenet")
_steps = {"lrs_with_lengths": [(1, 100000), (0.1, 100000), (0.1, 100000), (0.01, 100000000)]}
root.imagenet.update({
    "root_name": "imagenet", "series": "img", "root_path": _root_path,
    "decision": {"fail_iterations": 10000, "max_epochs": 10000},
    "snapshotter": {"prefix": "imagenet", "interval": 1, "time_interval": 0},
    "add_plotters": False,
    "loss_function": "softmax",
    "lr_adjuster": {"lr_policy_name": "arbitrary_step", "bias_lr_policy_name": "arbitrary_step",
                    "lr_parameters": dict(_steps), "bias_lr_parameters": dict(_steps)},
    "image_saver": {"out_dirs": [os.path.join(_root_path, "image_saver", d)
                                 for d in ("test", "validation", "train")]},
    "loader_name": "imagenet_pickle_loader",
    "loader": {"sx": 256, "sy": 256, "crop_size_sx": 227, "crop_size_sy": 227, "mirror": True,
               "channels": 3, "minibatch_size": 256, "normalization_type": "none",
               "shuffle_limit": 1,
               "original_labels_filename": os.path.join(
                   _root_path, "original_labels_imagenet_img.pickle"),
               "samples_filename": os.path.join(_root_path, "original_data_imagenet_img.dat"),
               "matrixes_filename": os.path.join(_root_path, "matrixes_imagenet_img.pickle"),
               "count_samples_filename": os.path.join(
                   _root_path, "count_samples_imagenet_img.json")},
    "weights_plotter": {"limit": 256, "split_channels": False},
    "layers": alexnet_layers()})

# the LMDB flavour of the same experiment (imagenet_workflow_lmdb_config.py)
LMDB_LOADER = {"loader_name": "lmdb",
               "loader": {"minibatch_size": 256, "normalization_type": "internal_mean",
                          "train_path": os.path.join(_root_path, "ilsvrc12_train_lmdb"),
                          "validation_path": os.path.join(_root_path, "ilsvrc12_val_lmdb"),
                          "crop": (227, 227), "mirror": "random"}}


class ImagenetWorkflow(StandardWorkflow):
    def create_workflow(self):
        self.link_repeater(self.start_point)
        self.link_loader(self.repeater)
        self.link_forwards(("input", "minibatch_data"), self.loader)
        self.link_evaluator(self.forwards[-1])
        self.link_decision(self.evaluator)
        self.link_snapshotter(self.decision)
        parallel_units = []
        if root.imagenet.add_plotters:
            parallel_units.extend(link(self.snapshotter) for link in (
                self.link_error_plotter, self.link_err_y_plotter))
            parallel_units.append(self.link_weights_plotter("weights", self.snapshotter))
        else:
            parallel_units.append(self.snapshotter)
        last_gd = self.link_gds(*parallel_units)
        self.link_lr_adjuster(last_gd)
        self.link_loop(self.lr_adjuster)
        self.link_end_point(self.lr_adjuster)


def kwargs_from_config():
    c = root.imagenet
    return dict(loader_name=c.loader_name, loader_config=c.loader, decision_config=c.decision,
                snapshotter_config=c.snapshotter, weights_plotter_config=c.weights_plotter,
                lr_adjuster_config=c.lr_adjuster, layers=c.layers,
                image_saver_config=c.image_saver, loss_function=c.loss_function)


def build(launcher=None, **overrides):
    from ..core.workflow import DummyLauncher
    kw = kwargs_from_config()
    kw.update(overrides)
    return ImagenetWorkflow(launcher or DummyLauncher(), **kw)


def run(load, main):
    load(ImagenetWorkflow, **kwargs_from_config())
    main()
