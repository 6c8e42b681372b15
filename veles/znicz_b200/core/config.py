"""Global auto-vivifying configuration tree (``root``).

Capability parity with the absent Veles core's ``veles.config.root`` as it is
consumed by the reference (e.g. /root/reference/samples/Wine/wine_config.py:43-58,
/root/reference/samples/CIFAR10/cifar_caffe_config.py:52-145): sample configs
are plain python files doing ``root.<ns>.update({...})``; engine keys live under
``root.common.engine`` and directories under ``root.common.dirs``.

Design notes (H100-first): the tree also carries the H100 engine switches
(``root.common.engine.backend`` in {"numpy", "cuda"}, ``precision_type`` in
{"float", "double", "bf16"}, ``graphs`` for CUDA-graph capture of the
minibatch step).
"""
from __future__ import annotations

import os
import pprint
import tempfile


class Config(object):
    """A node of the configuration tree. Unknown attributes become sub-nodes."""

    def __init__(self, path=""):
        object.__setattr__(self, "__path__", path)

    # -- attribute protocol -------------------------------------------------
    def __getattr__(self, name):
        if name.startswith("__") and name.endswith("__"):
            raise AttributeError(name)
        node = Config("%s.%s" % (self.__path__, name) if self.__path__ else name)
        object.__setattr__(self, name, node)
        return node

    def __setattr__(self, name, value):
        if isinstance(value, dict) and not isinstance(value, Config):
            node = Config("%s.%s" % (self.__path__, name))
            node.update(value)
            value = node
        object.__setattr__(self, name, value)

    def __getitem__(self, name):
        return getattr(self, name)

    def __setitem__(self, name, value):
        setattr(self, name, value)

    def __contains__(self, name):
        return name in self.__dict__ and not (
            isinstance(self.__dict__[name], Config) and not self.__dict__[name])

    def __bool__(self):
        return any(k != "__path__" for k in self.__dict__)

    __nonzero__ = __bool__

    def __iter__(self):
        return iter(self.__content__.items())

    # mapping protocol, so ``dict(node)`` / ``**node`` work on config sub-trees
    def keys(self):
        return self.__content__.keys()

    def values(self):
        return self.__content__.values()

    def items(self):
        return self.__content__.items()

    # -- helpers ------------------------------------------------------------
    def update(self, value=None, **kwargs):
        if value is None:
            value = {}
        if isinstance(value, Config):
            value = value.__content__
        if not isinstance(value, dict):
            raise ValueError("Config.update() takes a dict (got %s)" % type(value))
        value = dict(value)
        value.update(kwargs)
        for k, v in value.items():
            if isinstance(v, dict):
                getattr(self, k).update(v) if isinstance(
                    self.__dict__.get(k), Config) else setattr(self, k, v)
            else:
                setattr(self, k, v)
        return self

    def get(self, name, default=None):
        v = self.__dict__.get(name, default)
        if isinstance(v, Config) and not v:
            return default
        return v

    def protect(self, *names):  # kept for API parity; values are plain attrs
        return self

    @property
    def __content__(self):
        return {k: v for k, v in self.__dict__.items() if k != "__path__"}

    def to_dict(self):
        out = {}
        for k, v in self.__content__.items():
            out[k] = v.to_dict() if isinstance(v, Config) else v
        return out

    def print_(self, indent=1, width=80, file=None):
        pprint.pprint(self.to_dict(), indent=indent, width=width, stream=file)

    def __repr__(self):
        return "<Config %s: %s>" % (self.__path__, sorted(self.__content__))

    # pickling: a Config is its dict
    def __getstate__(self):
        return {"path": self.__path__, "content": self.to_dict()}

    def __setstate__(self, state):
        object.__setattr__(self, "__path__", state["path"])
        self.update(state["content"])


root = Config("root")


def get(value, default=None):
    """``veles.config.get``: unwrap a possibly-empty Config node."""
    if isinstance(value, Config):
        return default if not value else value
    return value


def validate_kwargs(caller, **kwargs):
    for k, v in kwargs.items():
        if isinstance(v, Config) and not v:
            raise ValueError("%s: kwarg %s is an empty Config node" % (caller, k))


def _defaults():
    base = os.environ.get("ZNICZ_B200_HOME",
                          os.path.join(tempfile.gettempdir(), "znicz_b200"))
    root.common.update({
        "engine": {
            # "numpy" (CPU oracle) or "cuda" (sm_90a). "auto" picks cuda when present.
            "backend": "auto",
            # host/master dtype: "float" | "double"; device compute dtype is
            # selected with compute_type: "fp32" | "bf16" | "fp8"
            "precision_type": "float",
            "compute_type": "fp32",
            "precision_level": 0,
            "graphs": True,
            "source_dirs": [],
        },
        "dirs": {
            "datasets": os.path.join(base, "datasets"),
            "cache": os.path.join(base, "cache"),
            "snapshots": os.path.join(base, "snapshots"),
            "user": base,
            "veles": base,
        },
        "disable": {"plotting": True, "snapshotting": False, "publishing": True},
        "trace": {"run": False, "nvtx": os.environ.get("ZNICZ_NVTX", "0") == "1"},
    })


_defaults()
