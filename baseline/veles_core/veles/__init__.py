"""Minimal stand-in for the Veles core platform (package ``veles``), which the reference
(Samsung/veles.znicz, a *plugin* of that platform) needs but which is neither in
/root/reference nor installable offline. Written from the plugin's usage of the core
(SURVEY.md §1.3, §8): unit graph runtime, config tree, Array with map/unmap coherence,
NVRTC program build, driver-API launches, cuBLAS GEMM, full-batch loaders.

It exists ONLY so that ``bench.py --impl reference`` can run the UNMODIFIED reference
units (``oracle/_ref/veles/znicz``) through their stock ``cuda_run`` path on an H100.
Nothing of veles.znicz_b200 (the product) is imported here.
"""
import importlib.abc
import importlib.util
import os
import sys
import types

__root__ = os.path.dirname(os.path.abspath(__file__))
__version__ = "0.0.shim"
__plugins__ = set()

_ref = os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(__root__))), "oracle", "_ref",
                    "veles")
if os.path.isdir(_ref):
    __path__.append(_ref)          # veles.znicz = the vendored, unmodified reference


class _StubModule(types.ModuleType):
    """Core modules the training path never executes (plotters, publishing, web status,
    interactive shell, downloader...): importable, every attribute is a placeholder class
    derived from Unit so that ``class X(veles.something.Base)`` and isinstance checks work."""

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        from veles.units import Unit
        if name[:1] == "I" and name[1:2].isupper():          # interface marker
            from zope.interface import Interface
            cls = type(name, (Interface,), {"__module__": self.__name__})
        else:
            cls = type(name, (Unit,), {"__module__": self.__name__,
                                       "hide_from_registry": True, "_is_stub": True})
        setattr(self, name, cls)
        return cls


class _StubFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, fullname, path=None, target=None):
        if not fullname.startswith("veles.") or fullname.startswith("veles.znicz"):
            return None
        return importlib.util.spec_from_loader(fullname, self, is_package=True)

    def create_module(self, spec):
        m = _StubModule(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        pass


sys.meta_path.append(_StubFinder())      # last: real shim modules win
