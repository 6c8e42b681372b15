"""``veles`` namespace of the H100-native framework.

The real code lives in :mod:`veles.znicz_b200`. For users of the reference,
reference-style import paths keep working through lazy aliases installed by
:mod:`veles.znicz_b200.compat` (``from veles.znicz.all2all import All2AllTanh``,
``from veles.config import root``, ``from veles.memory import Array`` …), which
also lets whole-workflow pickles carry stable class paths.
"""
from .znicz_b200 import compat as _compat

_compat.install()
