"""Avatar: a stand-in that mirrors selected attributes of a "real" unit so the
real unit (a loader) can run ahead of the main contour
(``veles.avatar.Avatar``; /root/reference/standard_workflow.py:386-404).

On H100 the overlap itself is done with a copy stream + double buffered device
minibatches inside the loader; the Avatar keeps the graph-level API: it clones the
exported attributes on every run so downstream units read a stable snapshot.
"""
from __future__ import annotations

import copy

from .memory import Array
from .mutable import Bool
from .units import Unit


class Avatar(Unit):
    hide_from_registry = True

    def __init__(self, workflow, **kwargs):
        super().__init__(workflow, **kwargs)
        self.reals = {}

    def clone(self):
        for real, attrs in self.reals.items():
            for name in attrs:
                value = getattr(real, name, None)
                if isinstance(value, Array):
                    mine = self.__dict__.get(name)
                    if not isinstance(mine, Array):
                        mine = Array(shallow_pickle=value.shallow_pickle)
                        self.__dict__[name] = mine
                    if value:
                        value.map_read()
                        if not mine or mine.shape != value.shape:
                            mine.reset(value.mem.copy())
                        else:
                            mine.map_invalidate()
                            mine.mem[...] = value.mem
                elif isinstance(value, Bool):
                    mine = self.__dict__.get(name)
                    if not isinstance(mine, Bool):
                        mine = Bool(bool(value))
                        self.__dict__[name] = mine
                    else:
                        mine <<= bool(value)
                else:
                    self.__dict__[name] = copy.copy(value)

    def initialize(self, **kwargs):
        self.clone()

    def run(self):
        self.clone()
