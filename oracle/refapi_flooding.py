"""ctypes binding of oracle/_ref/libsmref_flooding.so: the reference context of refapi.Ref plus the sweep-flood
driver (oracle/refharness/sweep_flood.cpp).  TEST INFRASTRUCTURE: import only from tests/ and scripts/."""
import ctypes as C
import os
import numpy as np

from oracle import refapi

LIB_PATH = os.path.join(refapi.HERE, "_ref", "libsmref_flooding.so")


def available():
    return os.path.exists(LIB_PATH)


class Ref(refapi.Ref):
    """refapi.Ref on its own copy of the reference (a separate library with its own globals)."""

    def __init__(self):
        saved = refapi.LIB_PATH
        refapi.LIB_PATH = LIB_PATH
        try:
            super().__init__()
        finally:
            refapi.LIB_PATH = saved
        self.lib.smref_water_sweep_flood.restype = C.c_int64

    def water_sweep_flood(self, xy, max_sweeps=0):
        """A lockstep water batch whose particles flood() at the end of the sweep they stop in, ascending index.
        Returns (Stats, number of floods that passed flood()'s guard)."""
        xy = np.ascontiguousarray(xy, np.float32)
        self._nw = len(xy)
        st = refapi.Stats()
        nfl = self.lib.smref_water_sweep_flood(len(xy), xy.ctypes.data_as(C.POINTER(C.c_float)), int(max_sweeps),
                                               C.byref(st))
        return st, int(nfl)


_singleton = None


def get():
    global _singleton
    if _singleton is None:
        _singleton = Ref()
    return _singleton
