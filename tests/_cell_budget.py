"""ctypes bindings of the per-cell budget test tools (tests/cell_budget/): the oracle port and the host emulation with
the per-cell maps of the mass budget.  TEST INFRASTRUCTURE.  Each library is compiled on first use into a temporary
directory (the tree stays as it is), named by a hash of its sources."""
import ctypes as C
import os
import numpy as np
import _hostsim
from _hydro_budget import _build
from oracle import portapi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "soilmachine_b200", "csrc")
TERMS = ("eroded", "deposited", "cascade_net")


def _maps(flat, dimx, dimy):
    m = flat.reshape(dimx, dimy, 3)
    return {k: np.ascontiguousarray(m[:, :, i]) for i, k in enumerate(TERMS)}


class CellPort(portapi.Port):
    """portapi.Port on a library whose water_run / wind_run also keep the per-cell maps
    (tests/cell_budget/port_cells.cpp)"""

    def __init__(self):
        src = os.path.join(HERE, "cell_budget", "port_cells.cpp")
        lib = _build("port_cells", src, [os.path.join(ROOT, "oracle", f) for f in ("sm_oracle.cpp", "sm_oracle.h")])
        self.lib = C.CDLL(lib)
        L = self.lib
        L.smo_nsections.restype = C.c_int64
        L.smo_height_i.restype = C.c_double
        L.smo_height_i.argtypes = [C.c_int, C.c_int]
        L.smo_height_f.restype = C.c_double
        L.smo_height_f.argtypes = [C.c_float, C.c_float]

    def water_run(self, xy, max_sweeps=0):
        self._nw = len(xy)
        return self._run(self.lib.smc_water_run, xy, max_sweeps)

    def wind_run(self, xy, max_sweeps=0):
        self._nd = len(xy)
        return self._run(self.lib.smc_wind_run, xy, max_sweeps)

    def cell_budget(self):
        """(maps of the last batch: dict of three (dimx, dimy) float64 arrays, measurements per cell (dimx, dimy))"""
        out = np.zeros(self.cells * 3)
        nops = np.zeros(self.cells, np.int64)
        self.lib.smc_cell_budget(out.ctypes.data_as(C.POINTER(C.c_double)), nops.ctypes.data_as(C.POINTER(C.c_int64)))
        return _maps(out, self.dimx, self.dimy), nops.reshape(self.dimx, self.dimy)


class CellHostSim(_hostsim.HostSim):
    """tests/hostsim on a library that also holds the warp-cooperative step with the per-cell maps (host_cells.cpp);
    its water_run / wind_run always run that step.  split: stage as the exact-footprint schedule does."""

    def __init__(self, split=0):
        src = os.path.join(HERE, "cell_budget", "host_cells.cpp")
        deps = [_hostsim.SRC, _hostsim.CORE, _hostsim.NOISE, _hostsim.HYDRO, _hostsim.COOP, _hostsim.HCOOP,
                os.path.join(CSRC, "sm_foot.cuh")]
        self.lib = C.CDLL(_build("host_cells", src, deps))
        self.split = int(split)
        L = self.lib
        L.hs_nsections.restype = C.c_int64
        L.hs_height_f.restype = C.c_double
        L.hs_height_f.argtypes = [C.c_float, C.c_float]

    def water_begin(self, xy):
        super().water_begin(xy)
        self.lib.hc_reset_cells()

    def water_sweep(self, st):
        return self.lib.hc_water_sweep(C.byref(st), self.split)

    def wind_begin(self, xy):
        super().wind_begin(xy)
        self.lib.hc_reset_cells()

    def wind_sweep(self, st):
        return self.lib.hc_wind_sweep(C.byref(st), self.split)

    def wind_run(self, xy):
        self.wind_begin(xy)
        st = _hostsim.Stats()
        while self.wind_sweep(st) > 0:
            pass
        return st

    def cell_budget(self):
        out = np.zeros(self.dimx * self.dimy * 3)
        self.lib.hc_cell_budget(out.ctypes.data_as(C.POINTER(C.c_double)))
        return _maps(out, self.dimx, self.dimy)
