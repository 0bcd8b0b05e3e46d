"""ctypes bindings of the hydrology per-cell budget test tools (tests/hydro_cells/): the oracle port and the host
emulation with the per-cell maps of the pooling hydrology's mass budget.  TEST INFRASTRUCTURE.  Each library is
compiled on first use into a temporary directory (the tree stays as it is), named by a hash of its sources."""
import ctypes as C
import os
import numpy as np
import _hostsim
from _cell_budget import CellPort
from _hydro_budget import _build
from oracle import portapi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "soilmachine_b200", "csrc")
TERMS = ("eroded", "deposited", "cascade_net", "water_net")
# the sm_hydro_budget slots (tests/_hydro_budget.TERMS order) each map refines, with their signs
SLOTS = {"eroded": ((6, 1),), "deposited": ((0, 1), (7, 1)), "cascade_net": ((1, 1), (8, 1)),
         "water_net": ((2, 1), (3, -1), (4, -1), (5, 1))}


def _maps(flat, dimx, dimy):
    m = flat.reshape(dimx, dimy, 4)
    return {k: np.ascontiguousarray(m[:, :, i]) for i, k in enumerate(TERMS)}


def slot_sum(b, term):
    """the group of hydrology-budget slots `term` refines"""
    return sum(s * b[i] for i, s in SLOTS[term])


class HydroCellPort(CellPort):
    """portapi.Port on a library whose water_flood / seep (smh_*) also keep the hydrology's per-cell maps
    (tests/hydro_cells/port_hydro_cells.cpp).  The library holds port_cells.cpp as well, so water_run / wind_run and
    cell_budget() are CellPort's: the batches with their maps."""

    def __init__(self):
        src = os.path.join(HERE, "hydro_cells", "port_hydro_cells.cpp")
        deps = [os.path.join(HERE, "cell_budget", "port_cells.cpp")] + \
            [os.path.join(ROOT, "oracle", f) for f in ("sm_oracle.cpp", "sm_oracle.h")]
        self.lib = C.CDLL(_build("port_hydro_cells", src, deps))
        L = self.lib
        L.smo_nsections.restype = C.c_int64
        L.smo_height_i.restype = C.c_double
        L.smo_height_i.argtypes = [C.c_int, C.c_int]
        L.smo_height_f.restype = C.c_double
        L.smo_height_f.argtypes = [C.c_float, C.c_float]

    def water_flood(self):
        hy = portapi.Hydro()
        self.lib.smh_water_flood(C.byref(hy))
        return hy

    def seep(self):
        hy = portapi.Hydro()
        self.lib.smh_seep(C.byref(hy))
        return hy

    def hydro_cell_budget(self):
        """(maps of the last water_flood / seep: dict of four (dimx, dimy) float64 arrays, measurements per cell)"""
        out = np.zeros(self.cells * 4)
        nops = np.zeros(self.cells, np.int64)
        self.lib.smh_cell_budget(out.ctypes.data_as(C.POINTER(C.c_double)), nops.ctypes.data_as(C.POINTER(C.c_int64)))
        return _maps(out, self.dimx, self.dimy), nops.reshape(self.dimx, self.dimy)


class HydroCellHostSim(_hostsim.HostSim):
    """tests/hostsim on a library that also holds the warp hydrology with the budget and the per-cell maps
    (host_hydro_cells.cpp); its water_flood / seep always run the warp executor"""

    def __init__(self):
        src = os.path.join(HERE, "hydro_cells", "host_hydro_cells.cpp")
        deps = [_hostsim.SRC, _hostsim.CORE, _hostsim.NOISE, _hostsim.HYDRO, _hostsim.COOP, _hostsim.HCOOP,
                os.path.join(CSRC, "sm_foot.cuh")]
        self.lib = C.CDLL(_build("host_hydro_cells", src, deps))
        L = self.lib
        L.hs_nsections.restype = C.c_int64
        L.hs_height_f.restype = C.c_double
        L.hs_height_f.argtypes = [C.c_float, C.c_float]
        L.hs_remove.restype = C.c_double
        L.hs_remove.argtypes = [C.c_int, C.c_int, C.c_double]
        L.hs_add.argtypes = [C.c_int, C.c_int, C.c_double, C.c_int]
        L.hs_cascade.argtypes = [C.c_float, C.c_float, C.c_int]

    def water_flood(self):
        hc = _hostsim.HydroCount()
        self.lib.hhc_water_flood(C.byref(hc))
        return hc

    def seep(self, mode=1):
        hc = _hostsim.HydroCount()
        self.lib.hhc_seep(int(mode), C.byref(hc))
        return hc

    def hydro_cell_budget(self):
        out = np.zeros(self.dimx * self.dimy * 4)
        self.lib.hhc_cell_budget(out.ctypes.data_as(C.POINTER(C.c_double)))
        return _maps(out, self.dimx, self.dimy)

    def hydro_budget(self):
        out = np.zeros(11)
        self.lib.hhc_hydro_budget(out.ctypes.data_as(C.POINTER(C.c_double)))
        return out
