"""ctypes bindings of the hydrology mass-budget test tools (tests/hydro_budget/): the oracle port and the host
emulation with the budget of the pooling hydrology.  TEST INFRASTRUCTURE.  Each library is compiled on first use
into a temporary directory (the tree stays as it is), named by a hash of its sources."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
import numpy as np
import _hostsim
from oracle import portapi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "soilmachine_b200", "csrc")
TERMS = ("flood_sediment", "flood_cascade_net", "flood_water", "seeped", "to_particles", "transfer_net",
         "nested_eroded", "nested_deposited", "nested_cascade_net", "nested_discarded", "nested_clamped")


def _build(name, src, deps):
    h = hashlib.sha256()
    for p in [src] + deps:
        with open(p, "rb") as f:
            h.update(f.read())
    out = os.path.join(tempfile.gettempdir(), "sm_%s_%s_%d.so" % (name, h.hexdigest()[:16], os.getuid()))
    if not os.path.exists(out):
        tmp = out + ".%d.tmp" % os.getpid()
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", src, "-o", tmp])
        os.replace(tmp, out)
    return out


def identity(b):
    """the change of the height sum the eleven terms account for"""
    return b[0] + b[1] + b[2] - b[3] - b[4] + b[5] + b[7] - b[6] + b[8]


class BudgetPort(portapi.Port):
    """portapi.Port on a library that also holds the budget's flood / seep (tests/hydro_budget/port_budget.cpp)"""

    def __init__(self):
        src = os.path.join(HERE, "hydro_budget", "port_budget.cpp")
        lib = _build("port_budget", src, [os.path.join(ROOT, "oracle", f) for f in ("sm_oracle.cpp", "sm_oracle.h")])
        self.lib = C.CDLL(lib)
        L = self.lib
        L.smo_nsections.restype = C.c_int64
        L.smo_height_i.restype = C.c_double
        L.smo_height_i.argtypes = [C.c_int, C.c_int]
        L.smo_height_f.restype = C.c_double
        L.smo_height_f.argtypes = [C.c_float, C.c_float]
        L.smo_surface.argtypes = [C.c_int, C.c_int]
        L.smo_normal.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_float)]
        L.smo_add.argtypes = [C.c_int, C.c_int, C.c_double, C.c_int]
        L.smo_remove.restype = C.c_double
        L.smo_remove.argtypes = [C.c_int, C.c_int, C.c_double]
        L.smo_cascade.argtypes = [C.c_float, C.c_float, C.c_int]

    def water_flood(self):
        hy = portapi.Hydro()
        self.lib.smob_water_flood(C.byref(hy))
        return hy

    def seep(self):
        hy = portapi.Hydro()
        self.lib.smob_seep(C.byref(hy))
        return hy

    def hydro_budget(self):
        """the eleven sums of the last water_flood / seep call, in the order of TERMS"""
        out = np.zeros(11)
        self.lib.smob_hydro_budget(out.ctypes.data_as(C.POINTER(C.c_double)))
        return out


class BudgetHostSim(_hostsim.HostSim):
    """tests/hostsim on a library that also holds the warp hydrology with the budget (host_budget.cpp); its
    water_flood / seep always run the warp executor"""

    def __init__(self):
        src = os.path.join(HERE, "hydro_budget", "host_budget.cpp")
        deps = [_hostsim.SRC, _hostsim.CORE, _hostsim.NOISE, _hostsim.HYDRO, _hostsim.COOP, _hostsim.HCOOP,
                os.path.join(CSRC, "sm_foot.cuh")]
        lib = _build("host_budget", src, deps)
        self.lib = C.CDLL(lib)
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
        self.lib.hsb_water_flood(C.byref(hc))
        return hc

    def seep(self, mode=1):
        hc = _hostsim.HydroCount()
        self.lib.hsb_seep(int(mode), C.byref(hc))
        return hc

    def hydro_budget(self):
        out = np.zeros(11)
        self.lib.hsb_hydro_budget(out.ctypes.data_as(C.POINTER(C.c_double)))
        return out
