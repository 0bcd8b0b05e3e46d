"""ctypes binding of oracle/_ref/libsmref.so -- the reference's own hot path (see
oracle/refharness/harness.cpp).  TEST INFRASTRUCTURE: import only from tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
"""
import ctypes as C
import os
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "_ref", "libsmref.so")
SOIL_DIR = os.path.join(HERE, "_ref", "soil")
GOLDEN_SOIL_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden", "soil")

SOIL_DTYPE = np.dtype([
    ("name", "S32"),
    ("transports", "<i4"), ("erodes", "<i4"), ("cascades", "<i4"), ("abrades", "<i4"),
    ("density", "<f4"), ("porosity", "<f4"), ("solubility", "<f4"), ("equrate", "<f4"),
    ("friction", "<f4"), ("erosionrate", "<f4"), ("maxdiff", "<f4"), ("settling", "<f4"),
    ("suspension", "<f4"), ("abrasion", "<f4"), ("color", "<f4", (4,)),
])
LAYER_DTYPE = np.dtype([
    ("type", "<i4"), ("min", "<f4"), ("bias", "<f4"), ("scale", "<f4"), ("octaves", "<f4"),
    ("lacunarity", "<f4"), ("gain", "<f4"), ("frequency", "<f4"),
])


class Stats(C.Structure):
    _fields_ = [("steps", C.c_int64), ("sweeps", C.c_int64), ("exit_oob", C.c_int64),
                ("exit_evap", C.c_int64), ("exit_stall", C.c_int64), ("seconds", C.c_double)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def available():
    return os.path.exists(LIB_PATH)


def soil_path(name):
    """Preset .soil file: the run-time copy under oracle/_ref/soil (made by `make -C oracle ref`),
    else the copy stored with the test fixtures (tests/golden/soil)."""
    if not name.endswith(".soil"):
        name += ".soil"
    for d in (SOIL_DIR, GOLDEN_SOIL_DIR):
        p = os.path.join(d, name)
        if os.path.exists(p):
            return p
    raise FileNotFoundError(name)


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


class Ref:
    """One process-wide reference context (the reference keeps its state in globals)."""

    def __init__(self):
        self.lib = C.CDLL(LIB_PATH)
        L = self.lib
        L.smref_init.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        L.smref_nsections.restype = C.c_int64
        L.smref_pool_free.restype = C.c_int64
        L.smref_height_i.restype = C.c_double
        L.smref_height_i.argtypes = [C.c_int, C.c_int]
        L.smref_height_f.restype = C.c_double
        L.smref_height_f.argtypes = [C.c_float, C.c_float]
        L.smref_surface.argtypes = [C.c_int, C.c_int]
        L.smref_normal.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_float)]
        L.smref_add.argtypes = [C.c_int, C.c_int, C.c_double, C.c_int]
        L.smref_remove.restype = C.c_double
        L.smref_remove.argtypes = [C.c_int, C.c_int, C.c_double]
        L.smref_cascade.argtypes = [C.c_float, C.c_float, C.c_int]
        L.smref_srand.argtypes = [C.c_uint]
        self.dimx = self.dimy = self.scale = 0

    # ---- setup -------------------------------------------------------------------------------
    def init(self, soil, seed=42, dimx=0, dimy=0, poolsize=0, quiet=True):
        path = soil if os.path.exists(soil) else soil_path(soil)
        rc = self.lib.smref_init(path.encode(), seed, dimx, dimy, poolsize, int(quiet))
        if rc != 0:
            raise RuntimeError("smref_init failed for %s" % path)
        w = (C.c_int * 5)()
        self.lib.smref_world(w)
        self.dimx, self.dimy, self.scale, self.nwater, self.nwind = list(w)
        return self

    @property
    def cells(self):
        return self.dimx * self.dimy

    def soils(self):
        out = np.zeros(self.lib.smref_nsoils(), SOIL_DTYPE)
        self.lib.smref_get_soils(out.ctypes.data_as(C.c_void_p))
        return out

    def layers(self):
        out = np.zeros(self.lib.smref_nlayers(), LAYER_DTYPE)
        self.lib.smref_get_layers(out.ctypes.data_as(C.c_void_p))
        return out

    # ---- columns -----------------------------------------------------------------------------
    def nsections(self):
        return self.lib.smref_nsections()

    def columns(self):
        n = self.nsections()
        off = np.zeros(self.cells + 1, np.int64)
        typ = np.zeros(n, np.int32)
        size = np.zeros(n, np.float64)
        floor = np.zeros(n, np.float64)
        sat = np.zeros(n, np.float64)
        self.lib.smref_get_columns(_p(off, C.c_int64), _p(typ, C.c_int32), _p(size, C.c_double),
                                   _p(floor, C.c_double), _p(sat, C.c_double))
        return {"offsets": off, "type": typ, "size": size, "floor": floor, "saturation": sat}

    def set_columns(self, offsets, typ, size, saturation=None):
        offsets = np.ascontiguousarray(offsets, np.int64)
        typ = np.ascontiguousarray(typ, np.int32)
        size = np.ascontiguousarray(size, np.float64)
        sat = None if saturation is None else np.ascontiguousarray(saturation, np.float64)
        self.lib.smref_set_columns(_p(offsets, C.c_int64), _p(typ, C.c_int32), _p(size, C.c_double),
                                   _p(sat, C.c_double))

    def heights(self):
        out = np.zeros(self.cells, np.float64)
        self.lib.smref_heights(_p(out, C.c_double))
        return out.reshape(self.dimx, self.dimy)

    def surfaces(self):
        out = np.zeros(self.cells, np.int32)
        self.lib.smref_surfaces(_p(out, C.c_int32))
        return out.reshape(self.dimx, self.dimy)

    def frequency(self):
        a = [np.zeros(self.cells, np.float32) for _ in range(3)]
        self.lib.smref_get_frequency(*[_p(x, C.c_float) for x in a])
        return {"water_frequency": a[0], "water_track": a[1], "wind_frequency": a[2]}

    def set_frequency(self, water_frequency=None, water_track=None, wind_frequency=None):
        arrs = [None if x is None else np.ascontiguousarray(x, np.float32)
                for x in (water_frequency, water_track, wind_frequency)]
        self.lib.smref_set_frequency(*[_p(x, C.c_float) for x in arrs])

    def frequency_update(self):
        self.lib.smref_frequency_update()

    def mesh(self, slice_):
        out = np.zeros((self.cells, 11), np.float32)
        self.lib.smref_mesh(int(slice_), _p(out, C.c_float))
        return out

    def export(self):
        h = np.zeros(self.cells, np.float32); c = np.zeros((self.cells, 4), np.float32)
        self.lib.smref_export(_p(h, C.c_float), _p(c, C.c_float))
        return h, c

    # ---- KAT entry points ----------------------------------------------------------------------
    def height(self, x, y):
        if isinstance(x, (int, np.integer)) and isinstance(y, (int, np.integer)):
            return self.lib.smref_height_i(int(x), int(y))
        return self.lib.smref_height_f(float(x), float(y))

    def surface(self, x, y):
        return self.lib.smref_surface(int(x), int(y))

    def normal(self, x, y):
        out = (C.c_float * 3)()
        self.lib.smref_normal(int(x), int(y), out)
        return np.array(list(out), np.float32)

    def add(self, x, y, size, typ):
        self.lib.smref_add(int(x), int(y), float(size), int(typ))

    def remove(self, x, y, h):
        return self.lib.smref_remove(int(x), int(y), float(h))

    def cascade(self, x, y, transferloop=0):
        self.lib.smref_cascade(float(x), float(y), int(transferloop))

    # ---- spawn lists ------------------------------------------------------------------------------
    def spawn_list(self, n, seed=None):
        """n spawn positions drawn exactly as the particle ctor draws them (water.h:13)."""
        if seed is not None:
            self.lib.smref_srand(int(seed))
        xy = np.zeros((n, 2), np.float32)
        self.lib.smref_spawn_list(n, _p(xy, C.c_float))
        return xy

    # ---- lockstep ---------------------------------------------------------------------------------
    def water_begin(self, xy):
        xy = np.ascontiguousarray(xy, np.float32)
        self._nw = len(xy)
        self.lib.smref_water_begin(len(xy), _p(xy, C.c_float))

    def water_sweep(self, st=None):
        st = st or Stats()
        return self.lib.smref_water_sweep(C.byref(st)), st

    def water_state(self):
        n = self._nw
        pos = np.zeros((n, 2), np.float32); speed = np.zeros((n, 2), np.float32)
        vol = np.zeros(n, np.float64); sed = np.zeros(n, np.float64)
        cont = np.zeros(n, np.int32); alive = np.zeros(n, np.int32)
        self.lib.smref_water_state(_p(pos, C.c_float), _p(speed, C.c_float), _p(vol, C.c_double),
                                   _p(sed, C.c_double), _p(cont, C.c_int32), _p(alive, C.c_int32))
        return {"pos": pos, "speed": speed, "volume": vol, "sediment": sed, "contains": cont, "alive": alive}

    def water_run(self, xy, max_sweeps=0):
        xy = np.ascontiguousarray(xy, np.float32)
        self._nw = len(xy)
        st = Stats()
        self.lib.smref_water_run(len(xy), _p(xy, C.c_float), int(max_sweeps), C.byref(st))
        return st

    def set_volume_factor(self, v):
        self.lib.smref_set_volume_factor.argtypes = [C.c_double]
        self.lib.smref_set_volume_factor(float(v))

    def water_flood(self):
        """flood() for every finished particle of the last water batch, ascending index; returns the count."""
        self.lib.smref_water_flood.restype = C.c_int64
        return int(self.lib.smref_water_flood())

    def seep(self):
        """WaterParticle::seep(map, vertexpool): the per-frame full-grid pass."""
        self.lib.smref_seep()

    def wind_begin(self, xy):
        xy = np.ascontiguousarray(xy, np.float32)
        self._nd = len(xy)
        self.lib.smref_wind_begin(len(xy), _p(xy, C.c_float))

    def wind_sweep(self, st=None):
        st = st or Stats()
        return self.lib.smref_wind_sweep(C.byref(st)), st

    def wind_state(self):
        n = self._nd
        pos = np.zeros((n, 2), np.float32); speed = np.zeros((n, 3), np.float32)
        h = np.zeros(n, np.float64); sed = np.zeros(n, np.float64)
        cont = np.zeros(n, np.int32); alive = np.zeros(n, np.int32)
        self.lib.smref_wind_state(_p(pos, C.c_float), _p(speed, C.c_float), _p(h, C.c_double),
                                  _p(sed, C.c_double), _p(cont, C.c_int32), _p(alive, C.c_int32))
        return {"pos": pos, "speed": speed, "height": h, "sediment": sed, "contains": cont, "alive": alive}

    def wind_run(self, xy, max_sweeps=0):
        xy = np.ascontiguousarray(xy, np.float32)
        self._nd = len(xy)
        st = Stats()
        self.lib.smref_wind_run(len(xy), _p(xy, C.c_float), int(max_sweeps), C.byref(st))
        return st

    # ---- sequential reference loops -----------------------------------------------------------------
    def water_seq(self, n, xy=None, flood=False, seep=False):
        st = Stats()
        if xy is not None:
            xy = np.ascontiguousarray(xy, np.float32)
            n = len(xy)
        self.lib.smref_water_seq(int(n), _p(xy, C.c_float), int(flood) | (int(seep) << 1), C.byref(st))
        return st

    def wind_seq(self, n, xy=None):
        st = Stats()
        if xy is not None:
            xy = np.ascontiguousarray(xy, np.float32)
            n = len(xy)
        self.lib.smref_wind_seq(int(n), _p(xy, C.c_float), 0, C.byref(st))
        return st


_singleton = None


def get():
    global _singleton
    if _singleton is None:
        _singleton = Ref()
    return _singleton
