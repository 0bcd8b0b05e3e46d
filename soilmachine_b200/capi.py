"""ctypes binding of lib/libsoilmachine_b200.so (the C ABI in include/soilmachine_b200.h).

This is plumbing for tests and bench.py; the product is the shared library.  There is no CPU
fallback: loading fails loudly when the library has not been built, and sm_create fails when no
CUDA device is present.
"""
import ctypes as C
import os
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libsoilmachine_b200.so")

SM_OK, SM_ERR_INVALID, SM_ERR_CUDA, SM_ERR_POOL, SM_ERR_REACH, SM_ERR_NOGPU = range(6)
SM_MAX_SOILS = 64

SOIL_DTYPE = np.dtype([
    ("transports", "<i4"), ("erodes", "<i4"), ("cascades", "<i4"), ("abrades", "<i4"),
    ("density", "<f4"), ("porosity", "<f4"), ("solubility", "<f4"), ("equrate", "<f4"),
    ("friction", "<f4"), ("erosionrate", "<f4"), ("maxdiff", "<f4"), ("settling", "<f4"),
    ("suspension", "<f4"), ("abrasion", "<f4"),
])
LAYER_DTYPE = np.dtype([
    ("type", "<i4"), ("min", "<f4"), ("bias", "<f4"), ("scale", "<f4"), ("octaves", "<f4"),
    ("lacunarity", "<f4"), ("gain", "<f4"), ("frequency", "<f4"),
])

# every symbol include/soilmachine_b200.h declares (tests check the library exports them all)
SYMBOLS = [
    "sm_create", "sm_destroy", "sm_last_error", "sm_sync", "sm_set_soils", "sm_initialize",
    "sm_upload_columns", "sm_section_count", "sm_download_columns", "sm_download_height",
    "sm_download_surface", "sm_height_sum", "sm_checksum", "sm_get_frequency", "sm_set_frequency",
    "sm_frequency_update", "sm_cell_add", "sm_cell_remove", "sm_cell_cascade", "sm_cell_query",
    "sm_height_bilinear", "sm_cell_column", "sm_cell_seep", "sm_cell_water_cascade", "sm_set_volume_factor", "sm_water_run", "sm_wind_run", "sm_water_run_device", "sm_wind_run_device",
    "sm_last_stats", "sm_water_begin", "sm_water_sweeps", "sm_water_state", "sm_wind_begin",
    "sm_wind_sweeps", "sm_wind_state", "sm_launch_count", "sm_device_alloc", "sm_device_free",
    "sm_device_upload", "sm_timer_start", "sm_timer_stop", "sm_set_soil_colors", "sm_mesh_update",
    "sm_mesh_device_ptr", "sm_export_height", "sm_export_color", "sm_create_sharded", "sm_shard_range",
    "sm_peer_export", "sm_peer_attach", "sm_hydro_issuer", "sm_parse_soil_file", "sm_water_flood", "sm_seep", "sm_last_budget", "sm_budget_particles", "sm_last_cell_budget", "sm_last_hydro_budget", "sm_last_hydro_cell_budget", "sm_lbm_create", "sm_lbm_set_boundary", "sm_lbm_init",
    "sm_lbm_step", "sm_lbm_get", "sm_lbm_advect", "sm_wind_use_lbm",
    "sm_create_group", "sm_group_size", "sm_group_rank", "sm_group_layout",
    "sm_snapshot_bytes", "sm_snapshot_save", "sm_snapshot_restore",
    "sm_apply_layer", "sm_relax", "sm_composition", "sm_voxelize",
    "sm_water_run_flooding",
]


class Config(C.Structure):
    _fields_ = [("dimx", C.c_int32), ("dimy", C.c_int32), ("scale", C.c_int32), ("device", C.c_int32),
                ("pool_capacity", C.c_int64), ("max_particles", C.c_int32), ("flags", C.c_int32)]


class Stats(C.Structure):
    _fields_ = [("steps", C.c_int64), ("sweeps", C.c_int64), ("exit_oob", C.c_int64),
                ("exit_evap", C.c_int64), ("exit_stall", C.c_int64), ("pool_drops", C.c_int64),
                ("alive", C.c_int64), ("device_ms", C.c_double)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class HydroStats(C.Structure):
    _fields_ = [("floods", C.c_int64), ("nested", C.c_int64), ("nested_steps", C.c_int64),
                ("transfers", C.c_int64), ("cells", C.c_int64), ("device_ms", C.c_double),
                ("classify_ms", C.c_double)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class Budget(C.Structure):
    _fields_ = [("eroded", C.c_double), ("deposited", C.c_double), ("cascade_net", C.c_double),
                ("discarded", C.c_double), ("clamped", C.c_double), ("wind_negative", C.c_double),
                ("particles", C.c_int64)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class HydroBudget(C.Structure):
    _fields_ = [(k, C.c_double) for k in (
        "flood_sediment", "flood_cascade_net", "flood_water", "seeped", "to_particles", "transfer_net",
        "nested_eroded", "nested_deposited", "nested_cascade_net", "nested_discarded", "nested_clamped")]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class LayerStats(C.Structure):
    _fields_ = [("cells", C.c_int64), ("pushed", C.c_int64), ("free_slots", C.c_int64), ("emptied", C.c_int64),
                ("device_ms", C.c_double)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class RelaxStats(C.Structure):
    _fields_ = [("passes", C.c_int64), ("stable", C.c_int64), ("visits", C.c_int64), ("transfers", C.c_int64),
                ("pool_drops", C.c_int64), ("device_ms", C.c_double)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class ViewStats(C.Structure):
    _fields_ = [("cells", C.c_int64), ("sections", C.c_int64), ("bytes_out", C.c_int64), ("device_ms", C.c_double)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


SM_COMP_BELOW_SURFACE = 1
SM_COMP_PORE_WATER = 2
SM_VOXEL_NONE = 255
SM_VOXEL_MAX_NZ = 65536


CELL_TERMS = ("eroded", "deposited", "cascade_net")     # sm_last_cell_budget
HYDRO_CELL_TERMS = ("eroded", "deposited", "cascade_net", "water_net")     # sm_last_hydro_cell_budget


class SoilMachineError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("soilmachine_b200 error %d: %s" % (code, msg))
        self.code = code


_lib = None


def load():
    """Load the shared library; raises if it was not built (no fallback)."""
    global _lib
    if _lib is None:
        path = os.environ.get("SM_LIB_PATH", LIB_PATH)   # debugging builds (e.g. -DSM_PROFILE) only
        if not os.path.exists(path):
            raise FileNotFoundError(
                "%s not built: run ./build.sh (or python -c 'import __graft_entry__ as g; g.build()')" % LIB_PATH)
        _lib = C.CDLL(path)
        _lib.sm_last_error.restype = C.c_char_p
        _lib.sm_last_error.argtypes = [C.c_void_p]
        _lib.sm_destroy.argtypes = [C.c_void_p]
        _lib.sm_destroy.restype = None
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


def parse_soil_file(path):
    """loadsoil() of the reference (source/io.h:7-230) through the library's own parser."""
    lib = load()
    soils = np.zeros(SM_MAX_SOILS, SOIL_DTYPE); names = np.zeros((SM_MAX_SOILS, 32), np.uint8)
    colors = np.zeros((SM_MAX_SOILS, 4), np.float32); layers = np.zeros(16, LAYER_DTYPE)
    ns, nl = C.c_int32(), C.c_int32()
    world = (C.c_int32 * 5)()
    rc = lib.sm_parse_soil_file(str(path).encode(), soils.ctypes.data_as(C.c_void_p), names.ctypes.data_as(C.c_char_p),
                                _p(colors, C.c_float), SM_MAX_SOILS, C.byref(ns), layers.ctypes.data_as(C.c_void_p), 16,
                                C.byref(nl), world)
    if rc != SM_OK:
        raise SoilMachineError(rc, lib.sm_last_error(None).decode())
    n = ns.value
    return {"soils": soils[:n].copy(), "colors": colors[:n].copy(), "layers": layers[:nl.value].copy(),
            "soil_names": [bytes(names[i]).split(b"\0")[0].decode() for i in range(n)],
            "world": dict(zip(("sizex", "sizey", "scale", "nwater", "nwind"), list(world)))}


def soils_from(table):
    """numpy structured table (any dtype carrying the SurfParam field names) -> sm_soil array."""
    out = np.zeros(len(table), SOIL_DTYPE)
    for k in SOIL_DTYPE.names:
        out[k] = table[k]
    return out


class PeerBlob(C.Structure):
    _fields_ = [("ptr", C.c_uint64 * 24), ("ipc", (C.c_ubyte * 64) * 24), ("pool_cap", C.c_uint64),
                ("rank", C.c_int32), ("device", C.c_int32)]


class Context:
    """One sm_context: one GPU, one rank of a sharded map, or (gpus > 1) a group over a map sharded in this process."""

    def __init__(self, dimx, dimy, scale=80, device=0, pool_capacity=0, max_particles=0,
                 nranks=1, rank=0, share=1, budget=False, cell_budget=False, hydro_cell_budget=False,
                 gpus=1, devices=None):
        """cell_budget=True keeps the per-cell budget maps of the batches as well (SM_FLAG_BUDGET | SM_FLAG_CELL_BUDGET),
        hydro_cell_budget=True those of the hydrology calls (SM_FLAG_BUDGET | SM_FLAG_HYDRO_CELL_BUDGET).
        gpus=N (or devices=[ordinal of rank 0, ...]) creates the context with sm_create_group: the map is cut into N
        x-strips, one rank per entry of `devices` (default: device, device + 1, ...; equal entries share a GPU), and
        every method below acts on the whole map exactly as on one context."""
        self.lib = load()
        self.dimx, self.dimy, self.scale = int(dimx), int(dimy), int(scale)
        flags = 3 if cell_budget else (1 if budget else 0)     # SM_FLAG_BUDGET | SM_FLAG_CELL_BUDGET
        if hydro_cell_budget:
            flags |= 1 | 4                                     # SM_FLAG_BUDGET | SM_FLAG_HYDRO_CELL_BUDGET
        cfg = Config(self.dimx, self.dimy, self.scale, int(device), int(pool_capacity), int(max_particles), flags)
        h = C.c_void_p()
        if devices is not None:
            gpus = len(devices)
        if gpus > 1 or devices is not None:
            assert nranks == 1, "a group creates its own ranks"
            devs = (C.c_int32 * gpus)(*(devices if devices is not None else range(int(device), int(device) + gpus)))
            rc = self.lib.sm_create_group(C.byref(cfg), int(gpus), devs, C.byref(h))
        elif nranks == 1:
            rc = self.lib.sm_create(C.byref(cfg), C.byref(h))
        else:
            rc = self.lib.sm_create_sharded(C.byref(cfg), int(nranks), int(rank), int(share), C.byref(h))
        if rc != SM_OK:
            raise SoilMachineError(rc, self.lib.sm_last_error(None).decode())
        self.h = h
        self.nranks, self.rank = int(nranks), int(rank)
        x0, x1 = C.c_int32(), C.c_int32()
        self.lib.sm_shard_range(self.h, C.byref(x0), C.byref(x1))
        self.x0, self.x1 = x0.value, x1.value
        self.map_cells = self.dimx * self.dimy                 # whole map (frequency arrays)
        self.cells = (self.x1 - self.x0) * self.dimy           # this rank's strip (columns, heights)
        self._n = {"water": 0, "wind": 0}

    def group_size(self):
        n = C.c_int32()
        self._ck(self.lib.sm_group_size(self.h, C.byref(n)))
        return n.value

    def group_rank(self, rank):
        """the raw handle of rank `rank` of a group (owned by the group), for tests and tools"""
        h = C.c_void_p()
        self._ck(self.lib.sm_group_rank(self.h, int(rank), C.byref(h)))
        return h

    def peer_export(self):
        b = PeerBlob()
        self._ck(self.lib.sm_peer_export(self.h, C.byref(b)))
        return b

    def peer_attach(self, blobs, use_ipc):
        arr = (PeerBlob * len(blobs))(*blobs)
        self._ck(self.lib.sm_peer_attach(self.h, arr, len(blobs), int(use_ipc)))

    def hydro_issuer(self, on=True):
        """sharded map: make this rank the one that issues water_flood / seep for the whole map (or stop it)"""
        self._ck(self.lib.sm_hydro_issuer(self.h, int(bool(on))))

    def close(self):
        if getattr(self, "h", None):
            self.lib.sm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc == SM_ERR_POOL and getattr(self, "pool_warn", True):
            # as upstream (layermap.h:92-95: print and drop the section, keep running): a warning, not an error;
            # the call's stats count the drops.  Calls that cannot proceed (a pool too small for the terrain)
            # turn the warning off around themselves and raise.
            import warnings
            warnings.warn("soilmachine_b200: " + self.lib.sm_last_error(self.h).decode(), RuntimeWarning)
            return
        if rc != SM_OK:
            raise SoilMachineError(rc, self.lib.sm_last_error(self.h).decode())

    def _ck_strict(self, rc):
        if rc != SM_OK:
            raise SoilMachineError(rc, self.lib.sm_last_error(self.h).decode())

    # ---- tables / terrain ---------------------------------------------------------------------------
    def set_soils(self, table):
        s = soils_from(table)
        self._ck(self.lib.sm_set_soils(self.h, s.ctypes.data_as(C.c_void_p), len(s)))

    def initialize(self, seed, layers):
        lay = np.zeros(len(layers), LAYER_DTYPE)
        for k in LAYER_DTYPE.names:
            lay[k] = layers[k]
        self._ck_strict(self.lib.sm_initialize(self.h, int(seed), lay.ctypes.data_as(C.c_void_p), len(lay)))

    def upload_columns(self, offsets, typ, size, saturation=None):
        offsets = np.ascontiguousarray(offsets, np.int64)
        typ = np.ascontiguousarray(typ, np.int32)
        size = np.ascontiguousarray(size, np.float64)
        sat = None if saturation is None else np.ascontiguousarray(saturation, np.float64)
        assert len(offsets) == self.cells + 1
        self._ck_strict(self.lib.sm_upload_columns(self.h, _p(offsets, C.c_int64), _p(typ, C.c_int32),
                                                   _p(size, C.c_double), _p(sat, C.c_double)))

    def section_count(self):
        n = C.c_int64()
        self._ck(self.lib.sm_section_count(self.h, C.byref(n)))
        return n.value

    def download_columns(self):
        n = self.section_count()
        off = np.zeros(self.cells + 1, np.int64)
        typ = np.zeros(n, np.int32)
        size = np.zeros(n); floor = np.zeros(n); sat = np.zeros(n)
        self._ck(self.lib.sm_download_columns(self.h, C.c_int64(n), _p(off, C.c_int64), _p(typ, C.c_int32),
                                              _p(size, C.c_double), _p(floor, C.c_double), _p(sat, C.c_double)))
        return {"offsets": off, "type": typ, "size": size, "floor": floor, "saturation": sat}

    def heights(self):
        out = np.zeros(self.cells)
        self._ck(self.lib.sm_download_height(self.h, _p(out, C.c_double)))
        return out.reshape(self.x1 - self.x0, self.dimy)

    def surfaces(self):
        out = np.zeros(self.cells, np.int32)
        self._ck(self.lib.sm_download_surface(self.h, _p(out, C.c_int32)))
        return out.reshape(self.x1 - self.x0, self.dimy)

    def height_sum(self):
        s = C.c_double()
        self._ck(self.lib.sm_height_sum(self.h, C.byref(s)))
        return s.value

    def checksum(self):
        """position-sensitive checksum of all sections of this context's columns (see checksum.py)"""
        v = C.c_uint64()
        self._ck(self.lib.sm_checksum(self.h, C.byref(v)))
        return int(v.value)

    def frequency(self):
        a = [np.zeros(self.map_cells, np.float32) for _ in range(3)]
        self._ck(self.lib.sm_get_frequency(self.h, *[_p(x, C.c_float) for x in a]))
        return {"water_frequency": a[0], "water_track": a[1], "wind_frequency": a[2]}

    def set_frequency(self, water_frequency=None, water_track=None, wind_frequency=None):
        arrs = [None if x is None else np.ascontiguousarray(x, np.float32)
                for x in (water_frequency, water_track, wind_frequency)]
        self._ck(self.lib.sm_set_frequency(self.h, *[_p(x, C.c_float) for x in arrs]))

    def frequency_update(self):
        self._ck(self.lib.sm_frequency_update(self.h))

    # ---- snapshots (soilmachine_b200/snapshot.py has the format) ----------------------------------------------------
    def snapshot_bytes(self):
        n = C.c_int64()
        self._ck_strict(self.lib.sm_snapshot_bytes(self.h, C.byref(n)))
        return n.value

    def snapshot(self):
        """the snapshot of this context's columns and frequency arrays (its strip on a rank of a sharded map, the
        whole map otherwise) as a np.uint8 array"""
        out = np.empty(self.snapshot_bytes(), np.uint8)
        self._ck_strict(self.lib.sm_snapshot_save(self.h, out.ctypes.data_as(C.c_void_p), C.c_int64(out.size), 0))
        return out

    def snapshot_device(self):
        """the snapshot in device memory from sm_device_alloc: (dptr, nbytes); free it with device_free(dptr)"""
        n = self.snapshot_bytes()
        d = C.c_void_p()
        self._ck_strict(self.lib.sm_device_alloc(self.h, C.c_int64(n), C.byref(d)))
        rc = self.lib.sm_snapshot_save(self.h, d, C.c_int64(n), 1)
        if rc != SM_OK:
            self.lib.sm_device_free(self.h, d)
            self._ck_strict(rc)
        return d, n

    def restore(self, buf):
        """restore a snapshot: host bytes / a np.uint8 array, or (dptr, nbytes) of snapshot_device()"""
        if isinstance(buf, tuple):
            d, n = buf
            self._ck_strict(self.lib.sm_snapshot_restore(self.h, C.c_void_p(d.value if isinstance(d, C.c_void_p) else d),
                                                         C.c_int64(n), 1))
            return
        a = np.frombuffer(memoryview(buf), np.uint8)
        self._ck_strict(self.lib.sm_snapshot_restore(self.h, a.ctypes.data_as(C.c_void_p), C.c_int64(a.size), 0))

    # ---- layer rasters ---------------------------------------------------------------------------------------------
    def apply_layer(self, delta, type, leftover=False, check=False):
        """sm_apply_layer: deposit (delta > 0) or strip (delta < 0) soil `type` on every cell in one call.  delta is a
        float64 array of shape (x1 - x0, dimy) - the whole map, or this rank's strip of a sharded map - or a device
        pointer from device_alloc holding that many doubles.  leftover=True (host raster) returns the leftovers as an
        array of that shape; with a device raster, leftover may be a device pointer to write them to.  check=True runs
        the all-or-nothing check alone.  Returns (LayerStats, leftovers or None); a refusal raises with the map
        unchanged (SM_ERR_POOL included)."""
        st = LayerStats()
        if isinstance(delta, np.ndarray):
            d = np.ascontiguousarray(delta, np.float64)
            if d.shape != (self.x1 - self.x0, self.dimy):
                raise SoilMachineError(SM_ERR_INVALID, "apply_layer: the raster has shape %s, the map (%d, %d)"
                                       % (d.shape, self.x1 - self.x0, self.dimy))
            left = np.zeros_like(d) if leftover else None
            self._ck_strict(self.lib.sm_apply_layer(self.h, _p(d, C.c_double), int(type), _p(left, C.c_double), 0,
                                                    int(bool(check)), C.byref(st)))
            return st, left
        if leftover is True:
            raise SoilMachineError(SM_ERR_INVALID, "apply_layer: a device raster writes leftovers to a device pointer")
        d = C.c_void_p(delta.value if isinstance(delta, C.c_void_p) else delta)
        left = None if leftover is False or leftover is None else \
            C.c_void_p(leftover.value if isinstance(leftover, C.c_void_p) else leftover)
        self._ck_strict(self.lib.sm_apply_layer(self.h, d, int(type), left, 1, int(bool(check)), C.byref(st)))
        return st, left

    # ---- slope relaxation -------------------------------------------------------------------------------------------
    def relax(self, max_passes, transferloop=0):
        """sm_relax: up to max_passes passes of Particle::cascade(vec2(x, y), map, vp, transferloop) over every cell in
        the phase order of the header; stops after the first pass that changes nothing.  Returns RelaxStats.  A refusal
        (transferloop outside 0..3, max_passes < 1, a rank of a sharded map) raises with the map unchanged; sections the
        pool could not serve warn, as the batches do, and are counted in pool_drops."""
        st = RelaxStats()
        self._ck(self.lib.sm_relax(self.h, int(max_passes), int(transferloop), C.byref(st)))
        return st

    # ---- strata views ------------------------------------------------------------------------------------------------
    def composition(self, types, lo, hi, below_surface=False, pore_water=False, out=None):
        """sm_composition: per cell, how much of each soil of `types` lies inside the height window [lo, hi] (measured
        down from the surface with below_surface=True), or how much pore water it holds there (pore_water=True).
        Returns a float64 array (len(types), x1 - x0, dimy) - the whole map, or this rank's strip of a sharded map.
        out: a device pointer (device_alloc) of len(types) * (x1 - x0) * dimy doubles to write instead; then returns
        None.  The call's ViewStats are kept in self.view_stats.  A refusal raises with nothing written."""
        t = np.ascontiguousarray(np.atleast_1d(types), np.int32)
        flags = (SM_COMP_BELOW_SURFACE if below_surface else 0) | (SM_COMP_PORE_WATER if pore_water else 0)
        st = ViewStats()
        res = None
        if out is None:
            res = np.empty((len(t), self.x1 - self.x0, self.dimy))
            ptr, dev = res.ctypes.data_as(C.c_void_p), 0
        else:
            ptr, dev = C.c_void_p(out.value if isinstance(out, C.c_void_p) else out), 1
        self._ck_strict(self.lib.sm_composition(self.h, _p(t, C.c_int32), len(t), C.c_double(lo), C.c_double(hi),
                                                flags, ptr, dev, C.byref(st)))
        self.view_stats = st
        return res

    def voxelize(self, x0, x1, y0, y1, z0, dz, nz, out=None):
        """sm_voxelize: the soil type at the heights z0 + k*dz (k < nz) of every cell of the window [x0, x1) x [y0, y1)
        (global coordinates; inside this rank's strip on a sharded map), the first section met top -> bottom that
        contains the height, SM_VOXEL_NONE where none does.  Returns uint8 (nz, x1 - x0, y1 - y0); out: a device pointer
        of that many bytes to write instead (returns None).  ViewStats in self.view_stats."""
        st = ViewStats()
        res = None
        if out is None:
            res = np.empty((max(int(nz), 0), max(x1 - x0, 0), max(y1 - y0, 0)), np.uint8)
            ptr, dev = res.ctypes.data_as(C.c_void_p), 0
        else:
            ptr, dev = C.c_void_p(out.value if isinstance(out, C.c_void_p) else out), 1
        self._ck_strict(self.lib.sm_voxelize(self.h, int(x0), int(x1), int(y0), int(y1), C.c_double(z0), C.c_double(dz),
                                             int(nz), ptr, dev, C.byref(st)))
        self.view_stats = st
        return res

    def set_soil_colors(self, rgba):
        rgba = np.ascontiguousarray(rgba, np.float32).reshape(-1, 4)
        self._ck(self.lib.sm_set_soil_colors(self.h, _p(rgba, C.c_float), len(rgba)))

    def mesh_update(self, slice_, download=True):
        """Layermap::update(Vertexpool&): (cells, 11) float32 = position3, normal3, color4, index."""
        out = np.zeros((self.cells, 11), np.float32) if download else None
        self._ck(self.lib.sm_mesh_update(self.h, int(slice_), _p(out, C.c_float)))
        return out

    def export_height(self):
        out = np.zeros(self.cells, np.float32)
        self._ck(self.lib.sm_export_height(self.h, _p(out, C.c_float)))
        return out

    def export_color(self):
        out = np.zeros((self.cells, 4), np.float32)
        self._ck(self.lib.sm_export_color(self.h, _p(out, C.c_float)))
        return out

    def sync(self):
        self._ck(self.lib.sm_sync(self.h))

    # ---- single-cell -----------------------------------------------------------------------------------
    def cell_add(self, x, y, size, typ):
        self._ck(self.lib.sm_cell_add(self.h, int(x), int(y), C.c_double(size), int(typ)))

    def cell_remove(self, x, y, h):
        out = C.c_double()
        self._ck(self.lib.sm_cell_remove(self.h, int(x), int(y), C.c_double(h), C.byref(out)))
        return out.value

    def cell_cascade(self, x, y, transferloop=0):
        self._ck(self.lib.sm_cell_cascade(self.h, C.c_float(x), C.c_float(y), int(transferloop)))

    def cell_query(self, x, y):
        h = C.c_double(); s = C.c_int32(); n = (C.c_float * 3)()
        self._ck(self.lib.sm_cell_query(self.h, int(x), int(y), C.byref(h), C.byref(s), n))
        return h.value, s.value, np.array(list(n), np.float32)

    def height_bilinear(self, x, y):
        h = C.c_double()
        self._ck(self.lib.sm_height_bilinear(self.h, C.c_float(x), C.c_float(y), C.byref(h)))
        return h.value

    # ---- hot path ------------------------------------------------------------------------------------------
    def _run(self, fn, xy, max_sweeps):
        xy = np.ascontiguousarray(xy, np.float32)
        st = Stats()
        self._ck(fn(self.h, len(xy), _p(xy, C.c_float), int(max_sweeps), C.byref(st)))
        return st

    def water_run(self, xy, max_sweeps=0):
        self._n["water"] = len(xy)
        return self._run(self.lib.sm_water_run, xy, max_sweeps)

    def water_run_flooding(self, xy, max_sweeps=0):
        """sm_water_run_flooding: a water batch whose particles flood at the end of the sweep they stop in, so later
        sweeps of the batch meet the ponds.  Returns (Stats, HydroStats)."""
        self._n["water"] = len(xy)
        xy = np.ascontiguousarray(xy, np.float32)
        st, hs = Stats(), HydroStats()
        self._ck(self.lib.sm_water_run_flooding(self.h, len(xy), _p(xy, C.c_float), int(max_sweeps), C.byref(st),
                                                C.byref(hs)))
        return st, hs

    def wind_run(self, xy, max_sweeps=0):
        self._n["wind"] = len(xy)
        return self._run(self.lib.sm_wind_run, xy, max_sweeps)

    def set_volume_factor(self, v):
        self.lib.sm_set_volume_factor.argtypes = [C.c_void_p, C.c_double]
        self._ck(self.lib.sm_set_volume_factor(self.h, float(v)))

    def cell_column(self, x, y, capacity=64):
        n = C.c_int32()
        typ = np.zeros(capacity, np.int32); size = np.zeros(capacity); fl = np.zeros(capacity); sat = np.zeros(capacity)
        self._ck(self.lib.sm_cell_column(self.h, int(x), int(y), int(capacity), C.byref(n), _p(typ, C.c_int32),
                                         _p(size, C.c_double), _p(fl, C.c_double), _p(sat, C.c_double)))
        m = min(n.value, capacity)
        return {"n": n.value, "type": typ[:m], "size": size[:m], "floor": fl[:m], "saturation": sat[:m]}

    def cell_seep(self, x, y):
        self._ck(self.lib.sm_cell_seep(self.h, int(x), int(y)))

    def cell_water_cascade(self, x, y, spill=0):
        self._ck(self.lib.sm_cell_water_cascade(self.h, int(x), int(y), int(spill)))

    def budget_particles(self, n):
        """raw mass-budget accumulators [n, 6] of the last batch (context created with budget=True)"""
        per = np.zeros((int(n), 6))
        self._ck(self.lib.sm_budget_particles(self.h, int(n), _p(per, C.c_double)))
        return per

    def last_budget(self):
        b = Budget()
        self._ck(self.lib.sm_last_budget(self.h, C.byref(b)))
        return b

    def last_cell_budget(self):
        """per-cell budget maps of the last batch (context created with cell_budget=True): a dict of three float64
        arrays "eroded", "deposited", "cascade_net" of shape (x1 - x0, dimy)"""
        out = {k: np.zeros(self.cells) for k in CELL_TERMS}
        self._ck_strict(self.lib.sm_last_cell_budget(self.h, *[_p(out[k], C.c_double) for k in CELL_TERMS]))
        return {k: v.reshape(self.x1 - self.x0, self.dimy) for k, v in out.items()}

    # ---- wind field (D3Q19 lattice Boltzmann) ----
    def lbm_create(self, nx, ny, nz):
        self._lbm = (int(nx), int(ny), int(nz))
        self._ck(self.lib.sm_lbm_create(self.h, int(nx), int(ny), int(nz)))

    def lbm_set_boundary(self, boundary=None):
        b = None if boundary is None else np.ascontiguousarray(boundary, np.float32)
        self._ck(self.lib.sm_lbm_set_boundary(self.h, _p(b, C.c_float)))

    def lbm_init(self):
        self._ck(self.lib.sm_lbm_init(self.h))

    def lbm_step(self, n=1):
        ms = C.c_double()
        self._ck(self.lib.sm_lbm_step(self.h, int(n), C.byref(ms)))
        return ms.value

    def lbm_get(self):
        nx, ny, nz = self._lbm
        n = nx * ny * nz
        f = np.zeros((n, 19), np.float32); rho = np.zeros(n, np.float32); v = np.zeros((n, 4), np.float32)
        self._ck(self.lib.sm_lbm_get(self.h, _p(f, C.c_float), _p(rho, C.c_float), _p(v, C.c_float)))
        return {"f": f, "rho": rho, "v": v}

    def wind_use_lbm(self, on=True):
        self._ck(self.lib.sm_wind_use_lbm(self.h, 1 if on else 0))

    def lbm_advect(self, pos4):
        pos = np.ascontiguousarray(pos4, np.float32).copy()
        self._ck(self.lib.sm_lbm_advect(self.h, len(pos), _p(pos, C.c_float)))
        return pos

    def water_flood(self):
        """flood() of every finished particle of the last water batch (water.h:123-145), ascending index."""
        st = HydroStats()
        self._ck(self.lib.sm_water_flood(self.h, C.byref(st)))
        return st

    def seep(self):
        """The per-frame full-grid pass WaterParticle::seep(map, vertexpool) (water.h:335-343)."""
        st = HydroStats()
        self._ck(self.lib.sm_seep(self.h, C.byref(st)))
        return st

    def last_hydro_budget(self):
        """mass budget of the last water_flood or seep call (context created with budget=True): a dict of the
        eleven sm_hydro_budget terms (include/soilmachine_b200.h)"""
        b = HydroBudget()
        self._ck(self.lib.sm_last_hydro_budget(self.h, C.byref(b)))
        return b.asdict()

    def last_hydro_cell_budget(self):
        """per-cell maps of the hydrology's budget for the last water_flood or seep call (context created with
        hydro_cell_budget=True): a dict of four float64 arrays "eroded", "deposited", "cascade_net", "water_net" of
        shape (dimx, dimy)"""
        out = {k: np.zeros(self.cells) for k in HYDRO_CELL_TERMS}
        self._ck_strict(self.lib.sm_last_hydro_cell_budget(self.h, *[_p(out[k], C.c_double) for k in HYDRO_CELL_TERMS]))
        return {k: v.reshape(self.dimx, self.dimy) for k, v in out.items()}

    def water_begin(self, xy):
        xy = np.ascontiguousarray(xy, np.float32)
        self._n["water"] = len(xy)
        self._ck(self.lib.sm_water_begin(self.h, len(xy), _p(xy, C.c_float)))

    def wind_begin(self, xy):
        xy = np.ascontiguousarray(xy, np.float32)
        self._n["wind"] = len(xy)
        self._ck(self.lib.sm_wind_begin(self.h, len(xy), _p(xy, C.c_float)))

    def water_sweeps(self, k=1):
        st = Stats()
        self._ck(self.lib.sm_water_sweeps(self.h, int(k), C.byref(st)))
        return st

    def wind_sweeps(self, k=1):
        st = Stats()
        self._ck(self.lib.sm_wind_sweeps(self.h, int(k), C.byref(st)))
        return st

    def water_state(self):
        n = self._n["water"]
        pos = np.zeros((n, 2), np.float32); speed = np.zeros((n, 2), np.float32)
        vol = np.zeros(n); sed = np.zeros(n); cont = np.zeros(n, np.int32); alive = np.zeros(n, np.int32)
        self._ck(self.lib.sm_water_state(self.h, _p(pos, C.c_float), _p(speed, C.c_float), _p(vol, C.c_double),
                                         _p(sed, C.c_double), _p(cont, C.c_int32), _p(alive, C.c_int32)))
        return {"pos": pos, "speed": speed, "volume": vol, "sediment": sed, "contains": cont, "alive": alive}

    def wind_state(self):
        n = self._n["wind"]
        pos = np.zeros((n, 2), np.float32); speed = np.zeros((n, 3), np.float32)
        h = np.zeros(n); sed = np.zeros(n); cont = np.zeros(n, np.int32); alive = np.zeros(n, np.int32)
        self._ck(self.lib.sm_wind_state(self.h, _p(pos, C.c_float), _p(speed, C.c_float), _p(h, C.c_double),
                                        _p(sed, C.c_double), _p(cont, C.c_int32), _p(alive, C.c_int32)))
        return {"pos": pos, "speed": speed, "height": h, "sediment": sed, "contains": cont, "alive": alive}

    # device-resident spawn lists (bench "value": inputs already in HBM)
    def device_spawn(self, xy):
        xy = np.ascontiguousarray(xy, np.float32)
        d = C.c_void_p()
        self._ck(self.lib.sm_device_alloc(self.h, C.c_int64(xy.nbytes), C.byref(d)))
        self._ck(self.lib.sm_device_upload(self.h, d, xy.ctypes.data_as(C.c_void_p), C.c_int64(xy.nbytes)))
        return d

    def device_free(self, d):
        self._ck(self.lib.sm_device_free(self.h, d))

    def water_run_device(self, d_xy, n, max_sweeps=0):
        self._n["water"] = n
        self._ck(self.lib.sm_water_run_device(self.h, int(n), d_xy, int(max_sweeps)))

    def wind_run_device(self, d_xy, n, max_sweeps=0):
        self._n["wind"] = n
        self._ck(self.lib.sm_wind_run_device(self.h, int(n), d_xy, int(max_sweeps)))

    def last_stats(self):
        st = Stats()
        self._ck(self.lib.sm_last_stats(self.h, C.byref(st)))
        return st

    def timer_start(self):
        self._ck(self.lib.sm_timer_start(self.h))

    def timer_stop(self):
        ms = C.c_double()
        self._ck(self.lib.sm_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def launch_count(self):
        n = C.c_int64()
        self._ck(self.lib.sm_launch_count(self.h, C.byref(n)))
        return n.value
