"""Host-side mirror of the GL-free part of the reference's main() (SoilMachine.cpp:34-48,82-83,
283-320) on top of the C ABI: load a preset, build the terrain on the GPU, run frames.

A frame = one water batch run to completion, optionally the pooling hydrology (the batch's floods and
the full-grid seep pass, SoilMachine.cpp:296,300-301), one wind batch run to completion, the frequency
update.  Spawn positions are drawn with
the C library's rand() in the order the particle constructors draw them (water.h:13, wind.h:15:
GCC evaluates the two arguments right to left, so y takes the first draw).
"""
import ctypes as C
import ctypes.util
import os
import numpy as np
from . import capi, presets

_libc = None
_draws = 0       # rand() draws since the last srand (Simulation.save stores it, Simulation.load replays it)


def _c():
    global _libc
    if _libc is None:
        _libc = C.CDLL(ctypes.util.find_library("c") or "libc.so.6")
        _libc.rand.restype = C.c_int
        _libc.srand.argtypes = [C.c_uint]
    return _libc


def srand(seed):
    global _draws
    _c().srand(int(seed) & 0xFFFFFFFF)
    _draws = 0


def draws():
    """rand() draws made by spawn_list since the last srand"""
    return _draws


def spawn_list(n, dimx, dimy):
    """n (x, y) spawn positions = n constructor calls' worth of rand() draws."""
    global _draws
    lc = _c()
    _draws += 2 * n
    out = np.empty((n, 2), np.float32)
    for i in range(n):
        y = lc.rand() % dimy
        x = lc.rand() % dimx
        out[i, 0] = x
        out[i, 1] = y
    return out


class Simulation:
    """soil preset + GPU context + frame loop."""

    def __init__(self, soil, seed=42, dimx=0, dimy=0, device=0, max_particles=0, pool_capacity=0, gpus=1,
                 devices=None, budget=False, cell_budget=False):
        """gpus / devices: the map sharded over several GPUs of this process (capi.Context); the frame loop is the
        same.  budget / cell_budget: keep the mass budgets (capi.Context)."""
        # a preset name (JSON tables dumped from the reference loader) or a path to a `.soil` file
        self.preset = capi.parse_soil_file(soil) if str(soil).endswith(".soil") and os.path.exists(str(soil)) \
            else presets.load(soil)
        w = self.preset["world"]
        self.dimx = int(dimx or w["sizex"])
        self.dimy = int(dimy or w["sizey"])
        self.scale = int(w["scale"])
        self.seed = int(seed)
        srand(self.seed)                                   # SoilMachine.cpp:41
        self.soil = str(soil)
        self.ctx = capi.Context(self.dimx, self.dimy, self.scale, device=device,
                                pool_capacity=pool_capacity, max_particles=max_particles, gpus=gpus, devices=devices,
                                budget=budget, cell_budget=cell_budget)
        self.ctx.set_soils(self.preset["soils"])
        self.ctx.set_soil_colors(self.preset["colors"])
        self.ctx.initialize(self.seed, self.preset["layers"])   # Layermap(SEED, dim), SoilMachine.cpp:83

    def frame(self, nwater, nwind, water_xy=None, wind_xy=None, hydrology=False, water_chunk=0, floods="batch"):
        """SoilMachine.cpp:287-320.  hydrology=False: the hot path only (flood disabled, no seep pass);
        True: the water batch is followed by its floods and by the seep pass (self.last_hydrology holds the
        counter sets).  water_chunk > 0 splits the frame's water particles into lockstep batches of that
        size, each followed by its floods: upstream floods every particle right after its own loop, so later
        particles of a frame meet the ponds earlier ones left; smaller chunks follow that interleaving more
        closely (chunk 1 = upstream's order) at the price of fewer particles in flight (DESIGN.md K6).
        floods="sweep" (with hydrology=True): each water batch floods its particles at the end of the sweep they stop
        in (capi.Context.water_run_flooding), so the batch's later sweeps meet its own ponds; "batch" (the default)
        floods them once the batch has ended.
        Returns (water_stats of the last batch, wind_stats)."""
        if floods not in ("batch", "sweep"):
            raise ValueError("floods must be 'batch' or 'sweep'")
        if floods == "sweep" and not hydrology:
            raise ValueError("floods='sweep' needs hydrology=True")
        ws = ds = None
        self.last_hydrology = None
        if nwater:
            xy = water_xy if water_xy is not None else spawn_list(nwater, self.dimx, self.dimy)
            chunk = int(water_chunk) if (hydrology and water_chunk and water_chunk > 0) else len(xy)
            flooded = []
            for i in range(0, len(xy), chunk):
                if floods == "sweep":
                    ws, fs = self.ctx.water_run_flooding(xy[i:i + chunk])
                    flooded.append(fs)
                    continue
                ws = self.ctx.water_run(xy[i:i + chunk])
                if hydrology:
                    flooded.append(self.ctx.water_flood())
            if hydrology:
                self.last_hydrology = (flooded, self.ctx.seep())
        if nwind:
            xy = wind_xy if wind_xy is not None else spawn_list(nwind, self.dimx, self.dimy)
            ds = self.ctx.wind_run(xy)
        if nwater:
            self.ctx.frequency_update()
        return ws, ds

    def apply_layer(self, delta, soil, leftover=False):
        """Deposit (delta > 0) or strip (delta < 0) one soil on every cell (capi.Context.apply_layer, sm_apply_layer):
        delta is a (dimx, dimy) float64 raster, soil a name of the preset's soil table or an index.  Returns the stats
        and, with leftover=True, the height each strip could not take."""
        typ = self.preset["soil_names"].index(soil) if isinstance(soil, str) else int(soil)
        return self.ctx.apply_layer(delta, typ, leftover=leftover)

    def _soil(self, soil):
        return self.preset["soil_names"].index(soil) if isinstance(soil, str) else int(soil)

    def composition(self, soils, lo, hi, below_surface=False, pore_water=False):
        """Per cell, how much of each soil (names of the preset's table or indices) lies inside the height window [lo,
        hi], or how much pore water it holds there (capi.Context.composition, sm_composition): (len(soils), dimx, dimy)
        float64."""
        if isinstance(soils, (str, int, np.integer)):
            soils = [soils]
        return self.ctx.composition([self._soil(s) for s in soils], lo, hi, below_surface, pore_water)

    def voxelize(self, x0, x1, y0, y1, z0, dz, nz):
        """The soil index at the heights z0 + k*dz of every cell of [x0, x1) x [y0, y1) (capi.Context.voxelize,
        sm_voxelize): (nz, x1 - x0, y1 - y0) uint8, 255 where no section holds the height."""
        return self.ctx.voxelize(x0, x1, y0, y1, z0, dz, nz)

    def drainage(self, ground=False):
        """How the map drains (capi.Context.drainage, sm_drainage): a dict of (dimx, dimy) rasters - spill (the spill
        height), dir (the receiver's neighbour index, -1 on the border), area (cells draining through each cell) and
        basin (the border cell each cell drains to, as x*dimy + y).  ground=True reads the ground under standing water.
        The call's stats are kept in self.ctx.drain_stats."""
        return self.ctx.drainage(ground)

    def relax(self, max_passes, transferloop=0):
        """Relax the slopes of the whole map (capi.Context.relax, sm_relax): Particle::cascade at every cell, pass after
        pass in a fixed phase order, until a pass changes nothing or max_passes passes have run.  Returns the stats."""
        return self.ctx.relax(max_passes, transferloop)

    def save(self, path):
        """Write the simulation to `path`: the snapshot of the map (columns and frequency arrays), the soil preset, the
        seed and the rand() draws made since srand.  A Simulation.load of the file continues the run with the same
        spawn lists.  Not saved: the volume factor, the wind lattice, budgets (snapshot.py lists the rest)."""
        with open(path, "wb") as f:
            np.savez(f, snapshot=self.ctx.snapshot(), soil=np.array(self.soil), seed=np.int64(self.seed),
                     draws=np.int64(_draws))

    @classmethod
    def load(cls, path, device=0, gpus=1, devices=None, **kw):
        """A Simulation from a file of save(), on any number of GPUs (gpus / devices as in __init__, other keyword
        arguments too): the map is restored from the snapshot, rand() is re-seeded and the saved number of draws is
        discarded, so later frames draw the spawn lists the uninterrupted run would have drawn."""
        global _draws
        with np.load(path) as z:
            buf, soil, seed, n = z["snapshot"], str(z["soil"]), int(z["seed"]), int(z["draws"])
        from . import snapshot
        h = snapshot.header(buf)
        sim = cls(soil, seed=seed, dimx=h["dimx"], dimy=h["dimy"], device=device, gpus=gpus, devices=devices, **kw)
        sim.ctx.restore(buf)
        srand(seed)
        lc = _c()
        for _ in range(n):
            lc.rand()
        _draws = n
        return sim

    def close(self):
        self.ctx.close()
