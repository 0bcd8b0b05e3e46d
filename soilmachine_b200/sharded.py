"""Sharded maps: one sm_context per rank, x-strips, peer pointers (DESIGN.md section 7).

VirtualShards  - all ranks are contexts of THIS process on one GPU (share = nranks).  Same kernels, same
                 cross-rank barrier and hand-over protocol as the multi-GPU path, exercised on a single
                 device (what the 1-GPU test tier runs).
DistShard      - one rank per process / GPU under torch.distributed: peer blobs are all-gathered and the
                 other GPUs' arrays are opened with CUDA IPC, so halo records, bins and `done` words are
                 read and written over NVLink by the sweep kernel itself.
"""
import ctypes as C
import numpy as np
from . import capi, snapshot as snap


def split_columns(cols, dimx, dimy, x0, x1):
    """global bottom->top CSR (cell order x*dimy+y) -> the CSR of the strip [x0, x1)."""
    off = np.asarray(cols["offsets"])
    lo, hi = off[x0 * dimy], off[x1 * dimy]
    out = {"offsets": (off[x0 * dimy:x1 * dimy + 1] - lo).astype(np.int64)}
    for k in ("type", "size", "saturation"):
        out[k] = None if cols.get(k) is None else np.asarray(cols[k])[lo:hi]
    return out


def merge_columns(parts):
    off = [np.zeros(1, np.int64)]
    base = 0
    for p in parts:
        off.append(p["offsets"][1:] + base)
        base += p["offsets"][-1]
    out = {"offsets": np.concatenate(off)}
    for k in ("type", "size", "floor", "saturation"):
        out[k] = np.concatenate([p[k] for p in parts])
    return out


def merge_frequency(parts, ranges, dimx, dimy):
    """frequency arrays are indexed y*dimx + x; rank q's copy is authoritative for its own columns."""
    out = {}
    for k in parts[0]:
        m = np.zeros((dimy, dimx), np.float32)
        for p, (x0, x1) in zip(parts, ranges):
            m[:, x0:x1] = p[k].reshape(dimy, dimx)[:, x0:x1]
        out[k] = m.reshape(-1)
    return out


def check_restored(buf, checksums):
    """A rank restoring its slice of a whole-map snapshot cannot check the header's checksum alone: the ranks'
    checksums after the restore must add up (mod 2^64) to it."""
    h = snap.header(buf)
    if h["x0"] == 0 and h["x1"] == h["dimx"] and sum(checksums) % (1 << 64) != h["checksum"]:
        raise capi.SoilMachineError(capi.SM_ERR_INVALID, "snapshot: the restored columns do not match the header's "
                                                         "checksum")


def sum_layer_stats(stats):
    tot = capi.LayerStats()
    for f, _ in capi.LayerStats._fields_:
        vals = [getattr(s, f) for s in stats]
        setattr(tot, f, max(vals) if f == "device_ms" else sum(vals))
    return tot


def _layer_check(ctx, delta, type):
    """one rank's check pass: (accepted, stats, refusal)"""
    try:
        return True, ctx.apply_layer(delta, type, check=True)[0], None
    except capi.SoilMachineError as e:
        return False, None, e


def sum_view_stats(stats):
    tot = capi.ViewStats()
    for f, _ in capi.ViewStats._fields_:
        vals = [getattr(s, f) for s in stats]
        setattr(tot, f, max(vals) if f == "device_ms" else sum(vals))
    return tot


def voxel_part(ctx, x0, x1, y0, y1, z0, dz, nz):
    """one rank's part of a voxel window: the window cut at the rank's strip (nz, 0, y1 - y0) when it misses the strip;
    a window that is empty or leaves the map goes to the library whole, which refuses it"""
    xs, xe = max(x0, ctx.x0), min(x1, ctx.x1)
    if xs >= xe and 0 <= x0 < x1 <= ctx.dimx and 0 <= y0 < y1 <= ctx.dimy:
        return np.empty((int(nz), 0, y1 - y0), np.uint8), None
    out = ctx.voxelize(xs, xe, y0, y1, z0, dz, nz) if xs < xe else ctx.voxelize(x0, x1, y0, y1, z0, dz, nz)
    return out, ctx.view_stats


def sum_stats(stats):
    tot = capi.Stats()
    for f, _ in capi.Stats._fields_:
        vals = [getattr(s, f) for s in stats]
        setattr(tot, f, max(vals) if f in ("sweeps", "device_ms", "alive") else sum(vals))
    return tot


class VirtualShards:
    def __init__(self, nranks, dimx, dimy, scale=80, device=0, max_particles=0, pool_capacity=0, budget=False,
                 cell_budget=False):
        self.nranks, self.dimx, self.dimy = nranks, dimx, dimy
        self.ctx = [capi.Context(dimx, dimy, scale, device=device, max_particles=max_particles,
                                 pool_capacity=pool_capacity, nranks=nranks, rank=r, share=nranks, budget=budget,
                                 cell_budget=cell_budget)
                    for r in range(nranks)]
        blobs = [c.peer_export() for c in self.ctx]
        for c in self.ctx:
            c.peer_attach(blobs, use_ipc=False)
        self.ranges = [(c.x0, c.x1) for c in self.ctx]

    def close(self):
        for c in self.ctx:
            c.close()

    def set_soils(self, table):
        for c in self.ctx:
            c.set_soils(table)

    def initialize(self, seed, layers):
        for c in self.ctx:
            c.initialize(seed, layers)

    def upload_columns(self, cols):
        for c in self.ctx:
            p = split_columns(cols, self.dimx, self.dimy, c.x0, c.x1)
            c.upload_columns(p["offsets"], p["type"], p["size"], p["saturation"])

    def download_columns(self):
        return merge_columns([c.download_columns() for c in self.ctx])

    def snapshot(self):
        """the whole-map snapshot: every rank saves its strip, the strips are joined"""
        self.sync()
        return np.frombuffer(snap.join([c.snapshot() for c in self.ctx]), np.uint8)

    def restore(self, buf):
        """every rank restores its slice of a whole-map snapshot (host bytes); the ranks' checksums are then compared
        with the header's"""
        self.sync()
        for c in self.ctx:
            c.restore(buf)
        check_restored(buf, [c.checksum() for c in self.ctx])

    def apply_layer(self, delta, type, leftover=False):
        """sm_apply_layer over the whole map, all or nothing: every rank checks its strip of the (dimx, dimy) raster,
        and only when every rank accepts does every rank apply it.  Returns (summed stats, leftovers or None)."""
        delta = np.ascontiguousarray(delta, np.float64)
        self.sync()
        for c in self.ctx:
            ok, _, err = _layer_check(c, delta[c.x0:c.x1], type)
            if not ok:
                raise err
        out = [c.apply_layer(delta[c.x0:c.x1], type, leftover=leftover) for c in self.ctx]
        self.sync()
        return sum_layer_stats([o[0] for o in out]), (np.concatenate([o[1] for o in out]) if leftover else None)

    def composition(self, types, lo, hi, below_surface=False, pore_water=False):
        """sm_composition over the whole map: every rank computes its strip, the strips are joined along x.  Returns
        (len(types), dimx, dimy) float64; the summed ViewStats are kept in self.view_stats."""
        self.sync()
        parts = [c.composition(types, lo, hi, below_surface, pore_water) for c in self.ctx]
        self.view_stats = sum_view_stats([c.view_stats for c in self.ctx])
        return np.concatenate(parts, axis=1)

    def voxelize(self, x0, x1, y0, y1, z0, dz, nz):
        """sm_voxelize over the whole map: the window is cut at the strip edges, every rank voxelizes its part, the
        parts are joined along x.  Returns (nz, x1 - x0, y1 - y0) uint8; summed ViewStats in self.view_stats."""
        self.sync()
        parts = [voxel_part(c, x0, x1, y0, y1, z0, dz, nz) for c in self.ctx]
        self.view_stats = sum_view_stats([st for _, st in parts if st is not None])
        return np.concatenate([p for p, _ in parts], axis=1)

    def drainage(self, ground=False):
        """sm_drainage over the whole map: every rank computes the whole map and returns its strip, the strips are
        joined along x.  Returns the dict of (dimx, dimy) rasters; rank 0's DrainStats are kept in self.drain_stats."""
        self.sync()
        parts = [c.drainage(ground) for c in self.ctx]
        self.drain_stats = self.ctx[0].drain_stats
        return {k: np.concatenate([p[k] for p in parts], axis=0) for k in parts[0]}

    def heights(self):
        return np.concatenate([c.heights() for c in self.ctx], axis=0)

    def frequency(self):
        return merge_frequency([c.frequency() for c in self.ctx], self.ranges, self.dimx, self.dimy)

    def frequency_update(self):
        for c in self.ctx:
            c.frequency_update()

    def _run(self, kind, xy, max_sweeps):
        xy = np.ascontiguousarray(xy, np.float32)
        spawn = [c.device_spawn(xy) if len(xy) else None for c in self.ctx]
        for c, d in zip(self.ctx, spawn):          # launch every rank before waiting for any
            (c.water_run_device if kind == "water" else c.wind_run_device)(d, len(xy), max_sweeps)
        stats = [c.last_stats() for c in self.ctx]
        for c, d in zip(self.ctx, spawn):
            if d is not None:
                c.device_free(d)
        return sum_stats(stats)

    def water_run(self, xy, max_sweeps=0):
        return self._run("water", xy, max_sweeps)

    def wind_run(self, xy, max_sweeps=0):
        return self._run("wind", xy, max_sweeps)

    def last_cell_budget(self):
        """per-cell budget maps of the last batch over the whole map, shape (dimx, dimy): the strips concatenated
        along x (a step also writes into its neighbours' strips, so every rank is synchronised first)"""
        self.sync()
        parts = [c.last_cell_budget() for c in self.ctx]
        return {k: np.concatenate([p[k] for p in parts], axis=0) for k in capi.CELL_TERMS}

    # ---- pooling hydrology: one rank issues the call, which reads and writes every strip ----
    def _hydro(self, rank, call):
        self.sync()
        for r, c in enumerate(self.ctx):          # ctx[rank] is the only issuer
            c.hydro_issuer(r == rank)
        st = call(self.ctx[rank])
        self.sync()
        return st

    def water_flood(self, rank=0):
        """flood() of every finished particle of the last water batch over the whole map, issued by ctx[rank]; the
        stats, the budget (ctx[rank].last_hydro_budget()) and any error belong to that context"""
        return self._hydro(rank, lambda c: c.water_flood())

    def seep(self, rank=0):
        """the seep pass over the whole map, issued by ctx[rank]"""
        return self._hydro(rank, lambda c: c.seep())

    # ---- read-only views of the whole map (meshing, export, queries, wind-field boundary) ----
    # Each of these reads other ranks' strips, so every rank's earlier work must have completed first: sync() does
    # that for contexts of this process.
    def sync(self):
        for c in self.ctx:
            c.sync()

    def set_soil_colors(self, rgba):
        for c in self.ctx:
            c.set_soil_colors(rgba)

    def mesh_update(self, slice_):
        """the full-map vertex array (cells, 11), cell order x*dimy + y: every rank meshes its own strip"""
        self.sync()
        return np.concatenate([c.mesh_update(slice_) for c in self.ctx], axis=0)

    def export_height(self):
        return np.concatenate([c.export_height() for c in self.ctx])

    def export_color(self):
        return np.concatenate([c.export_color() for c in self.ctx], axis=0)

    def cell_query(self, x, y, rank=0):
        """global coordinates, any cell of the map; `rank` is the context that issues the call"""
        self.sync()
        return self.ctx[rank].cell_query(x, y)

    def height_bilinear(self, x, y, rank=0):
        self.sync()
        return self.ctx[rank].height_bilinear(x, y)

    def cell_column(self, x, y, capacity=64, rank=0):
        self.sync()
        return self.ctx[rank].cell_column(x, y, capacity)

    # ---- wind field: every rank keeps the whole lattice (identical on every rank) ----
    def lbm_create(self, nx, ny, nz):
        for c in self.ctx:
            c.lbm_create(nx, ny, nz)

    def lbm_set_boundary(self, boundary=None):
        """None: from the terrain of the whole map, built by every rank"""
        if boundary is None:
            self.sync()
        for c in self.ctx:
            c.lbm_set_boundary(boundary)

    def lbm_step(self, n=1):
        """device milliseconds of each rank's steps"""
        return [c.lbm_step(n) for c in self.ctx]

    def wind_use_lbm(self, on=True):
        for c in self.ctx:
            c.wind_use_lbm(on)

    def lbm_get(self, rank=0):
        return self.ctx[rank].lbm_get()


class DistShard:
    """This process's rank of a map sharded over torch.distributed ranks (one GPU each)."""

    def __init__(self, dimx, dimy, scale, device, max_particles=0, pool_capacity=0, share=1, cell_budget=False):
        """share > 1: that many ranks (processes) run their kernels on the SAME device - used by the one-GPU
        test of the CUDA-IPC path; every rank's grid must then be resident at the same time.  cell_budget: keep
        the per-cell budget maps (every rank must agree)."""
        import torch.distributed as dist
        self.dist = dist
        self.nranks, self.rank = dist.get_world_size(), dist.get_rank()
        self.dimx, self.dimy = dimx, dimy
        self.ctx = capi.Context(dimx, dimy, scale, device=device, max_particles=max_particles,
                                pool_capacity=pool_capacity, nranks=self.nranks, rank=self.rank, share=share,
                                cell_budget=cell_budget)
        mine = bytes(self.ctx.peer_export())
        blobs = [None] * self.nranks
        dist.all_gather_object(blobs, mine)
        self.ctx.peer_attach([capi.PeerBlob.from_buffer_copy(b) for b in blobs], use_ipc=True)
        dist.barrier()

    def snapshot(self):
        """the whole-map snapshot on every rank: all ranks must call it (each saves its strip, the strips are
        gathered and joined)"""
        self._settle()
        strips = [None] * self.nranks
        self.dist.all_gather_object(strips, self.ctx.snapshot().tobytes())
        return np.frombuffer(snap.join(strips), np.uint8)

    def restore(self, buf):
        """every rank restores its slice of the same whole-map snapshot (or a strip snapshot of its own range); all
        ranks must call it.  The ranks' checksums are then compared with a whole-map snapshot's header."""
        self._settle()
        self.ctx.restore(buf)
        sums = [None] * self.nranks
        self.dist.all_gather_object(sums, self.ctx.checksum())
        self.dist.barrier()
        check_restored(buf, sums)

    def apply_layer(self, delta, type, leftover=False):
        """sm_apply_layer over the whole map, all or nothing; all ranks must call it, each with its own strip
        (x1 - x0, dimy) of the raster.  Every rank checks, the outcomes are gathered, then every rank applies.  Returns
        this rank's (stats, leftovers or None); a refusal on any rank raises on every rank with no rank written."""
        self._settle()
        ok, _, err = _layer_check(self.ctx, delta, type)
        oks = [None] * self.nranks
        self.dist.all_gather_object(oks, ok)
        if not all(oks):
            raise err if err is not None else capi.SoilMachineError(
                capi.SM_ERR_INVALID, "apply_layer: refused on another rank")
        out = self.ctx.apply_layer(delta, type, leftover=leftover)
        self._settle()
        return out

    def composition(self, types, lo, hi, below_surface=False, pore_water=False):
        """sm_composition on this rank's strip: (len(types), x1 - x0, dimy) float64.  Every rank's earlier work must
        have completed, so all ranks call it; the caller joins the strips along x."""
        self._settle()
        return self.ctx.composition(types, lo, hi, below_surface, pore_water)

    def drainage(self, ground=False):
        """sm_drainage on this rank: the rank computes the whole map through the peer pointers and returns its strip,
        a dict of (x1 - x0, dimy) rasters (basin holds global indices).  Every rank's earlier work must have completed,
        so all ranks call it; each repeats the whole-map work."""
        self._settle()
        return self.ctx.drainage(ground)

    def voxelize(self, x0, x1, y0, y1, z0, dz, nz):
        """sm_voxelize on this rank's part of the window (global coordinates), the window cut at the strip edges:
        (nz, part width, y1 - y0) uint8, of width 0 where the window misses the strip.  All ranks call it."""
        self._settle()
        return voxel_part(self.ctx, x0, x1, y0, y1, z0, dz, nz)[0]

    def run(self, kind, d_xy, n, max_sweeps=0):
        """launch this rank's sweep kernel (all ranks must call it), wait, return local stats"""
        (self.ctx.water_run_device if kind == "water" else self.ctx.wind_run_device)(d_xy, n, max_sweeps)
        return self.ctx.last_stats()

    def last_cell_budget(self):
        """this rank's strip of the per-cell budget maps, shape (x1 - x0, dimy); all ranks must call it (the other
        ranks' steps write into this strip, so every rank's batch has to be complete first)"""
        self._settle()
        return self.ctx.last_cell_budget()

    # ---- pooling hydrology: every process calls, the issuer's context runs it over the whole map ----
    def water_flood(self, issuer=0):
        """flood() of every finished particle of the last water batch; all ranks must call it.  Returns the stats on
        the issuer and None elsewhere (the issuer's context also holds the budget and any error)."""
        self._settle()
        self.ctx.hydro_issuer(self.rank == issuer)
        st = self.ctx.water_flood() if self.rank == issuer else None
        self.dist.barrier()
        return st

    def seep(self, issuer=0):
        """the seep pass over the whole map; all ranks must call it.  Stats on the issuer, None elsewhere."""
        self._settle()
        self.ctx.hydro_issuer(self.rank == issuer)
        st = self.ctx.seep() if self.rank == issuer else None
        self.dist.barrier()
        return st

    # ---- read-only views of the whole map ----
    # The calls that read other ranks' strips first wait for this rank's work and then meet every other rank in a
    # barrier, so all ranks must call them (each with its own arguments).
    def _settle(self):
        self.ctx.sync()
        self.dist.barrier()

    def set_soil_colors(self, rgba):
        self.ctx.set_soil_colors(rgba)

    def mesh_update(self, slice_):
        """this rank's strip of the vertex array ((x1 - x0)*dimy, 11), cell order (x - x0)*dimy + y"""
        self._settle()
        return self.ctx.mesh_update(slice_)

    def export_height(self):
        return self.ctx.export_height()

    def export_color(self):
        return self.ctx.export_color()

    def cell_query(self, x, y):
        """global coordinates, any cell of the map"""
        self._settle()
        return self.ctx.cell_query(x, y)

    def height_bilinear(self, x, y):
        self._settle()
        return self.ctx.height_bilinear(x, y)

    def cell_column(self, x, y, capacity=64):
        self._settle()
        return self.ctx.cell_column(x, y, capacity)

    # ---- wind field: every rank keeps the whole lattice; all ranks make the same calls ----
    def lbm_create(self, nx, ny, nz):
        self.ctx.lbm_create(nx, ny, nz)

    def lbm_set_boundary(self, boundary=None):
        if boundary is None:
            self._settle()
        self.ctx.lbm_set_boundary(boundary)

    def lbm_step(self, n=1):
        return self.ctx.lbm_step(n)

    def wind_use_lbm(self, on=True):
        self.ctx.wind_use_lbm(on)

    def lbm_get(self):
        return self.ctx.lbm_get()

    def close(self):
        self.dist.barrier()
        self.ctx.close()
