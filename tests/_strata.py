"""The statement of the strata views, sm_composition and sm_voxelize, in plain numpy, written from the text of
include/soilmachine_b200.h (DESIGN.md section 13).  It works over any bottom -> top CSR of columns (offsets, type, size,
floor, saturation: sm_download_columns, the reference's columns, snapshot.parse) and walks every column top -> bottom
with the statement's operation order.  The walk is vectorised over cells one depth at a time (the top records, then
the records one below them, ...), so each cell still sees its sections top -> bottom."""
import numpy as np

BELOW_SURFACE = 1
PORE_WATER = 2
NONE = 255


def _arrays(cols):
    off = np.asarray(cols["offsets"], np.int64)
    return (off, np.diff(off), np.asarray(cols["type"], np.int64), np.asarray(cols["size"], np.float64),
            np.asarray(cols["floor"], np.float64), np.asarray(cols["saturation"], np.float64))


def heights(cols):
    """H per cell: top.floor + top.size, 0.0 for an empty column"""
    off, cnt, _, size, floor, _ = _arrays(cols)
    top = np.maximum(off[1:] - 1, 0)
    with np.errstate(all="ignore"):
        return np.where(cnt > 0, floor[top] + size[top], 0.0) if len(size) else np.zeros(len(cnt))


def composition(cols, porosity, types, lo, hi, flags=0, stop_below=False):
    """out[i, cell] for slot i of `types`; porosity: the soil table's float32 porosities.  stop_below=True is the
    negative control: a walk that stops at the first section lying wholly under the window."""
    off, cnt, typ, size, floor, sat = _arrays(cols)
    n = len(cnt)
    por = np.asarray(porosity, np.float32).astype(np.float64)
    slot = np.full(max(256, len(por)), -1, np.int64)
    slot[np.asarray(types, np.int64)] = np.arange(len(types))
    out = np.zeros((len(types), n))
    with np.errstate(all="ignore"):
        if flags & BELOW_SURFACE:
            H = heights(cols)
            a, b = H - hi, H - lo
        else:
            a, b = np.full(n, float(lo)), np.full(n, float(hi))
        live = np.ones(n, bool)
        for d in range(int(cnt.max()) if n else 0):
            cells = np.nonzero((cnt > d) & live)[0]
            i = off[cells + 1] - 1 - d
            t = floor[i] + size[i]
            ov = np.where(t < b[cells], t, b[cells]) - np.where(floor[i] > a[cells], floor[i], a[cells])
            sl = slot[typ[i]]
            m = (ov > 0) & (sl >= 0)
            v = ov * sat[i] * por[typ[i]] if flags & PORE_WATER else ov
            out[sl[m], cells[m]] += v[m]
            if stop_below:
                live[cells[t <= a[cells]]] = False
    return out


def samples(z0, dz, nz):
    """z_k = z0 + (double)k * dz"""
    return z0 + np.arange(nz, dtype=np.float64) * dz


def voxelize(cols, dimy, x0, x1, y0, y1, z0, dz, nz, cx0=0):
    """uint8 (nz, x1 - x0, y1 - y0): the type of the first section met top -> bottom with floor <= z_k < floor + size,
    NONE where no section holds z_k.  cx0: the first column of the CSR (a rank's strip)"""
    off, cnt, typ, size, floor, _ = _arrays(cols)
    z = samples(z0, dz, nz)
    xs, ys = np.meshgrid(np.arange(x0, x1), np.arange(y0, y1), indexing="ij")
    cell = ((xs - cx0) * dimy + ys).reshape(-1)
    out = np.full((len(cell), nz), NONE, np.uint8)
    c = cnt[cell]
    for d in range(int(c.max()) if len(c) else 0):
        w = np.nonzero(c > d)[0]
        i = off[cell[w] + 1] - 1 - d
        inside = (floor[i][:, None] <= z[None, :]) & (z[None, :] < (floor[i] + size[i])[:, None])
        blk = out[w]
        put = inside & (blk == NONE)
        blk[put] = np.broadcast_to(typ[i].astype(np.uint8)[:, None], blk.shape)[put]
        out[w] = blk
    return np.ascontiguousarray(out.T.reshape(nz, x1 - x0, y1 - y0))
