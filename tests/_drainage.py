"""The statement of the drainage view, sm_drainage, in numpy and heapq, written from the text of
include/soilmachine_b200.h (DESIGN.md section 14): a priority-flood for the spill height W, a breadth-first search for
the flat distances, the receiver rule, the areas in topological order and the basins down each chain.  It reads a
height raster (dimx, dimy), or a bottom -> top CSR of columns for the ground rule."""
import heapq
import math

import numpy as np

GROUND = 1
# n[] of the reference's water.h:155-164, as (dx, dy)
N8 = [(-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 1), (1, -1), (1, 0), (1, 1)]
SQRT2 = math.sqrt(2.0)


def heights(cols, ground=False):
    """H per cell of a CSR: top.floor + top.size (0.0 for an empty column); ground: floor + size of the first section
    met top -> bottom whose type is not Air, 0.0 if there is none"""
    off = np.asarray(cols["offsets"], np.int64)
    typ = np.asarray(cols["type"], np.int64)
    top = np.asarray(cols["floor"], np.float64) + np.asarray(cols["size"], np.float64)
    out = np.zeros(len(off) - 1)
    for c in range(len(off) - 1):
        for i in range(off[c + 1] - 1, off[c] - 1, -1):
            if not ground or typ[i] != 0:
                out[c] = top[i]
                break
    return out


def drainage(H):
    """H: float64 (dimx, dimy).  Returns dict spill, dir, area, basin (the header's outputs, (dimx, dimy)) and stats
    flat_cells, depressed_cells, outlets, plus dist (the flat distances)."""
    H = np.asarray(H, np.float64)
    dimx, dimy = H.shape
    border = np.zeros((dimx, dimy), bool)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
    # spill: priority-flood from the border, W(n) = max(H(n), W(c)) when first reached from the lowest c
    W = np.full((dimx, dimy), np.inf)
    done = np.zeros((dimx, dimy), bool)
    heap = [(float(H[x, y]), x, y) for x, y in zip(*np.nonzero(border))]
    for w, x, y in heap:
        W[x, y] = w
    heapq.heapify(heap)
    while heap:
        w, x, y = heapq.heappop(heap)
        if done[x, y]:
            continue
        done[x, y] = True
        for dx, dy in N8:
            u, v = x + dx, y + dy
            if 0 <= u < dimx and 0 <= v < dimy and not done[u, v]:
                nw = max(float(H[u, v]), w)
                if nw < W[u, v]:
                    W[u, v] = nw
                    heapq.heappush(heap, (nw, u, v))
    Wp = np.pad(W, 1, constant_values=np.inf)
    nb = np.stack([Wp[1 + dx:1 + dx + dimx, 1 + dy:1 + dy + dimy] for dx, dy in N8])
    drained = (nb < W[None]).any(0) & ~border
    flat = ~border & ~drained
    # dist: breadth-first from every drained or border cell, through cells of equal W
    dist = np.where(flat, -1, 0).astype(np.int64)
    frontier = list(zip(*np.nonzero(~flat)))
    d = 0
    while frontier:
        nxt = []
        for x, y in frontier:
            for dx, dy in N8:
                u, v = x + dx, y + dy
                if 0 <= u < dimx and 0 <= v < dimy and dist[u, v] < 0 and W[u, v] == W[x, y]:
                    dist[u, v] = d + 1
                    nxt.append((u, v))
        frontier, d = nxt, d + 1
    assert (dist >= 0).all(), "a flat cell the search did not reach"
    # receivers
    dirs = np.full((dimx, dimy), -1, np.int8)
    for x in range(1, dimx - 1):
        for y in range(1, dimy - 1):
            wc, best, bs = W[x, y], -1, 0.0
            for k, (dx, dy) in enumerate(N8):
                wn = W[x + dx, y + dy]
                if wn < wc:
                    s = (wc - wn) / (SQRT2 if dx and dy else 1.0)
                    if best < 0 or s > bs:
                        best, bs = k, s
            if best < 0:
                for k, (dx, dy) in enumerate(N8):
                    if W[x + dx, y + dy] == wc and dist[x + dx, y + dy] == dist[x, y] - 1:
                        best = k
                        break
            assert best >= 0, "no receiver at (%d, %d)" % (x, y)
            dirs[x, y] = best
    # every hop lowers W, or keeps W and lowers dist: sorting by (W, dist) descending puts donors before receivers
    idx = np.arange(dimx * dimy).reshape(dimx, dimy)
    dx_ = np.array([0] + [p[0] for p in N8])[dirs.astype(np.int64) + 1]
    dy_ = np.array([0] + [p[1] for p in N8])[dirs.astype(np.int64) + 1]
    rcv = np.where(dirs >= 0, idx + dx_ * dimy + dy_, -1).reshape(-1)
    order = np.lexsort((-dist.reshape(-1), -W.reshape(-1)))
    area = np.ones(dimx * dimy, np.int64)
    for i in order:
        if rcv[i] >= 0:
            area[rcv[i]] += area[i]
    basin = np.arange(dimx * dimy, dtype=np.int64)
    for i in order[::-1]:
        if rcv[i] >= 0:
            basin[i] = basin[rcv[i]]
    return {"spill": W, "dir": dirs, "area": area.reshape(dimx, dimy), "basin": basin.reshape(dimx, dimy),
            "dist": dist, "flat_cells": int(flat.sum()), "depressed_cells": int((W > H).sum()),
            "outlets": int((border & (area.reshape(dimx, dimy) > 1)).sum())}


# ---- crafted rasters --------------------------------------------------------------------------------------------------
def nested(dimx=24, dimy=20):
    """a rim with a pit, inside it a second rim with a deeper pit, on a tilted plain"""
    x, y = np.meshgrid(np.arange(dimx), np.arange(dimy), indexing="ij")
    H = 1.0 + 0.01 * x + 0.003 * y
    r = np.maximum(abs(x - dimx // 2), abs(y - dimy // 2))
    H[r == 7] = 5.0
    H[r < 7] = 2.0
    H[r == 3] = 4.0
    H[r < 3] = 0.5
    H[dimx // 2 + 7, dimy // 2] = 3.0          # the outer rim's spill point
    return H


def plateau(dimx=18, dimy=22):
    """a flat plateau that touches the border on one side, with a pit in it and a slope behind it"""
    x, y = np.meshgrid(np.arange(dimx), np.arange(dimy), indexing="ij")
    H = np.where(x < 9, 3.0, 3.0 + 0.25 * (x - 8))
    H[4:7, 8:11] = 2.0
    return H


def equal(dimx=13, dimy=11, h=1.5):
    return np.full((dimx, dimy), h)


def spiral(n=32):
    """a channel one cell wide that spirals inwards from an outlet on the border, between walls one cell wide: the
    water of the innermost cell passes about n^2 / 2 cells"""
    H = np.full((n, n), 10.0)
    path = [(0, 1), (1, 1)]
    on = np.zeros((n, n), bool)
    on[0, 1] = on[1, 1] = True
    x, y, dx, dy = 1, 1, 0, 1

    def free(u, v):
        return 1 <= u <= n - 2 and 1 <= v <= n - 2 and not on[u, v]
    turns = 0
    while turns < 2:
        if free(x + dx, y + dy) and free(x + 2 * dx, y + 2 * dy) or (free(x + dx, y + dy) and not (
                1 <= x + 2 * dx <= n - 2 and 1 <= y + 2 * dy <= n - 2)):
            x, y = x + dx, y + dy
            on[x, y] = True
            path.append((x, y))
            turns = 0
        else:
            dx, dy = dy, -dx
            turns += 1
    for i, (u, v) in enumerate(path):
        H[u, v] = 1.0 + 8.0 * i / len(path)         # rising inwards, below the walls everywhere
    return H


def ties():
    """exact slope ties between a diagonal and an edge neighbour.  With s = 2.0 / sqrt(2.0) rounded, a cell at 2.0
    has the diagonal slope s towards 0.0 and the edge slope 2.0 - (2.0 - s) = s towards 2.0 - s (both subtractions
    exact).  At (1, 1) the diagonal is k = 0 and the edge k = 3: dir 0.  At (4, 4) the edge is k = 4 and the diagonal
    k = 7: dir 4."""
    s = 2.0 / SQRT2
    H = np.full((6, 6), 3.0)
    H[1:5, 1:5] = 2.5
    H[1, 1] = H[4, 4] = 2.0
    H[0, 0], H[1, 0] = 0.0, 2.0 - s
    H[5, 5], H[4, 5] = 0.0, 2.0 - s
    return H


def narrow():
    """the narrowest maps sm_create accepts (2 cells) and one more, in x and in y, on random heights"""
    rng = np.random.default_rng(5)
    return [np.round(rng.random(s) * 4, 1) for s in ((2, 9), (9, 2), (3, 9), (9, 3), (2, 2), (3, 3))]


def crafted():
    out = [("nested", nested()), ("plateau", plateau()), ("equal", equal()), ("spiral", spiral()), ("ties", ties())]
    out += [("narrow%dx%d" % h.shape, h) for h in narrow()]
    return out
