// tests/drainage/host_drain.cpp -- the drainage view's per-cell logic (soilmachine_b200/csrc/sm_drain.cuh) compiled
// for the host and driven by a serial loop.  TEST TOOL ONLY.
//
// hdrain_heights  H of every cell of a top / pool image (ground: SM_DRAIN_GROUND)
// hdrain_run      spill, dir, area and basin of an H raster: the fill and the flat distances relaxed from a work
//                 queue (any order reaches the same fixed point; the flats' queue starts at the edges of the flats,
//                 so it runs breadth-first), the receivers cell by cell, the areas in Kahn's order, the basins down
//                 each chain
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../soilmachine_b200/csrc/sm_strata.cuh"
#include "../../soilmachine_b200/csrc/sm_drain.cuh"

namespace {
struct Grid {
  int dimx, dimy;
  bool border(int x, int y) const { return x == 0 || y == 0 || x == dimx - 1 || y == dimy - 1; }
  template <class T> void window(const T* a, int x, int y, T* out) const {
    for (int k = 0; k < 8; k++) out[k] = a[(size_t)(x + drain_dx(k)) * dimy + (y + drain_dy(k))];
  }
};
// relax the cells for which live(i) holds with step(i) (true: the cell's value dropped) until the queue empties; the
// queue starts with the cells for which seed(i) holds, and a cell that drops puts its live neighbours on it
template <class L, class S, class Q> void relax(const Grid& g, L live, S step, Q seed) {
  const size_t n = (size_t)g.dimx * g.dimy;
  std::vector<size_t> q;
  std::vector<char> inq(n, 0);
  for (size_t i = 0; i < n; i++)
    if (live(i) && seed(i)) { q.push_back(i); inq[i] = 1; }
  for (size_t h = 0; h < q.size(); h++) {
    const size_t i = q[h];
    inq[i] = 0;
    if (!step(i)) continue;
    const int x = (int)(i / g.dimy), y = (int)(i % g.dimy);
    for (int k = 0; k < 8; k++) {
      const size_t j = (size_t)(x + drain_dx(k)) * g.dimy + (y + drain_dy(k));
      if (!inq[j] && live(j)) { q.push_back(j); inq[j] = 1; }
    }
    if (h > (1u << 20) && h * 2 > q.size()) { q.erase(q.begin(), q.begin() + h + 1); h = (size_t)-1; }
  }
}
}  // namespace

extern "C" {
void hdrain_heights(int64_t ncells, const Sec32* top, const Sec32* pool, int32_t ground, double* H) {
  const StrataPool a{pool};
  for (int64_t c = 0; c < ncells; c++) H[c] = drain_column_height(a, top[c], ground != 0);
}

// stats: fill updates, flat cells, depressed cells, outlets.  Returns 0, or -1 when a cell has no receiver.
int hdrain_run(int32_t dimx, int32_t dimy, const double* H, double* W, int8_t* dir, int64_t* area, int64_t* basin,
               int64_t* stats) {
  const Grid g{dimx, dimy};
  const size_t n = (size_t)dimx * dimy;
  for (size_t i = 0; i < n; i++) W[i] = g.border((int)(i / dimy), (int)(i % dimy)) ? H[i] : (double)INFINITY;
  auto interior = [&](size_t i) { return !g.border((int)(i / dimy), (int)(i % dimy)); };
  int64_t updates = 0;
  relax(g, interior, [&](size_t i) {
    double wn[8];
    g.window(W, (int)(i / dimy), (int)(i % dimy), wn);
    const double v = drain_fill_value(H[i], wn);
    if (!(v < W[i])) return false;
    W[i] = v;
    updates++;
    return true;
  }, interior);
  std::vector<int32_t> D(n, SM_DRAIN_NOT_FLAT);
  int64_t flat = 0, dep = 0, outlets = 0;
  for (size_t i = 0; i < n; i++) {
    dep += W[i] > H[i];
    if (!interior(i)) continue;
    double wn[8];
    g.window(W, (int)(i / dimy), (int)(i % dimy), wn);
    if (!drain_drained(W[i], wn)) { D[i] = SM_DRAIN_FAR; flat++; }
  }
  relax(g, [&](size_t i) { return interior(i) && D[i] != SM_DRAIN_NOT_FLAT; }, [&](size_t i) {
    double wn[8];
    int32_t dn[8];
    g.window(W, (int)(i / dimy), (int)(i % dimy), wn);
    g.window(D.data(), (int)(i / dimy), (int)(i % dimy), dn);
    const int32_t v = drain_dist_value(W[i], D[i], wn, dn);
    if (!(v < D[i])) return false;
    D[i] = v;
    return true;
  }, [&](size_t i) {       // the flats next to the edge of their flat: first-in first-out is then breadth-first
    const int x = (int)(i / dimy), y = (int)(i % dimy);
    for (int k = 0; k < 8; k++) {
      const size_t j = (size_t)(x + drain_dx(k)) * dimy + (y + drain_dy(k));
      if (D[j] == SM_DRAIN_NOT_FLAT && W[j] == W[i]) return true;
    }
    return false;
  });
  std::vector<int64_t> rcv(n, -1);
  std::vector<int32_t> indeg(n, 0);
  for (size_t i = 0; i < n; i++) {
    int k = -1;
    if (interior(i)) {
      const int x = (int)(i / dimy), y = (int)(i % dimy);
      double wn[8];
      int32_t dn[8];
      g.window(W, x, y, wn);
      g.window(D.data(), x, y, dn);
      k = drain_receiver(W[i], D[i], wn, dn);
      if (k < 0) return -1;
      rcv[i] = (int64_t)(x + drain_dx(k)) * dimy + (y + drain_dy(k));
      indeg[rcv[i]]++;
    }
    dir[i] = (int8_t)k;
  }
  // Kahn's order: a cell is passed on when its last donor has been
  std::vector<int64_t> order;
  order.reserve(n);
  std::vector<int32_t> rem(indeg);
  for (size_t i = 0; i < n; i++) { area[i] = 1; if (indeg[i] == 0) order.push_back((int64_t)i); }
  for (size_t h = 0; h < order.size(); h++) {
    const int64_t i = order[h], r = rcv[i];
    if (r < 0) continue;
    area[r] += area[i];
    if (--rem[r] == 0) order.push_back(r);
  }
  if (order.size() != n) return -1;
  for (size_t h = n; h-- > 0;) {       // receivers before donors
    const int64_t i = order[h];
    basin[i] = rcv[i] < 0 ? i : basin[rcv[i]];
  }
  for (size_t i = 0; i < n; i++) outlets += !interior(i) && indeg[i] > 0;
  stats[0] = updates; stats[1] = flat; stats[2] = dep; stats[3] = outlets;
  return 0;
}
}
