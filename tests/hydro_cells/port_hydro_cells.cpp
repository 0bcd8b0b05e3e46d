// tests/hydro_cells/port_hydro_cells.cpp -- the oracle port with the per-cell maps of the pooling hydrology's mass
// budget.  TEST TOOL ONLY.
//
// tests/cell_budget/port_cells.cpp (the port compiled unchanged, plus its restated cascade and water interact, whose
// hooks credit terms 0-2 per cell) is compiled into this library as it is.  The port's flood, water-table cascade and
// nested-particle loop are restated here, as tests/hydro_budget/port_budget.cpp restates them for the sums: the same
// statements in the same order, plus the height reads and one addition per measurement.  smh_water_flood / smh_seep
// drive them next to the port's smo_* calls (same map, same particle batch); the tests check that they leave the columns
// and counters bit-identical to smo_water_flood / smo_seep.
//
// Maps (soilmachine_b200/csrc/sm_hydro_coop.cuh, include/soilmachine_b200.h sm_last_hydro_cell_budget): 4 f64 per
// cell, cell order x*dimy + y, terms eroded, deposited, cascade_net, water_net.  Terms 0-2 go through port_cells.cpp's
// cell_add (its map CB and count CN), term 3 into WN here (counted in CN as well); smh_cell_budget interleaves them.
// Each term is a separate running total per cell, so keeping them in two arrays changes no addition.
#include "../cell_budget/port_cells.cpp"

namespace {

std::vector<double> WN;   // term 3, water_net, per cell

inline void water_add(int x, int y, double d) {
  const size_t c = (size_t)x * W.dimy + y;
  WN[c] += d;
  CN[c]++;
}

void reset_hydro_cells() {
  reset_cells();
  WN.assign((size_t)W.dimx * W.dimy, 0.0);
}

// seep(cell), its removed height credited negative.  `pass`: a visit of the seep pass.  The port's pass visits every
// cell, the device's only the flagged ones; a visit that changes nothing adds -0.0, which leaves any total as it is
// (a total starts at +0.0 and a sum of two doubles is -0.0 only when both are), so it is not counted.
void water_seep_h(int x, int y, bool pass) {
  const double h0 = height(x, y);
  water_seep(x, y);
  const double d = h0 - height(x, y);
  if (!pass || d != 0.0) water_add(x, y, -d);
}

void water_cascade_h(int ix, int iy, int spill);

bool water_flood_h(Water& p) {                               // water_flood, WaterParticle::flood, water.h:123-145
  if (p.volume < 0.01 || p.spill-- <= 0) return false;
  H.floods++;
  p.ix = (int)p.pos.x; p.iy = (int)p.pos.y;
  double h0 = height(p.ix, p.iy);
  add(p.ix, p.iy, p.sediment * W.soils[p.contains].equrate, p.contains);
  cell_add(1, p.ix, p.iy, height(p.ix, p.iy) - h0);
  cascade_c(p.pos, 0);
  h0 = height(p.ix, p.iy);
  add(p.ix, p.iy, p.volume * volumeFactor, AIR);
  water_add(p.ix, p.iy, height(p.ix, p.iy) - h0);
  water_seep_h(p.ix, p.iy, false);
  water_cascade_h(p.ix, p.iy, p.spill);
  return false;
}

void water_to_completion_h(Water& p, int64_t* steps) {       // water_to_completion, water.h:252-256
  for (;;) {
    while (water_move(p)) {
      ++*steps;
      if (!water_interact_c(p)) break;
    }
    if (!water_flood_h(p)) break;
  }
}

void water_cascade_h(int ix, int iy, int spill) {            // water_cascade, WaterParticle::cascade, water.h:151-283
  static const int nx8[8] = {-1, -1, -1, 0, 0, 1, 1, 1};
  static const int ny8[8] = {-1, 0, 1, -1, 1, -1, 0, 1};
  struct Point { int x, y; double h; } sn[8];
  int num = 0;
  for (int k = 0; k < 8; k++) {
    const int nx = ix + nx8[k], ny = iy + ny8[k];
    if (nx >= W.dimx || ny >= W.dimy || nx < 0 || ny < 0) continue;
    sn[num++] = {nx, ny, height(nx, ny)};
  }
  for (int i = 1; i < num; i++) {
    Point v = sn[i];
    int j = i;
    while (j > 0 && v.h > sn[j - 1].h) { sn[j] = sn[j - 1]; j--; }
    sn[j] = v;
  }
  for (int i = 0; i < num; i++) {
    const int nx = sn[i].x, ny = sn[i].y;
    const Column& A = at(ix, iy);
    const Column& B = at(nx, ny);
    double whA = 0, whB = 0, fA = 0.0, fB = 0.0;
    if (!A.empty()) { whA = A.back().size; fA = A.back().floor; }
    if (!B.empty()) { whB = B.back().size; fB = B.back().floor; }
    const double diff = (fA + whA - fB - whB) * (double)W.SCALE / 80.0;
    if (diff == 0) continue;
    const int tx = (diff > 0) ? ix : nx, ty = (diff > 0) ? iy : ny;
    const int bx = (diff > 0) ? nx : ix, by = (diff > 0) ? ny : iy;
    const Column& top = at(tx, ty);
    if (top.empty() || top.back().type != AIR) continue;
    double transfer = std::fabs(diff) / 2.0;
    const double wh = top.back().size;
    transfer = (wh < transfer) ? wh : transfer;
    if (transfer <= 0) continue;
    bool recascade = false;
    if (transfer == wh) {                                    // the whole water section leaves as a particle
      const double h0 = height(tx, ty);
      remove(tx, ty, transfer);
      water_add(tx, ty, -(h0 - height(tx, ty)));
      Water q;
      water_spawn(q, (float)tx, (float)ty);
      const V2 d = {(float)bx - (float)tx, (float)by - (float)ty};
      const float inv = 1.0f / std::sqrt(d.x * d.x + d.y * d.y);
      const float r2 = std::sqrt(2.0f);
      q.speed = {r2 * (d.x * inv), r2 * (d.y * inv)};
      q.spill = spill;
      q.volume = transfer / volumeFactor;
      H.nested++;
      water_to_completion_h(q, &H.nested_steps);
    } else {
      const double ht0 = height(tx, ty), hb0 = height(bx, by);
      if (remove(tx, ty, transfer) != 0) recascade = true;
      if (transfer > 0) recascade = true;
      add(bx, by, transfer, AIR);
      at(bx, by).back().saturation = 1.0f;
      water_add(tx, ty, height(tx, ty) - ht0);
      water_add(bx, by, height(bx, by) - hb0);
      H.transfers++;
    }
    if (recascade && spill > 0) water_cascade_h(nx, ny, --spill);
  }
}

}  // namespace

extern "C" {
// smo_water_flood / smo_seep with the maps (reset at the start of the call)
void smh_water_flood(smo_hydro* out) {
  H = smo_hydro();
  reset_hydro_cells();
  std::vector<char> live(WP.size(), 0);
  for (int i : Wlive) live[i] = 1;
  for (size_t i = 0; i < WP.size(); i++) if (!live[i]) water_flood_h(WP[i]);
  if (out) *out = H;
}
void smh_seep(smo_hydro* out) {
  H = smo_hydro();
  reset_hydro_cells();
  for (int x = 0; x < W.dimx; x++) for (int y = 0; y < W.dimy; y++) {
    water_seep_h(x, y, true);
    water_cascade_h(x, y, 3);
    H.cells++;
  }
  if (out) *out = H;
}
// the maps of the last smh_* call (4 per cell, interleaved) and the number of measurements per cell
void smh_cell_budget(double* out4, int64_t* nops) {
  const size_t n = WN.size();
  if (out4)
    for (size_t c = 0; c < n; c++) {
      for (int k = 0; k < 3; k++) out4[c * 4 + k] = CB[c * 3 + k];
      out4[c * 4 + 3] = WN[c];
    }
  if (nops) memcpy(nops, CN.data(), n * sizeof(int64_t));
}
}
