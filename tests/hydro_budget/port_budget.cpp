// tests/hydro_budget/port_budget.cpp -- the oracle port (oracle/sm_oracle.cpp, compiled into this library unchanged)
// with the mass budget of the pooling hydrology.  TEST TOOL ONLY.
//
// The port's own flood / water-table cascade / nested-particle functions carry no accumulators, so the three are
// restated here with them - the same statements in the same order, plus the budget's height reads - and driven by
// smob_water_flood / smob_seep next to the port's smo_* calls (same map, same particle batch).  The tests check that
// these calls leave the map bit-identical to smo_water_flood / smo_seep, so the restatement is pinned to the port and,
// through it, to the reference.
//
// Eleven f64 accumulators per call, the same definitions and order of additions as the product's
// (soilmachine_b200/csrc/sm_hydro_coop.cuh; include/soilmachine_b200.h, sm_hydro_budget): flood_sediment,
// flood_cascade_net, flood_water, seeped, to_particles, transfer_net, then slots 0-4 of the step budget (the port's
// ACC) summed over the nested particles' steps.
#include "../../oracle/sm_oracle.cpp"

namespace {

double HB[11];

// run f with the port's step accumulators (ACC) pointed at `acc`, zeroed first
template <class F> inline void with_local_acc(double* acc, F f) {
  for (int k = 0; k < 6; k++) acc[k] = 0.0;
  double* const outer = ACC;
  ACC = acc;
  f();
  ACC = outer;
}

// seep(cell) with its budget term: the height it removes (a seep into a non-Air top changes saturation only)
void water_seep_b(int x, int y) {
  const double h0 = height(x, y);
  water_seep(x, y);
  HB[3] += h0 - height(x, y);
}

void water_cascade_b(int ix, int iy, int spill);

bool water_flood_b(Water& p) {                               // water_flood, WaterParticle::flood, water.h:123-145
  if (p.volume < 0.01 || p.spill-- <= 0) return false;
  H.floods++;
  p.ix = (int)p.pos.x; p.iy = (int)p.pos.y;
  double h0 = height(p.ix, p.iy);
  add(p.ix, p.iy, p.sediment * W.soils[p.contains].equrate, p.contains);
  HB[0] += height(p.ix, p.iy) - h0;
  double acc[6];
  with_local_acc(acc, [&]() { cascade(p.pos, 0); });
  HB[1] += acc[2];
  h0 = height(p.ix, p.iy);
  add(p.ix, p.iy, p.volume * volumeFactor, AIR);
  HB[2] += height(p.ix, p.iy) - h0;
  water_seep_b(p.ix, p.iy);
  water_cascade_b(p.ix, p.iy, p.spill);
  return false;
}

void water_to_completion_b(Water& p, int64_t* steps) {       // water_to_completion, water.h:252-256
  for (;;) {
    for (;;) {                                               // while (move() && interact())
      bool moved = false, lives = false;
      double acc[6];
      with_local_acc(acc, [&]() { moved = water_move(p); if (moved) lives = water_interact(p); });
      for (int k = 0; k < 5; k++) HB[6 + k] += acc[k];
      if (!moved) break;
      ++*steps;
      if (!lives) break;
    }
    if (!water_flood_b(p)) break;
  }
}

void water_cascade_b(int ix, int iy, int spill) {            // water_cascade, WaterParticle::cascade, water.h:151-283
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
      HB[4] += h0 - height(tx, ty);
      Water q;
      water_spawn(q, (float)tx, (float)ty);
      const V2 d = {(float)bx - (float)tx, (float)by - (float)ty};
      const float inv = 1.0f / std::sqrt(d.x * d.x + d.y * d.y);
      const float r2 = std::sqrt(2.0f);
      q.speed = {r2 * (d.x * inv), r2 * (d.y * inv)};
      q.spill = spill;
      q.volume = transfer / volumeFactor;
      H.nested++;
      water_to_completion_b(q, &H.nested_steps);
    } else {
      const double ht0 = height(tx, ty), hb0 = height(bx, by);
      if (remove(tx, ty, transfer) != 0) recascade = true;
      if (transfer > 0) recascade = true;
      add(bx, by, transfer, AIR);
      at(bx, by).back().saturation = 1.0f;
      HB[5] += (height(tx, ty) - ht0) + (height(bx, by) - hb0);
      H.transfers++;
    }
    if (recascade && spill > 0) water_cascade_b(nx, ny, --spill);
  }
}

}  // namespace

extern "C" {
// smo_water_flood / smo_seep with the budget; smob_hydro_budget: the eleven sums of the last of these calls
void smob_water_flood(smo_hydro* out) {
  H = smo_hydro();
  for (double& b : HB) b = 0.0;
  std::vector<char> live(WP.size(), 0);
  for (int i : Wlive) live[i] = 1;
  for (size_t i = 0; i < WP.size(); i++) if (!live[i]) water_flood_b(WP[i]);
  if (out) *out = H;
}
void smob_seep(smo_hydro* out) {
  H = smo_hydro();
  for (double& b : HB) b = 0.0;
  for (int x = 0; x < W.dimx; x++) for (int y = 0; y < W.dimy; y++) {
    water_seep_b(x, y);
    water_cascade_b(x, y, 3);
    H.cells++;
  }
  if (out) *out = H;
}
void smob_hydro_budget(double* out11) { memcpy(out11, HB, sizeof(HB)); }
}
