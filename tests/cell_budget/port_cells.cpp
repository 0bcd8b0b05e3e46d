// tests/cell_budget/port_cells.cpp -- the oracle port (oracle/sm_oracle.cpp, compiled into this library unchanged)
// with the per-cell maps of the mass budget.  TEST TOOL ONLY.
//
// The port's cascade / interact functions carry the per-particle accumulators (ACC) only, so the three are restated
// here with the maps as well - the same statements in the same order, plus one addition per measurement, at the ACC
// sites - and driven by smc_water_run / smc_wind_run (the port's move() functions are used as they are: they do not
// change the map).  The tests check that these runs leave the columns bit-identical to the golden frames and the
// per-particle budget identical to the port's, so the restatement is pinned to the port and, through it, to the
// reference.
//
// Maps (soilmachine_b200/csrc/sm_coop.cuh, include/soilmachine_b200.h sm_last_cell_budget): 3 f64 per cell, cell
// order x*dimy + y, terms eroded, deposited, cascade_net; each delta is credited to the cell whose height was read.
// CN counts the measurements per cell (the tests bound the rounding of the per-cell identity with it).
#include "../../oracle/sm_oracle.cpp"

namespace {

std::vector<double> CB;
std::vector<int64_t> CN;

inline void cell_add(int term, int x, int y, double d) {
  const size_t c = (size_t)x * W.dimy + y;
  CB[c * 3 + term] += d;
  CN[c]++;
}

void cascade_c(V2 pos, int transferloop) {                   // cascade, Particle::cascade, particle.h:24-101
  const int ix = (int)std::round(pos.x), iy = (int)std::round(pos.y);
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
    float diff = (height(ix, iy) - height(nx, ny)) * (float)W.SCALE / 80.0f;
    if (diff == 0) continue;
    const int tx = (diff > 0) ? ix : nx, ty = (diff > 0) ? iy : ny;
    const int bx = (diff > 0) ? nx : ix, by = (diff > 0) ? ny : iy;
    const int type = surface(tx, ty);
    const smo_soil param = W.soils[type];
    float excess = std::fabs(diff) - param.maxdiff;
    if (excess <= 0) continue;
    float transfer = param.settling * excess / 2.0f;
    bool recascade = false;
    const double topsize = at(tx, ty).empty() ? 0.0 : at(tx, ty).back().size;
    if (transfer > topsize) transfer = topsize;
    const double ht0 = height(tx, ty), hb0 = height(bx, by);
    if (remove(tx, ty, transfer) != 0) recascade = true;
    add(bx, by, transfer, param.cascades);
    const double dt = height(tx, ty) - ht0, db = height(bx, by) - hb0;
    if (ACC) ACC[2] += dt + db;
    cell_add(2, tx, ty, dt);
    cell_add(2, bx, by, db);
    if (recascade && transferloop > 0) cascade_c({(float)nx, (float)ny}, --transferloop);
  }
}

bool water_interact_c(Water& p) {                            // water_interact, water.h:75-121
  double c_eq = p.param.solubility * (height(p.ix, p.iy) - height_bilinear(p.pos)) * (double)W.SCALE / 80.0;
  if (c_eq < 0.0) c_eq = 0.0;
  if (c_eq > 1.0) c_eq = 1.0;
  const int ind = p.iy * W.dimx + p.ix;
  if ((double)(W.soils[p.contains].erosionrate) < W.wfreq[ind]) p.contains = W.soils[p.contains].erodes;
  const double cdiff = c_eq - p.sediment;
  if (cdiff > 0) {
    p.sediment += p.param.equrate * cdiff;
    p.contains = W.soils[surface(p.ix, p.iy)].transports;
    const double h0 = height(p.ix, p.iy);
    double diff = remove(p.ix, p.iy, p.param.equrate * cdiff * p.volume);
    while (std::fabs(diff) > 1E-8) diff = remove(p.ix, p.iy, diff);
    const double d = h0 - height(p.ix, p.iy);
    if (ACC) ACC[0] += d;
    cell_add(0, p.ix, p.iy, d);
  } else if (cdiff < 0) {
    p.sediment += W.soils[p.contains].equrate * cdiff;
    const double h0 = height(p.ix, p.iy);
    add(p.ix, p.iy, -W.soils[p.contains].equrate * cdiff * p.volume, p.contains);
    const double d = height(p.ix, p.iy) - h0;
    if (ACC) ACC[1] += d;
    cell_add(1, p.ix, p.iy, d);
  }
  cascade_c(p.pos, 0);
  p.sediment /= (1.0 - p.evaprate);
  const double over = p.sediment - 1.0;
  if (p.sediment > 1.0) p.sediment = 1.0;
  p.volume *= (1.0 - p.evaprate);
  if (ACC) {
    if (over > 0.0) ACC[4] += over * p.volume;
    if (!(p.volume > 0.01)) ACC[3] += p.sediment * p.volume;
  }
  return p.volume > 0.01;
}

bool wind_interact_c(Wind& p) {                              // wind_interact, wind.h:94-136
  const int nx = (int)std::round(p.pos.x), ny = (int)std::round(p.pos.y);
  if (p.height <= height_bilinear(p.pos) * (float)W.SCALE / 80.0f) {
    if (p.param.transports == p.contains) {
      const float len = std::sqrt(p.speed.x * p.speed.x + p.speed.y * p.speed.y + p.speed.z * p.speed.z);
      double force = len * (height(nx, ny) - p.height) * (float)W.SCALE / 80.0f * (1.0f - p.sediment);
      const double h0 = height(p.ix, p.iy);
      double diff = remove(p.ix, p.iy, p.param.suspension * force);
      const double d = h0 - height(p.ix, p.iy);
      if (ACC) { ACC[0] += d; if (p.param.suspension * force < 0.0) ACC[5] += p.param.suspension * force; }
      cell_add(0, p.ix, p.iy, d);
      p.sediment += (p.param.suspension * force - diff);
      cascade_c({(float)p.ix, (float)p.iy}, 1);
    }
  } else if (p.param.suspension > 0.0) {
    p.sediment -= W.soils[p.contains].suspension * p.sediment;
    double h0 = height(nx, ny);
    add(nx, ny, 0.5f * W.soils[p.contains].suspension * p.sediment, p.contains);
    double d = height(nx, ny) - h0;
    if (ACC) ACC[1] += d;
    cell_add(1, nx, ny, d);
    h0 = height(p.ix, p.iy);
    add(p.ix, p.iy, 0.5f * W.soils[p.contains].suspension * p.sediment, p.contains);
    d = height(p.ix, p.iy) - h0;
    if (ACC) ACC[1] += d;
    cell_add(1, p.ix, p.iy, d);
    cascade_c({(float)p.ix, (float)p.iy}, 1);
    cascade_c({(float)nx, (float)ny}, 1);
  }
  return true;
}

void reset_cells() {
  CB.assign((size_t)W.dimx * W.dimy * 3, 0.0);
  CN.assign((size_t)W.dimx * W.dimy, 0);
}

}  // namespace

extern "C" {
// smo_water_run / smo_wind_run with the maps (reset at the start of the batch)
void smc_water_run(int n, const float* xy, int max_sweeps, smo_stats* st) {
  memset(st, 0, sizeof(*st));
  smo_water_begin(n, xy);
  reset_cells();
  while (!Wlive.empty() && (max_sweeps <= 0 || st->sweeps < max_sweeps)) {   // smo_water_sweep
    std::vector<int> next;
    for (int i : Wlive) {
      Water& p = WP[i];
      bool moved = false, lives = false;
      with_budget(i, [&]() { moved = water_move(p); if (moved) lives = water_interact_c(p); });
      if (!moved) { if (p.volume == 0.0) st->exit_oob++; else st->exit_stall++; continue; }
      st->steps++;
      if (!lives) { st->exit_evap++; continue; }
      next.push_back(i);
    }
    Wlive.swap(next); st->sweeps++;
  }
}
void smc_wind_run(int n, const float* xy, int max_sweeps, smo_stats* st) {
  memset(st, 0, sizeof(*st));
  smo_wind_begin(n, xy);
  reset_cells();
  while (!Dlive.empty() && (max_sweeps <= 0 || st->sweeps < max_sweeps)) {    // smo_wind_sweep
    std::vector<int> next;
    for (int i : Dlive) {
      Wind& p = DP[i];
      bool moved = false, lives = false;
      with_budget(i, [&]() { moved = wind_move(p); if (moved) lives = wind_interact_c(p); });
      if (!moved) { st->exit_oob++; continue; }
      st->steps++;
      if (!lives) { st->exit_evap++; continue; }
      next.push_back(i);
    }
    Dlive.swap(next); st->sweeps++;
  }
}
// the maps of the last smc_*_run (3 per cell, interleaved) and the number of measurements per cell
void smc_cell_budget(double* out3, int64_t* nops) {
  if (out3) memcpy(out3, CB.data(), CB.size() * sizeof(double));
  if (nops) memcpy(nops, CN.data(), CN.size() * sizeof(int64_t));
}
}
