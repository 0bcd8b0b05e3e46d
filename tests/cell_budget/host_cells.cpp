// tests/cell_budget/host_cells.cpp -- tests/hostsim (compiled into this library unchanged) with the per-cell maps of
// the mass budget.  TEST TOOL ONLY.  HostCellBack is hostsim's HostBack plus the map hook (kCellBudget,
// cell_budget), so hc_water_sweep / hc_wind_sweep run the product's warp-cooperative step (sm_coop.cuh) with the maps
// on, as the device's k_sweep<..., CELLS = true> does; the lanes are loops in the order hs_set_mode chose.
#include "../hostsim/hostsim.cpp"

namespace {
std::vector<double> G_cells;   // 3 per cell, interleaved (eroded, deposited, cascade_net), cell order x*dimy + y

struct HostCellBack : HostBack {
  static constexpr bool kCellBudget = true;
  void cell_budget(int term, int x, int y, double d) { G_cells[((size_t)x * M.dimy + y) * 3 + term] += d; }
};

// one step of particle p: split = 1 stages only the plus-shaped stencil before move() and the rest after it, as the
// exact-footprint schedule does (sweep_exact), split = 0 stages the whole block (the conservative path)
template <class P, class MID>
int step_cells(P& p, int split, int (*mv)(WarpHost&, CoopWin<HostCellBack>&, P&, MID&, uint32_t),
               int (*ia)(WarpHost&, CoopWin<HostCellBack>&, P&, const MID&), double* acc) {
  WarpHost w; HostCellBack b; CoopScratch sc; CoopWin<HostCellBack> cw(b, &sc);
  MID mid;
  int r = mv(w, cw, p, mid, split ? SM_CW_PLUS : 0x1FFu);
  if (r == SM_ALIVE) r = ia(w, cw, p, mid);
  cw.flush(w);
  for (int k = 0; k < SM_BUDGET_SLOTS; k++) acc[k] = sc.acc[k];
  return r;
}
}  // namespace

extern "C" {
// the maps start from +0.0: call after hs_water_begin / hs_wind_begin
void hc_reset_cells(void) { G_cells.assign((size_t)M.dimx * M.dimy * 3, 0.0); }
void hc_cell_budget(double* out3) { memcpy(out3, G_cells.data(), G_cells.size() * sizeof(double)); }
// hs_water_sweep / hs_wind_sweep in coop mode, with the maps
int hc_water_sweep(Stats* st, int split) {
  std::vector<int> next;
  for (int i : Wlive) {
    double acc[SM_BUDGET_SLOTS];
    const int r = step_cells<WaterP, WaterMidCoop>(W[i], split, water_move_coop<WarpHost, CoopWin<HostCellBack> >,
                                                   water_interact_coop<WarpHost, CoopWin<HostCellBack> >, acc);
    for (int k = 0; k < SM_BUDGET_SLOTS; k++) BUD[(size_t)i * SM_BUDGET_SLOTS + k] += acc[k];
    if (r == SM_EXIT_OOB) { st->exit_oob++; continue; }
    if (r == SM_EXIT_STALL) { st->exit_stall++; continue; }
    st->steps++;
    if (r == SM_EXIT_EVAP) { st->exit_evap++; continue; }
    next.push_back(i);
  }
  Wlive.swap(next); st->sweeps++;
  return (int)Wlive.size();
}
int hc_wind_sweep(Stats* st, int split) {
  std::vector<int> next;
  for (int i : Dlive) {
    double acc[SM_BUDGET_SLOTS];
    const int r = step_cells<WindP, WindMidCoop>(D[i], split, wind_move_coop<WarpHost, CoopWin<HostCellBack> >,
                                                 wind_interact_coop<WarpHost, CoopWin<HostCellBack> >, acc);
    for (int k = 0; k < SM_BUDGET_SLOTS; k++) BUD[(size_t)i * SM_BUDGET_SLOTS + k] += acc[k];
    if (r != SM_ALIVE) { st->exit_oob++; continue; }
    st->steps++;
    next.push_back(i);
  }
  Dlive.swap(next); st->sweeps++;
  return (int)Dlive.size();
}
}
