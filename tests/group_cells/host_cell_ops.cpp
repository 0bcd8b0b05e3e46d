// tests/group_cells/host_cell_ops.cpp -- tests/sharded_hydro (compiled into this library unchanged, and with it
// tests/hostsim) plus the warp form of the single-cell calls that change the map (sm_cell_coop.cuh: what
// k_cell_op_w runs on the device), on a map cut into x-strips.  TEST TOOL ONLY.
//
// shc_cell_op runs one call through StripBack: one pool per strip, every pool access checked against the owner of
// the focused column (shs_violations).  nstrips = 0 runs the same warp code on hostsim's one-pool map.
// shc_cell_op_seq is the one-thread form k_cell_op runs (sm_core.cuh / sm_hydro.cuh), the statement both are checked
// against.
#include "../sharded_hydro/host_sharded.cpp"
#include "../../soilmachine_b200/csrc/sm_cell_coop.cuh"

extern "C" {
double shc_cell_op(int nstrips, int op, int x, int y, float fx, float fy, double v, int t) {
  HydroCount hc{};
  WarpHost w; CoopScratch sc{}; CellCascadeScratch deep{}; HydroScratchBudget hx{};
  double d;
  if (nstrips > 0) {
    split(nstrips);
    StripBack b;
    d = cell_op_coop(w, b, &sc, &deep, &hx, op, x, y, fx, fy, v, t, hc);
    merge();
  } else {
    HostBack b;
    d = cell_op_coop(w, b, &sc, &deep, &hx, op, x, y, fx, fy, v, t, hc);
  }
  return d;
}
double shc_cell_op_seq(int op, int x, int y, float fx, float fy, double v, int t) {
  HostAccess a;
  double d = 0.0;
  if (op == 0) col_add(a, *a.rec(x, y), v, (uint32_t)t);
  else if (op == 1) d = col_remove(a, *a.rec(x, y), v);
  else if (op == 2) Cascade<3, HostAccess>::run(a, (int)roundf(fx), (int)roundf(fy), t);
  else if (op == 5) hydro_seep_cell(a, x, y);
  else if (op == 6) {
    HydroCount hc{};
    WFrame st[SM_WSTACK];
    int sp = 0;
    hydro_push(a, st, sp, x, y, t, hc);
    hydro_drain(a, st, sp, hc);
  }
  return d;
}
}
