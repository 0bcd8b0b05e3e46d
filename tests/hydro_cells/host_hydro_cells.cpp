// tests/hydro_cells/host_hydro_cells.cpp -- tests/hostsim (compiled into this library unchanged) with the per-cell maps
// of the pooling hydrology's mass budget.  TEST TOOL ONLY.  HostHydroCellBack is hostsim's HostBack plus the 4-term map
// hook (kCellBudget, cell_budget), so hhc_water_flood / hhc_seep run the product's warp hydrology (sm_hydro_coop.cuh)
// with a HydroScratchBudget and the maps on, as the device's k_hydro_flood_w<true, true> / k_hydro_seep_w<true, true>
// do; the lanes are loops in the order hs_set_mode chose.
#include "../hostsim/hostsim.cpp"

namespace {
// SM_HYDRO_CELL_TERMS per cell, interleaved (eroded, deposited, cascade_net, water_net), cell order x*dimy + y
std::vector<double> G_hcells;
double G_hbud[SM_HYDRO_BUDGET_SLOTS] = {};   // the eleven sums of the last hhc_* call

struct HostHydroCellBack : HostBack {
  static constexpr bool kCellBudget = true;
  void cell_budget(int term, int x, int y, double d) {
    G_hcells[((size_t)x * M.dimy + y) * SM_HYDRO_CELL_TERMS + term] += d;
  }
};

void reset_hcells() { G_hcells.assign((size_t)M.dimx * M.dimy * SM_HYDRO_CELL_TERMS, 0.0); }
}  // namespace

extern "C" {
// hs_water_flood in coop mode, with the budget and the maps (both reset first)
void hhc_water_flood(HydroCount* out) {
  HydroCount hc{};
  reset_hcells();
  std::vector<char> live(W.size(), 0);
  for (int i : Wlive) live[i] = 1;
  WarpHost w; HostHydroCellBack b; CoopScratch sc; HydroScratchBudget hx{}; CoopWin<HostHydroCellBack> cw(b, &sc);
  for (size_t i = 0; i < W.size(); i++) if (!live[i]) hydro_flood_particle_coop(w, cw, &hx, W[i], hc);
  memcpy(G_hbud, hx.bud, sizeof(G_hbud));
  if (out) *out = hc;
}
// hs_seep in coop mode, with the budget and the maps.  mode 0: every cell in x-major order; mode 1: the flagged cells
// only, as the device
void hhc_seep(int mode, HydroCount* out) {
  HostAccess a; HydroCount hc{};
  reset_hcells();
  WarpHost w; HostHydroCellBack b; CoopScratch sc; HydroScratchBudget hx{}; CoopWin<HostHydroCellBack> cw(b, &sc);
  if (mode == 0) {
    for (int x = 0; x < M.dimx; x++) for (int y = 0; y < M.dimy; y++) hydro_seep_visit_coop(w, cw, &hx, x, y, hc);
  } else {
    ActiveMap am{};
    const unsigned long long cells = (unsigned long long)M.dimx * M.dimy;
    unsigned long long total = active_layout(cells, am.nwords, &am.nlevels);
    std::vector<unsigned long long> store(total, 0ull);
    unsigned long long off = 0;
    for (int l = 0; l < am.nlevels; l++) { am.lvl[l] = store.data() + off; off += am.nwords[l]; }
    am.ncells = cells;
    for (int x = 0; x < M.dimx; x++) for (int y = 0; y < M.dimy; y++) {
      bool airtop, holds;
      hydro_classify(a, x, y, airtop, holds);
      if (airtop) active_mark_block(am, x, y, M.dimx, M.dimy);
      if (holds) active_set(am, (unsigned long long)x * M.dimy + y);
    }
    G_act = &am;
    for (unsigned long long c = active_next(am, 0); c < cells; c = active_next(am, c + 1))
      hydro_seep_visit_coop(w, cw, &hx, (int)(c / M.dimy), (int)(c % M.dimy), hc);
    G_act = nullptr;
  }
  memcpy(G_hbud, hx.bud, sizeof(G_hbud));
  if (out) *out = hc;
}
void hhc_cell_budget(double* out4) { memcpy(out4, G_hcells.data(), G_hcells.size() * sizeof(double)); }
void hhc_hydro_budget(double* out11) { memcpy(out11, G_hbud, sizeof(G_hbud)); }
}
