// tests/hydro_budget/host_budget.cpp -- tests/hostsim (compiled into this library unchanged) with the warp hydrology's
// mass budget.  TEST TOOL ONLY.  hs_water_flood / hs_seep in coop mode run sm_hydro_coop.cuh with a HydroScratch,
// which keeps no budget; hsb_water_flood / hsb_seep are the same calls with a HydroScratchBudget - the scratch of the
// device's budget kernels (k_hydro_flood_w<true>, k_hydro_seep_w<true>) - and keep its eleven sums.
#include "../hostsim/hostsim.cpp"

namespace {
double G_hbud[SM_HYDRO_BUDGET_SLOTS] = {};   // mass budget of the last hsb_* call
}

extern "C" {
// hs_water_flood in coop mode, with the budget
void hsb_water_flood(HydroCount* out) {
  HydroCount hc{};
  std::vector<char> live(W.size(), 0);
  for (int i : Wlive) live[i] = 1;
  WarpHost w; HostBack b; CoopScratch sc; HydroScratchBudget hx{}; CoopWin<HostBack> cw(b, &sc);
  for (size_t i = 0; i < W.size(); i++) if (!live[i]) hydro_flood_particle_coop(w, cw, &hx, W[i], hc);
  memcpy(G_hbud, hx.bud, sizeof(G_hbud));
  if (out) *out = hc;
}
// hs_seep in coop mode, with the budget.  mode 0: every cell in x-major order; mode 1: the flagged cells only
void hsb_seep(int mode, HydroCount* out) {
  HostAccess a; HydroCount hc{};
  WarpHost w; HostBack b; CoopScratch sc; HydroScratchBudget hx{}; CoopWin<HostBack> cw(b, &sc);
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
void hsb_hydro_budget(double* out11) { memcpy(out11, G_hbud, sizeof(G_hbud)); }
}
