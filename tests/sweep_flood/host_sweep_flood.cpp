// tests/sweep_flood/host_sweep_flood.cpp -- tests/hostsim (compiled into this library unchanged) driven in the
// sweep-flood order of sm_water_run_flooding.  TEST TOOL ONLY.
//
// hssf_water_run_flooding  a water batch: after every sweep (hs_water_sweep) the particles that stopped in it flood,
//                          ascending index, on the warp executor (sm_hydro_coop.cuh, as k_hydro_flood_sweep); the
//                          counters add up over the call.  max_sweeps <= 0: until every particle is dead.
#include "../hostsim/hostsim.cpp"

extern "C" {
void hssf_water_run_flooding(int n, const float* xy, int max_sweeps, Stats* st, HydroCount* out) {
  memset(st, 0, sizeof(Stats));
  HydroCount hc{};
  hs_water_begin(n, xy);
  WarpHost w; HostBack b; CoopScratch sc; HydroScratch hx; CoopWin<HostBack> cw(b, &sc);
  while (!Wlive.empty() && (max_sweeps <= 0 || st->sweeps < max_sweeps)) {
    const std::vector<int> before = Wlive;
    hs_water_sweep(st);
    size_t k = 0;
    for (int i : before) {          // both lists ascend; the survivors are a subsequence of `before`
      if (k < Wlive.size() && Wlive[k] == i) { k++; continue; }
      hydro_flood_particle_coop(w, cw, &hx, W[i], hc);
    }
  }
  if (out) *out = hc;
}
}  // extern "C"
