// oracle/_ref/libsmref_flooding.so -- libsmref.so (harness.cpp, included whole) plus the SWEEP-FLOOD driver.
//
// TEST INFRASTRUCTURE, like harness.cpp.  A separate library, so that libsmref.so, which every other reference test
// loads, stays exactly what it was.  The driver calls the reference's own move() / interact() / flood() in this order:
//   1. sweep s: every live particle, ascending index, does move() && interact()   (smref_water_sweep)
//   2. every particle that stopped in sweep s, ascending index, calls flood() (water.h:123-145); flood() applies its
//      own guard (volume >= minvol, spill left) and runs its water-table cascade and nested particles to completion
//   3. sweep s+1 meets the ponds of step 2.
// smref_water_flood cannot be called per sweep: it floods every dead particle, and flood() decrements spill on every
// call, so particles that stopped in earlier sweeps would flood again.
#include "harness.cpp"

extern "C" {

// Returns the number of flood() calls that passed the guard.  max_sweeps <= 0: until every particle is dead.
int64_t smref_water_sweep_flood(int n, const float* xy, int max_sweeps, Stats* st) {
  memset(st, 0, sizeof(Stats));
  smref_water_begin(n, xy);
  int64_t floods = 0;
  double t0 = now();
  while (!g.water_live.empty() && (max_sweeps <= 0 || st->sweeps < max_sweeps)) {
    const vector<int> before = g.water_live;
    smref_water_sweep(st);
    size_t k = 0;
    for (int i : before) {        // both lists ascend; the survivors are a subsequence of `before`
      if (k < g.water_live.size() && g.water_live[k] == i) { k++; continue; }
      WaterParticle& p = *g.water[i];
      if (!(p.volume < p.minvol) && p.spill > 0) floods++;
      p.flood(*g.lmap, *g.vp);
    }
  }
  st->seconds = now() - t0;
  return floods;
}

}  // extern "C"
