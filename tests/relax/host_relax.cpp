// tests/relax/host_relax.cpp -- the slope relaxation's per-visit logic (soilmachine_b200/csrc/sm_relax.cuh) compiled
// for the host, driven the way sm_relax drives k_relax_phase.  TEST TOOL ONLY.
//
// hrelax_run   up to max_passes passes over a top / pool image with the device's pool discipline: phase launch j of
//              the call frees into ring[j & 1] and pops ring[(j & 1) ^ 1] first, then the bump counter up to pool_cap.
//              The cells of a phase run in a chosen order (0 x-major, 1 reversed, 2 shuffled); `period` and `radius`
//              override P and the marking radius R for the negative controls (period 0, radius -1: the real ones).
#include <stdint.h>
#include <algorithm>
#include <random>
#include <vector>
#include "../../soilmachine_b200/csrc/sm_relax.cuh"

namespace {
struct HostRelax {
  int dx, dy, sc;
  const SoilDev* soils;
  Sec32* top;
  Sec32* pool;
  int64_t cap, bump;
  std::vector<uint32_t> ring[2];
  size_t head[2] = {0, 0};
  unsigned int phase = 0;
  std::vector<uint32_t> stale;
  RelaxState rs;
  int64_t allocs = 0;
  int dimx() const { return dx; }
  int dimy() const { return dy; }
  int scale() const { return sc; }
  SoilDev soil(uint32_t t) const { return soils[t]; }
  Sec32* rec(int x, int y) { return &top[(size_t)x * dy + y]; }
  void query(int x, int y, double& h, uint32_t& t) { const Sec32* r = rec(x, y); h = rec_height(*r); t = rec_surface(*r); }
  void cascade_prefetch(int, int) {}
  void mark(int) {}
  void note_transfer() { rs.pending = true; }
  void focus(int x, int y) { relax_focus(*this, x, y); }
  void dirty_rec(Sec32* r, int x, int y) { relax_dirty(*this, *r, x, y); }
  Sec32 pool_load(uint32_t i) { return pool[i]; }
  void pool_store(uint32_t i, const Sec32& r) { pool[i] = r; }
  uint32_t pool_alloc() {
    allocs++;
    std::vector<uint32_t>& R = ring[phase ^ 1u];
    size_t& h = head[phase ^ 1u];
    if (h < R.size()) return R[h++];
    if (bump < cap) return (uint32_t)bump++;
    rs.drops++;
    return SM_NIL;
  }
  void pool_free(uint32_t i) { ring[phase].push_back(i); }
  uint32_t* stale_word(int x, int y, uint32_t& bit) {
    const size_t i = (size_t)x * dy + y;
    bit = 1u << (i & 31);
    return &stale[i >> 5];
  }
  uint32_t stale_peek(const uint32_t* w) { return *w; }
  void stale_set(uint32_t* w, uint32_t m) { *w |= m; }
  void stale_clear(uint32_t* w, uint32_t b) { *w &= ~b; }
};
}  // namespace

extern "C" {
// 0: done; 3: a section was dropped (the call finished that phase and stopped).  The free rings start with ring1
// (what the device pops first); stats: passes, stable, visits, transfers, pool drops, changed columns, pool_alloc calls; pass_changes[k]:
// the columns pass k + 1 changed.
int hrelax_run(int dimx, int dimy, int scale, const SoilDev* soils, Sec32* top, Sec32* pool, int64_t pool_cap,
               int64_t* bump, const uint32_t* ring1, int64_t nring1, int max_passes, int transferloop, int order,
               uint64_t seed, int period, int radius, int64_t* stats, int64_t* pass_changes) {
  HostRelax a{dimx, dimy, scale, soils, top, pool, pool_cap, *bump};
  a.ring[1].assign(ring1, ring1 + nring1);
  a.stale.assign(((size_t)dimx * dimy + 31) / 32, 0xFFFFFFFFu);
  relax_state_init(a.rs, transferloop);
  if (radius >= 0) a.rs.radius = radius;
  const int P = period > 0 ? period : relax_period(transferloop);
  std::mt19937_64 rng(seed);
  std::vector<int64_t> cells;
  int64_t visits = 0, passes = 0, stable = 0;
  unsigned int j = 0;
  for (int pass = 1; pass <= max_passes && !a.rs.drops; pass++) {
    const unsigned long long before = a.rs.changes;
    for (int p = 0; p < P * P && !a.rs.drops; p++, j++) {
      // launch j: its frees go to ring[j & 1]; ring[(j & 1) ^ 1] is popped from its head, the entries it has left
      // are served first (the device's rings are FIFOs)
      a.phase = j & 1u;
      a.ring[a.phase].erase(a.ring[a.phase].begin(), a.ring[a.phase].begin() + (long)a.head[a.phase]);
      a.head[a.phase] = 0;
      cells.clear();
      for (int x = p / P; x < dimx; x += P)
        for (int y = p % P; y < dimy; y += P) cells.push_back((int64_t)x * dimy + y);
      if (order == 1) std::reverse(cells.begin(), cells.end());
      if (order == 2) std::shuffle(cells.begin(), cells.end(), rng);
      for (int64_t c : cells) visits += relax_visit(a, (int)(c / dimy), (int)(c % dimy), transferloop);
    }
    passes = pass;
    pass_changes[pass - 1] = (int64_t)(a.rs.changes - before);
    stable = a.rs.changes == before;
    if (stable) break;
  }
  *bump = a.bump;
  stats[0] = passes; stats[1] = stable; stats[2] = visits; stats[3] = (int64_t)a.rs.transfers;
  stats[4] = (int64_t)a.rs.drops; stats[5] = (int64_t)a.rs.changes;
  stats[6] = a.allocs;
  return a.rs.drops ? 3 : 0;
}
}
