// tests/sharded_hydro/host_sharded.cpp -- tests/hostsim (compiled into this library unchanged) with the warp hydrology
// (sm_hydro_coop.cuh) run on a map cut into x-strips, the way a sharded context runs it.  TEST TOOL ONLY.
//
// StripBack routes as the device's HydroBack<MULTI = true> does: every strip has its own section pool, and pool
// loads, stores, allocations and frees go to the pool of the strip that owns the column the last focus() named; the
// frequency words of a cell are read and written in the copy of the strip that owns its column.  The slots of strip q
// are numbered q * kSlotBase + k, so a slot handed to the wrong strip is recognised: every pool access checks that the
// slot belongs to the focused strip and is allocated there, and counts a violation otherwise.  The copies of the
// frequency arrays hold NaN outside their own strip.  The batches themselves run on the one-pool map of hostsim; each
// hydrology call splits the map into the strips first and merges it back afterwards.
#include "../hostsim/hostsim.cpp"
#include <limits>

namespace {
const uint32_t kSlotBase = 1u << 24;
struct Strip {
  std::vector<Sec32> pool;
  std::vector<uint32_t> freelist;
  std::vector<char> used;
  std::vector<float> wfreq, wtrack;
};
std::vector<Strip> S;
int G_strip_w = 1;
long long G_viol = 0;          // pool accesses outside the focused column's strip
int G_ignore_focus = 0;        // negative control: focus() is ignored, allocations go to strip 0 and every access is
                               // checked against strip 0 (the check must then fire)

int strip_of(int x) {
  const int q = x / G_strip_w;
  return q < (int)S.size() ? q : (int)S.size() - 1;
}

struct StripBack {
  int cur_q = 0;
  static constexpr bool kBudget = true;
  static constexpr bool kHydroHooks = true;
  int dimx() const { return M.dimx; }
  int dimy() const { return M.dimy; }
  int scale() const { return M.scale; }
  const SoilDev* soilp(uint32_t t) const { return &M.soils[t]; }
  Sec32* cell_ptr(int x, int y) { return &M.top[(size_t)x * M.dimy + y]; }
  void focus(int x, int) { if (!G_ignore_focus) cur_q = strip_of(x); }
  // The slot's index in its strip's pool (strip i / kSlotBase), or -1 if no such slot is allocated.  A slot of any
  // strip but the focused one is a violation; it is still served from its own strip, so that the map stays whole.
  long slot(uint32_t i) {
    const uint32_t q = i / kSlotBase, k = i % kSlotBase;
    if (q != (uint32_t)cur_q) G_viol++;
    if (q >= S.size() || k >= S[q].pool.size() || !S[q].used[k]) { G_viol++; return -1; }
    return (long)k;
  }
  Sec32 pool_load(uint32_t i) {
    const long k = slot(i);
    if (k < 0) { Sec32 e; rec_set_empty(e); return e; }
    return S[i / kSlotBase].pool[k];
  }
  void pool_store(uint32_t i, const Sec32& r) {
    const long k = slot(i);
    if (k >= 0) S[i / kSlotBase].pool[k] = r;
  }
  uint32_t pool_alloc() {
    Strip& s = S[cur_q];
    uint32_t k;
    if (!s.freelist.empty()) { k = s.freelist.back(); s.freelist.pop_back(); }
    else { k = (uint32_t)s.pool.size(); s.pool.push_back(Sec32{}); s.used.push_back(0); }
    s.used[k] = 1;
    return (uint32_t)cur_q * kSlotBase + k;
  }
  void pool_free(uint32_t i) {
    const long k = slot(i);
    if (k < 0) return;
    S[i / kSlotBase].used[k] = 0;
    S[i / kSlotBase].freelist.push_back((uint32_t)k);
  }
  float wfreq(int i) const { return S[strip_of(i % M.dimx)].wfreq[i]; }
  float wtrack(int i) const { return S[strip_of(i % M.dimx)].wtrack[i]; }
  float windfreq(int i) const { return M.windfreq[i]; }
  void set_wtrack(int i, float v) { S[strip_of(i % M.dimx)].wtrack[i] = v; }
  void set_windfreq(int i, float v) { M.windfreq[i] = v; }
  void note_transfer() {}
  void air_mark(Sec32* r, int x, int y) { if (G_act && r->type == SM_AIR) active_mark_block(*G_act, x, y, M.dimx, M.dimy); }
  void wet_mark(int x, int y) { if (G_act) active_set(*G_act, (unsigned long long)x * M.dimy + y); }
  double volume_factor() const { return M.volume_factor; }
  void pspeed(float px, float py, double height, float* ps) const { wind_field_pspeed(G_field, px, py, height, ps); }
};

// hostsim's one pool -> one pool per strip (each column's sections move to its owner's pool, in column order)
void split(int nstrips) {
  S.assign(nstrips, Strip());
  G_strip_w = (M.dimx + nstrips - 1) / nstrips;
  const size_t cells = (size_t)M.dimx * M.dimy;
  const float nan = std::numeric_limits<float>::quiet_NaN();
  for (int q = 0; q < nstrips; q++) { S[q].wfreq.assign(cells, nan); S[q].wtrack.assign(cells, nan); }
  for (int x = 0; x < M.dimx; x++) {
    Strip& s = S[strip_of(x)];
    const uint32_t base = (uint32_t)strip_of(x) * kSlotBase;
    for (int y = 0; y < M.dimy; y++) {
      const size_t c = (size_t)y * M.dimx + x;
      s.wfreq[c] = M.wfreq[c];
      s.wtrack[c] = M.wtrack[c];
      Sec32& top = M.top[(size_t)x * M.dimy + y];
      if (top.type == SM_EMPTY || top.below == SM_NIL) continue;
      uint32_t src = top.below;
      top.below = base + (uint32_t)s.pool.size();
      for (;;) {                  // section k of the chain goes to slot k of the strip (pushed in chain order)
        const uint32_t k = (uint32_t)s.pool.size();
        s.pool.push_back(M.pool[src]);
        s.used.push_back(1);
        src = s.pool[k].below;
        if (src == SM_NIL) break;
        s.pool[k].below = base + k + 1;
      }
    }
  }
}
// and back: every column's sections into hostsim's pool again, the frequency words from their owners
void merge() {
  M.pool.clear();
  M.freelist.clear();
  for (int x = 0; x < M.dimx; x++) {
    const Strip& s = S[strip_of(x)];
    for (int y = 0; y < M.dimy; y++) {
      const size_t c = (size_t)y * M.dimx + x;
      M.wfreq[c] = s.wfreq[c];
      M.wtrack[c] = s.wtrack[c];
      Sec32& top = M.top[(size_t)x * M.dimy + y];
      if (top.type == SM_EMPTY || top.below == SM_NIL) continue;
      uint32_t src = top.below;
      top.below = (uint32_t)M.pool.size();
      for (size_t n = 0;; n++) {
        const uint32_t q = src / kSlotBase, k0 = src % kSlotBase;
        if (q != (uint32_t)strip_of(x)) G_viol++;   // a column's sections live in its owner's pool
        const uint32_t k = (uint32_t)M.pool.size();
        // (after a violation the chain may lead anywhere: stop at a slot that does not exist or after too many)
        const bool ok = q < S.size() && k0 < S[q].pool.size() && n < S[q].pool.size();
        if (!ok) G_viol++;
        M.pool.push_back(ok ? S[q].pool[k0] : Sec32{});
        src = M.pool[k].below;
        if (src == SM_NIL || !ok) { M.pool[k].below = SM_NIL; break; }
        M.pool[k].below = k + 1;
      }
    }
  }
}
}  // namespace

extern "C" {
// hs_water_flood in coop mode, on `nstrips` strips
void shs_water_flood(int nstrips, HydroCount* out) {
  HydroCount hc{};
  std::vector<char> live(W.size(), 0);
  for (int i : Wlive) live[i] = 1;
  split(nstrips);
  WarpHost w; StripBack b; CoopScratch sc; HydroScratchBudget hx{}; CoopWin<StripBack> cw(b, &sc);
  for (size_t i = 0; i < W.size(); i++) if (!live[i]) hydro_flood_particle_coop(w, cw, &hx, W[i], hc);
  merge();
  if (out) *out = hc;
}
// hs_seep in coop mode, on `nstrips` strips.  mode 0: every cell in x-major order; mode 1: the flagged cells only, the
// classification reading each column's sections from its owner's pool
void shs_seep(int nstrips, int mode, HydroCount* out) {
  HydroCount hc{};
  split(nstrips);
  WarpHost w; StripBack b; CoopScratch sc; HydroScratchBudget hx{}; CoopWin<StripBack> cw(b, &sc);
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
    cw.detach();                  // rec() hands out the records in place
    for (int x = 0; x < M.dimx; x++) for (int y = 0; y < M.dimy; y++) {
      bool airtop, holds;
      cw.focus(x, y);
      hydro_classify(cw, x, y, airtop, holds);
      if (airtop) active_mark_block(am, x, y, M.dimx, M.dimy);
      if (holds) active_set(am, (unsigned long long)x * M.dimy + y);
    }
    G_act = &am;
    for (unsigned long long c = active_next(am, 0); c < cells; c = active_next(am, c + 1))
      hydro_seep_visit_coop(w, cw, &hx, (int)(c / M.dimy), (int)(c % M.dimy), hc);
    G_act = nullptr;
  }
  merge();
  if (out) *out = hc;
}
// pool accesses outside the focused column's strip since the last call
long long shs_violations(void) { const long long v = G_viol; G_viol = 0; return v; }
void shs_ignore_focus(int on) { G_ignore_focus = on; }
}
