// sm_coop.cuh -- one particle-step executed by ONE WARP (the hot path of the sweep kernel, sm_sweep.cuh).
//
// A particle-step is a chain of ~2 500 dependent instructions when one thread runs it (two 3x3 gathers, a
// normal, a bilinear sample, one or two cascades over eight neighbours each, the write-back).  The sweep is
// latency-bound - it waits for the slowest chain of dependent steps - so the step itself is what has to get
// shorter.  Here the 32 lanes of a warp share one particle:
//   * gathers / write-back: one record per lane, all in flight at once;
//   * the arithmetic that depends on the whole patch (normal, move, bilinear height, equilibrium) is computed
//     by every lane redundantly from the staged records - identical inputs, identical instructions, no
//     divergence and nothing to broadcast;
//   * the cascade evaluates its (up to) eight neighbours on eight lanes at once; the lowest-ranked neighbour
//     that would transfer is committed by one lane, then the remaining ones are evaluated again.  A
//     neighbour that does not transfer has no side effect, so this visits exactly the states the reference
//     loop visits (particle.h:62-99): ranks below the first acting one see the state they see sequentially,
//     the acting one commits, the later ones are re-evaluated on the new state;
//   * column mutations (remove / add, pool pushes and pops) are done by a single lane.
// The arithmetic is sm_core.cuh's (same expressions, same promotions); only the control structure differs.
//
// Everything is written against two policies so that the CPU test-suite can run the very same code:
//   W  warp policy     each(n, f): lanes 0..n-1 run f(lane)        ballot(n, f): bit l = f(l), l < n
//                      one(f): a single lane runs f                 lead(): the lane doing single-lane stores
//                      All of them are full-warp synchronisation points: what lanes wrote before is visible
//                      to every lane after.  Device: sm_sweep.cuh (WarpDev); host: tests/hostsim (loops).
//   A  accessor        CoopWin<B> below (B = backing store: device memory / host vectors).
// Inside each()/ballot() a lane may write only its own slots and read only what earlier phases wrote.
#pragma once
#include "sm_core.cuh"

#if defined(__CUDA_ARCH__)
#define SM_POPC(x) __popc((unsigned int)(x))
#else
#define SM_POPC(x) __builtin_popcount((unsigned int)(x))
#endif

#define SM_CW_SLOTS 18   // patch A = 3x3 around ipos (slots 0-8), patch B = 3x3 around npos (slots 9-17)
#define SM_CW_PLUS 186u   // (1<<1)|(1<<3)|(1<<4)|(1<<5)|(1<<7): the 5-point stencil inside a 3x3 block

// Mass budget (SURVEY.md A.7; the reference is not conservative, so "mass conservation" is a budget): six f64
// accumulators per particle, summed in step order, identical in the oracle port (oracle/sm_oracle.cpp).  Heights
// are column heights (floor + size of the top section) read right before and right after the column operation.
//   0 eroded        height taken off the map by a particle's erosion      (water.h:98-100, wind.h:109)
//   1 deposited     height put on the map by a particle's deposition      (water.h:109, wind.h:123-124)
//   2 cascade_net   (height gained by the lower cell + height lost by the higher cell) summed over the cascade
//                   transfers: zero but for the f64->f32 narrowing of `transfer` (particle.h:87-91) and rounding
//   3 discarded     water: sediment x volume the particle still held when it evaporated or left the map
//                   (water.h:65-69,118-119); wind: sediment it held when it died (wind.h:83-88)
//   4 clamped       water.h:117: (sediment - 1) x volume cut off by the clamp
//   5 wind_negative wind.h:107-110: negative suspension*force, i.e. sediment lowered without touching the map
// Budget identity: d(sum of heights) = deposited - eroded + cascade_net (+ rounding), checked by the tests.
#define SM_BUDGET_SLOTS 6

// Per-cell maps of the mass budget (SM_FLAG_CELL_BUDGET): terms 0 eroded, 1 deposited, 2 cascade_net, measured where
// slots 0-2 above are, but each delta is credited to the cell whose height was read (a cascade transfer credits the
// higher and the lower cell separately).  A backing that declares `static constexpr bool kCellBudget = true` gets
// cell_budget(term, x, y, delta) at every measurement point, called by the lane that mutates the column, in execution
// order; a backing without the member (the host emulation's HostBack, the hydrology's HydroBack<BUDGET>) compiles as
// before.  The hydrology's HydroBack<true, true> routes the same calls into its own 4-term map (sm_hydro_coop.cuh).
template <class B, class = void> struct CellBudgetOf { static constexpr bool value = false; };
template <class B> struct CellBudgetOf<B, decltype(void(B::kCellBudget))> { static constexpr bool value = B::kCellBudget; };

// per-warp scratch (shared memory on the device)
struct
#if defined(__CUDACC__)
    __align__(32)
#else
    alignas(32)
#endif
        CoopScratch {
  Sec32 win[SM_CW_SLOTS];     // staged top records; a cell inside both patches resolves to patch A
  double hs[2][8];            // cascade: initial neighbour heights, per nesting depth
  double d;                   // result of a single-lane column operation
  uint32_t u;
  unsigned char ord[2][8];    // cascade: ord[depth][rank] = neighbour index
  uint32_t pad_[3];
  double acc[SM_BUDGET_SLOTS]; // mass budget of the current step (single lane; only with B::kBudget)
  double pad2_[2];
};

// Prevailing wind of a WindParticle from a lattice velocity field (extension; upstream: the constant (-2, 0, 1),
// wind.h:29).  The lattice maps to the world as upstream's boundary construction does (SoilMachine.cpp:234-239 with
// lbmwind.h:119): lattice (x, y, z) <-> map cell (x*SIZEX/NX, z*SIZEY/NZ) at map height y*(SCALE/32)/SCALE.  A
// particle's `height` is in units of map height * SCALE/80 (wind.h:67).  Nearest lattice cell, clamped to the
// lattice; velocity / 0.05 (the lattice is driven with 0.05 * pspeed, lbm.cs:35) and each component clamped to
// the reference's magnitude (|x| <= 2, |y| <= 2, |z| <= 2), which keeps the conflict reach of a step valid.
struct WindField {
  const float* v4;          // 4 floats per lattice cell, cell = (x*ny + y)*nz + z; null = no field
  int nx, ny, nz;
  int dimx, dimy, scale;    // of the map
};
SM_HD void wind_field_pspeed(const WindField& f, float px, float py, double height, float* ps) {
  if (!f.v4) { ps[0] = -2.0f; ps[1] = 0.0f; ps[2] = 1.0f; return; }
  const float sx = (float)f.dimx / (float)f.nx, sy = (float)f.scale / 32.0f, sz = (float)f.dimy / (float)f.nz;
  int lx = (int)(px / sx), lz = (int)(py / sz);
  int ly = (int)((float)(height * 80.0 / (double)f.scale) * (float)f.scale / sy);
  lx = lx < 0 ? 0 : (lx > f.nx - 1 ? f.nx - 1 : lx);
  ly = ly < 0 ? 0 : (ly > f.ny - 1 ? f.ny - 1 : ly);
  lz = lz < 0 ? 0 : (lz > f.nz - 1 ? f.nz - 1 : lz);
  const float* v = f.v4 + (((size_t)lx * f.ny + ly) * f.nz + lz) * 4;
  for (int k = 0; k < 3; k++) {
    float c = v[k] / 0.05f;
    c = c < -2.0f ? -2.0f : (c > 2.0f ? 2.0f : c);
    ps[k] = c;
  }
}

// ------------------------------------------------------------------------------------------------
// the window accessor
// ------------------------------------------------------------------------------------------------
// B provides: dimx() dimy() scale(), soilp(t) -> const SoilDev*, cell_ptr(x, y) -> Sec32* (global record),
// focus(x, y), pool_load/pool_store/pool_alloc/pool_free, wfreq(ind) wtrack(ind) windfreq(ind),
// set_wtrack(ind, v) set_windfreq(ind, v), note_transfer(), pspeed(px, py, height, out3), kBudget, kHydroHooks
// (+ air_mark(rec, x, y), wet_mark(x, y), volume_factor() when kHydroHooks; + cell_budget(term, x, y, d) when it
// declares kCellBudget = true).
// ax..f_track are warp-uniform: every lane holds the same values and updates them identically.
template <class B> struct CoopWin {
  B& b;
  CoopScratch* s;
  int ax, ay, bx, by;
  uint32_t valid, dirtym;
  bool has_b;
  float f_freq, f_track;
  static constexpr bool kBudget = B::kBudget;
  static constexpr bool kCellBudget = CellBudgetOf<B>::value;
  SM_HD CoopWin(B& b_, CoopScratch* s_) : b(b_), s(s_), ax(0), ay(0), bx(0), by(0), valid(0), dirtym(0), has_b(false),
                                          f_freq(0.f), f_track(0.f) {}
  SM_HD int dimx() const { return b.dimx(); }
  SM_HD int dimy() const { return b.dimy(); }
  SM_HD int scale() const { return b.scale(); }
  SM_HD const SoilDev& soil(uint32_t t) const { return *b.soilp(t); }

  SM_HD int slot_of(int x, int y) const {
    int dx = x - ax + 1, dy = y - ay + 1;
    if ((unsigned)dx < 3u && (unsigned)dy < 3u) return dx * 3 + dy;
    if (has_b) {
      dx = x - bx + 1; dy = y - by + 1;
      if ((unsigned)dx < 3u && (unsigned)dy < 3u) return 9 + dx * 3 + dy;
    }
    return -1;
  }
  // stage the in-bounds cells of patch A that `want` names (bit k = cell k of the 3x3 block): one record per lane
  template <class W> SM_HD void fetch_a(W& w, uint32_t want) {
    const int nx_ = b.dimx(), ny_ = b.dimy();
    const uint32_t have = valid;
    const uint32_t got = w.ballot(9, [&](int k) {
      const int x = ax + k / 3 - 1, y = ay + k % 3 - 1;
      const bool need = ((want >> k) & 1u) && !((have >> k) & 1u) && x >= 0 && y >= 0 && x < nx_ && y < ny_;
      if (need) s->win[k] = *b.cell_ptr(x, y);
      return need;
    });
    valid |= got;
  }
  // `mask`: which cells of the 3x3 block around ipos to stage now.  The default stages all nine.  The exact-footprint
  // schedule stages only the plus-shaped stencil move() reads (SM_CW_PLUS): the corners may still be written by a
  // lower-index particle this one has not had to wait for yet, and are staged by target() after the second wait.
  template <class W> SM_HD void begin(W& w, int ix, int iy, int kind, uint32_t mask = 0x1FFu) {
    ax = ix; ay = iy; has_b = false; valid = 0; dirtym = 0;
    const int ind = iy * b.dimx() + ix;
    if (kind == 0) { f_freq = b.wfreq(ind); f_track = b.wtrack(ind); }
    else f_freq = b.windfreq(ind);
    fetch_a(w, mask);
  }
  // patch B = the 3x3 block around the new position: lanes 0-8 stage its cells that do not resolve to patch A,
  // lanes 9-17 the cells of patch A inside that block that are not staged yet
  template <class W> SM_HD void target(W& w, int nx, int ny) {
    bx = nx; by = ny; has_b = true;
    const int nx_ = b.dimx(), ny_ = b.dimy();
    const uint32_t have = valid;
    const uint32_t got = w.ballot(18, [&](int l) {
      if (l < 9) {
        const int x = nx + l / 3 - 1, y = ny + l % 3 - 1;
        bool need = x >= 0 && y >= 0 && x < nx_ && y < ny_;
        const int dx = x - ax + 1, dy = y - ay + 1;
        if ((unsigned)dx < 3u && (unsigned)dy < 3u) need = false;     // resolves to patch A
        if (need) s->win[9 + l] = *b.cell_ptr(x, y);
        return need;
      }
      const int k = l - 9;
      const int x = ax + k / 3 - 1, y = ay + k % 3 - 1;
      const int dx = x - nx + 1, dy = y - ny + 1;
      const bool need = !((have >> k) & 1u) && (unsigned)dx < 3u && (unsigned)dy < 3u && x >= 0 && y >= 0 && x < nx_ && y < ny_;
      if (need) s->win[k] = *b.cell_ptr(x, y);
      return need;
    });
    valid |= ((got & 0x1FFu) << 9) | (got >> 9);
  }
  // every cell a step touches inside the two blocks is staged before it is touched; anything else (only the nested
  // re-cascade of a wind step reaches it) is accessed in place
  SM_HD Sec32* rec(int x, int y) {
    const int sl = slot_of(x, y);
    return sl >= 0 ? &s->win[sl] : b.cell_ptr(x, y);
  }
  SM_HD double height(int x, int y) { return rec_height(*rec(x, y)); }
  SM_HD void dirty(int x, int y) {
    const int sl = slot_of(x, y);
    if (sl >= 0) dirtym |= 1u << sl;
  }
  SM_HD void dirty_rec(const Sec32* r) {
    const long off = (long)(r - s->win);
    if (off >= 0 && off < SM_CW_SLOTS) dirtym |= 1u << (int)off;
  }
  // a record was modified: window bookkeeping (every lane) + the backing's hook for Air-topped cells (one lane;
  // only the pooling-hydrology executor has one: it keeps the active-cell index of the seep pass up to date)
  template <class W> SM_HD void touched(W& w, Sec32* r, int x, int y) {
    dirty_rec(r);
    if (B::kHydroHooks && w.lead()) b.air_mark(r, x, y);
  }
  // no staged patches: rec() hands out the records in place (the hydrology frames work that way)
  SM_HD void detach() { ax = ay = bx = by = -(1 << 28); has_b = false; valid = 0; dirtym = 0; }
  // single-lane services of sm_hydro.cuh's sequential pieces (hydro_seep_cell)
  SM_HD void dirty_rec(Sec32* r, int x, int y) { dirty_rec(r); if (B::kHydroHooks) b.air_mark(r, x, y); }
  SM_HD void wet_mark(int x, int y) { if (B::kHydroHooks) b.wet_mark(x, y); }
  SM_HD double volume_factor() const { return b.volume_factor(); }
  // per-cell budget maps: add `d` to term `term` of cell (x, y) (single lane; nothing without kCellBudget)
  SM_HD void cell_budget(int term, int x, int y, double d) {
    if constexpr (kCellBudget) b.cell_budget(term, x, y, d);
  }
  // write the modified records back: one record per lane
  template <class W> SM_HD void flush(W& w) {
    const uint32_t m = dirtym;
    w.each(SM_CW_SLOTS, [&](int l) {
      if ((m >> l) & 1u) {
        const int ox = l < 9 ? ax : bx, oy = l < 9 ? ay : by, k = l < 9 ? l : l - 9;
        *b.cell_ptr(ox + k / 3 - 1, oy + k % 3 - 1) = s->win[l];
      }
    });
    dirtym = 0;
  }
  // single-lane services used by col_* (sm_core.cuh)
  SM_HD void focus(int x, int y) { b.focus(x, y); }
  SM_HD Sec32 pool_load(uint32_t i) { return b.pool_load(i); }
  SM_HD void pool_store(uint32_t i, const Sec32& r) { b.pool_store(i, r); }
  SM_HD uint32_t pool_alloc() { return b.pool_alloc(); }
  SM_HD void pool_free(uint32_t i) { b.pool_free(i); }
};

// ------------------------------------------------------------------------------------------------
// Particle::cascade, particle.h:24-101
// ------------------------------------------------------------------------------------------------
// One neighbour of the transfer loop (particle.h:62-88) on the CURRENT records: does it transfer, how much,
// which soil lands on the lower cell, and is the centre the higher cell.  No side effects.
template <class A>
SM_HD bool cascade_eval(A& a, const Sec32* pc, const Sec32* pn, int SCALE, float& transfer, uint32_t& cascades,
                        bool& centre_top) {
  const double dd = (rec_height(*pc) - rec_height(*pn)) * (float)SCALE;   // :66, before the division by 80
  const Sec32* const tr = (dd > 0) ? pc : pn;                             // :71-72 the higher cell
  const SoilDev& sp = a.soil(rec_surface(*tr));                           // :74-75
  // diff = (float)(dd / 80.0f).  |dd| < 80*maxdiff*(1 - 2^-20) already proves |diff| <= maxdiff (rounding is
  // monotone): no excess, and the IEEE double division is only paid near or above the threshold.
  if (fabs(dd) < 80.0 * (double)sp.maxdiff * (1.0 - 9.5367431640625e-07)) return false;
  const float diff = (float)(dd / 80.0f);
  if (diff == 0) return false;                                            // :68-69
  const float excess = fabsf(diff) - sp.maxdiff;                          // :78
  if (excess <= 0) return false;                                          // :79-80
  transfer = sp.settling * excess / 2.0f;                                 // :83
  const double tsize = (tr->type == SM_EMPTY) ? 0.0 : tr->size;
  if (transfer > tsize) transfer = (float)tsize;                          // :87-88 (f64 -> f32 narrowing)
  cascades = sp.cascades;
  centre_top = dd > 0;
  return true;
}

template <int DEPTH, class W, class A> struct CascadeCoop {
  static SM_HD void run(W& w, A& a, int cx, int cy, int transferloop) {
    const int dimx = a.dimx(), dimy = a.dimy();
    const int SCALE = a.scale();
    double* const hs = a.s->hs[DEPTH];
    unsigned char* const ord = a.s->ord[DEPTH];
    // neighbour k = 0..7 in the order of particle.h:30-39: offset (kk/3 - 1, kk%3 - 1), kk = k + (k >= 4).
    // in-bounds mask (particle.h:51-52), same for every lane
    const unsigned int inb = ((cx > 0 ? 0x07u : 0u) | 0x18u | (cx < dimx - 1 ? 0xE0u : 0u)) &
                             ((cy > 0 ? 0x29u : 0u) | 0x42u | (cy < dimy - 1 ? 0x94u : 0u));
    const int num = SM_POPC(inb);
    Sec32* const pc = a.rec(cx, cy);
    // lane k: the neighbour's height BEFORE any transfer (the sort key, particle.h:58-60) and whether it
    // would transfer on the current state
    const unsigned int active = w.ballot(8, [&](int k) {
      if (!((inb >> k) & 1u)) { hs[k] = -1.0e300; return false; }          // out of bounds sorts last
      const int kk = k + (k >= 4 ? 1 : 0);
      const Sec32* pn = a.rec(cx + kk / 3 - 1, cy + kk % 3 - 1);
      hs[k] = rec_height(*pn);
      float t; uint32_t cs; bool ct;
      return cascade_eval(a, pc, pn, SCALE, t, cs, ct);
    });
    if (active == 0) return;     // nothing changes until the first transfer, and nobody would make one
    // The reference sorts the in-bounds neighbours by height, highest first, with std::sort = stable
    // insertion sort on <= 8 elements; (height desc, k asc) is a total order, so
    // rank[k] = #{j > k : h[j] > h[k]} + #{j < k : not h[k] > h[j]} and the sorted sequence is unique.
    w.each(8, [&](int k) {
      const double hk = hs[k];
      int r = 0;
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const double hj = hs[j];
        r += (j > k) ? (hj > hk ? 1 : 0) : ((j < k) ? (hk > hj ? 0 : 1) : 0);
      }
      ord[r] = (unsigned char)k;
    });
    // first acting rank of the first round: the speculative mask seen through the ranks
    int f = -1;
#pragma unroll
    for (int r = 7; r >= 0; r--) if (r < num && ((active >> ord[r]) & 1u)) f = r;
    for (;;) {
      const int k = (int)ord[f];
      const int kk = k + (k >= 4 ? 1 : 0);
      const int nx = cx + kk / 3 - 1, ny = cy + kk % 3 - 1;
      Sec32* const pn = a.rec(nx, ny);
      w.one([&]() {
        float transfer = 0.f; uint32_t casc = 0; bool ctop = false;
        cascade_eval(a, pc, pn, SCALE, transfer, casc, ctop);               // acts, by construction
        Sec32* const tr = ctop ? pc : pn;
        Sec32* const br = ctop ? pn : pc;
        a.b.note_transfer();
        double ht0 = 0.0, hb0 = 0.0;
        if (A::kBudget) { ht0 = rec_height(*tr); hb0 = rec_height(*br); }
        a.focus(ctop ? cx : nx, ctop ? cy : ny);
        const bool re = col_remove(a, *tr, (double)transfer) != 0;          // :90-91
        a.focus(ctop ? nx : cx, ctop ? ny : cy);
        col_add(a, *br, (double)transfer, casc);                            // :92
        if (A::kBudget) {
          const double dt = rec_height(*tr) - ht0, db = rec_height(*br) - hb0;
          a.s->acc[2] += dt + db;
          a.cell_budget(2, ctop ? cx : nx, ctop ? cy : ny, dt);
          a.cell_budget(2, ctop ? nx : cx, ctop ? ny : cy, db);
        }
        a.s->u = re ? 1u : 0u;
      });
      a.touched(w, pc, cx, cy);
      a.touched(w, pn, nx, ny);
      if constexpr (DEPTH > 0) {
        const bool recascade = a.s->u != 0;
        if (recascade && transferloop > 0) {                                // :96-97
          --transferloop;
          CascadeCoop<DEPTH - 1, W, A>::run(w, a, nx, ny, transferloop);
        }
      }
      // every later rank is evaluated on the new state
      const int start = f + 1;
      const unsigned int act = w.ballot(num, [&](int r) {
        if (r < start) return false;
        const int k2 = (int)ord[r];
        const int kk2 = k2 + (k2 >= 4 ? 1 : 0);
        const Sec32* pn2 = a.rec(cx + kk2 / 3 - 1, cy + kk2 % 3 - 1);
        float t; uint32_t cs; bool ct;
        return cascade_eval(a, pc, pn2, SCALE, t, cs, ct);
      });
      if (act == 0) return;
      f = SM_FFS(act) - 1;
    }
  }
};

// ------------------------------------------------------------------------------------------------
// WaterParticle::move && interact, water.h:43-121
// ------------------------------------------------------------------------------------------------
// What move() hands to interact() of the same step (the friction-modified `param` copy of water.h:48-54 is only
// read for solubility and equrate afterwards).
struct WaterMidCoop {
  float freq, solubility, equrate;
  double evaprate;
  int ix, iy;
};
// WaterParticle::move, water.h:43-73.  `amask`: cells of the 3x3 block around ipos staged now (see CoopWin::begin).
template <class W, class A> SM_HD int water_move_coop(W& w, A& a, WaterP& p, WaterMidCoop& m, uint32_t amask = 0x1FFu) {
  const int dimx = a.dimx(), dimy = a.dimy();
  if (A::kBudget && w.lead()) { for (int k = 0; k < SM_BUDGET_SLOTS; k++) a.s->acc[k] = 0.0; }
  const int ix = (int)roundf(p.px), iy = (int)roundf(p.py);        // :45
  a.begin(w, ix, iy, 0, amask);
  const sm_f3 n = map_normal(a, ix, iy);                            // :46
  Sec32* const ir = a.rec(ix, iy);
  SoilDev param = a.soil(rec_surface(*ir));                         // :47-48
  double evaprate = 0.01;                                           // :49
  const int ind = iy * dimx + ix;
  if (w.lead()) a.b.set_wtrack(ind, (float)(a.f_track + p.volume)); // :50, 348-351
  const float freq = a.f_freq;
  param.friction = param.friction * (1.0f - freq);                  // :53
  evaprate = evaprate * (1.0f - 0.2f * freq);                       // :54
  m.freq = freq; m.solubility = param.solubility; m.equrate = param.equrate; m.evaprate = evaprate;
  m.ix = ix; m.iy = iy;
  {
    const float vx = n.x * param.friction, vz = n.z * param.friction;   // :56
    if (sqrtf(vx * vx + vz * vz) < 1E-5) return SM_EXIT_STALL;
  }
  {
    const float f = param.friction;                                 // :60 mix(n.xz, speed, friction)
    const float mx = n.x * (1.0f - f) + p.sx * f;
    const float my = n.z * (1.0f - f) + p.sy * f;
    const float inv = 1.0f / sqrtf(mx * mx + my * my);              // :61 sqrt(2)*normalize
    p.sx = host_nan(SM_SQRT2F * (mx * inv));                        // host_nan: sm_core.cuh
    p.sy = host_nan(SM_SQRT2F * (my * inv));
  }
  p.px = host_nan(p.px + p.sx);                                     // :62
  p.py = host_nan(p.py + p.sy);
  if (!(p.px >= 0.0f && p.py >= 0.0f) ||                            // :65-69
      !(p.px < (float)dimx - 1.0f && p.py < (float)dimy - 1.0f)) {
    if (A::kBudget && w.lead()) a.s->acc[3] += p.sediment * p.volume;
    p.volume = 0.0;
    return SM_EXIT_OOB;
  }
  return SM_ALIVE;
}
// WaterParticle::interact, water.h:75-121
template <class W, class A> SM_HD int water_interact_coop(W& w, A& a, WaterP& p, const WaterMidCoop& m) {
  const int SCALE = a.scale();
  const int ix = m.ix, iy = m.iy;
  const float freq = m.freq;
  const double evaprate = m.evaprate;
  Sec32* const ir = a.rec(ix, iy);
  const int nx = (int)roundf(p.px), ny = (int)roundf(p.py);
  a.target(w, nx, ny);
  double c_eq = m.solubility * (rec_height(*ir) - map_height_bilinear(a, p.px, p.py)) *
                (double)SCALE / 80.0;                               // :78
  if (c_eq < 0.0) c_eq = 0.0;
  if (c_eq > 1.0) c_eq = 1.0;
  if ((double)(a.soil(p.contains).erosionrate) < freq)              // :83-84
    p.contains = a.soil(p.contains).erodes;
  const double cdiff = c_eq - p.sediment;                           // :87
  if (cdiff > 0) {                                                  // :91-101
    p.sediment += m.equrate * cdiff;
    p.contains = a.soil(rec_surface(*ir)).transports;
    const double amount = m.equrate * cdiff * p.volume;
    w.one([&]() {
      const double h0 = A::kBudget ? rec_height(*ir) : 0.0;
      a.focus(ix, iy);
      double diff = col_remove(a, *ir, amount);
      SM_UNROLL1
      while (fabs(diff) > 1E-8) diff = col_remove(a, *ir, diff);
      if (A::kBudget) { const double d = h0 - rec_height(*ir); a.s->acc[0] += d; a.cell_budget(0, ix, iy, d); }
    });
    a.dirty_rec(ir);
  } else if (cdiff < 0) {                                           // :105-110
    const float eq = a.soil(p.contains).equrate;
    p.sediment += eq * cdiff;
    const double amount = -eq * cdiff * p.volume;
    const uint32_t what = p.contains;
    w.one([&]() {
      const double h0 = A::kBudget ? rec_height(*ir) : 0.0;
      a.focus(ix, iy);
      col_add(a, *ir, amount, what);
      if (A::kBudget) { const double d = rec_height(*ir) - h0; a.s->acc[1] += d; a.cell_budget(1, ix, iy, d); }
    });
    a.dirty_rec(ir);
  }
  CascadeCoop<0, W, A>::run(w, a, nx, ny, 0);                       // :113
  p.sediment /= (1.0 - evaprate);                                   // :116-119
  const double over = p.sediment - 1.0;
  if (p.sediment > 1.0) p.sediment = 1.0;
  p.volume *= (1.0 - evaprate);
  const bool lives = p.volume > 0.01;
  if (A::kBudget && w.lead()) {
    if (over > 0.0) a.s->acc[4] += over * p.volume;
    if (!lives) a.s->acc[3] += p.sediment * p.volume;
  }
  return lives ? SM_ALIVE : SM_EXIT_EVAP;
}
// one move() && interact()
template <class W, class A> SM_HD int water_step_coop(W& w, A& a, WaterP& p, uint32_t amask = 0x1FFu) {
  WaterMidCoop m;
  const int r = water_move_coop(w, a, p, m, amask);
  if (r != SM_ALIVE) return r;
  return water_interact_coop(w, a, p, m);
}

// ------------------------------------------------------------------------------------------------
// WindParticle::move && interact, wind.h:54-136
// ------------------------------------------------------------------------------------------------
// What WindParticle::move hands to interact() of the same step.
struct WindMidCoop {
  float suspension;      // param.suspension of the surface at ipos
  uint32_t transports;   // param.transports
  int ix, iy;
};
// WindParticle::move, wind.h:54-92.  `amask`: cells of the 3x3 block around ipos staged now (see CoopWin::begin).
template <class W, class A> SM_HD int wind_move_coop(W& w, A& a, WindP& p, WindMidCoop& m, uint32_t amask = 0x1FFu) {
  const int dimx = a.dimx(), dimy = a.dimy();
  const int SCALE = a.scale();
  if (A::kBudget && w.lead()) { for (int k = 0; k < SM_BUDGET_SLOTS; k++) a.s->acc[k] = 0.0; }
  // ---- move ----
  if (a.soil(p.contains).suspension == 0.0) return SM_EXIT_OOB;     // :56-57
  const int ix = (int)roundf(p.px), iy = (int)roundf(p.py);         // :60
  a.begin(w, ix, iy, 1, amask);
  const sm_f3 n = map_normal(a, ix, iy);                            // :61
  Sec32* const ir = a.rec(ix, iy);
  const SoilDev& param = a.soil(rec_surface(*ir));                  // :62-63
  m.suspension = param.suspension; m.transports = param.transports; m.ix = ix; m.iy = iy;
  if (w.lead()) a.b.set_windfreq(iy * dimx + ix, (float)(0.5 * a.f_freq + 0.5f));   // :64, 49-52
  const double sheight = rec_height(*ir) * (float)SCALE / 80.0f;    // :67
  if (p.height < sheight) p.height = sheight;                       // :68-70
  if (p.height > sheight) {                                         // :73-74
    p.sy = (float)(p.sy - 0.25);
  } else {                                                          // :76 mix(speed, cross(cross(speed,n),n), 0.8)
    const sm_f3 s{p.sx, p.sy, p.sz};
    const sm_f3 v = f3_cross(f3_cross(s, n), n);
    const double wt = 0.8;
    p.sx = (float)((double)s.x * (1.0 - wt) + (double)v.x * wt);
    p.sy = (float)((double)s.y * (1.0 - wt) + (double)v.y * wt);
    p.sz = (float)((double)s.z * (1.0 - wt) + (double)v.z * wt);
  }
  {                                                                 // :78 mix(speed, pspeed, 0.2)
    // pspeed is the constant (-2, 0, 1) upstream (wind.h:29); with a wind field attached (sm_wind_use_lbm,
    // a modelling extension that is off by default) it is sampled from the lattice Boltzmann velocity
    float ps[3];
    a.b.pspeed(p.px, p.py, p.height, ps);
    const double wt = 0.2;
    p.sx = (float)((double)p.sx * (1.0 - wt) + (double)(ps[0]) * wt);
    p.sy = (float)((double)p.sy * (1.0 - wt) + (double)(ps[1]) * wt);
    p.sz = (float)((double)p.sz * (1.0 - wt) + (double)(ps[2]) * wt);
  }
  p.px += p.sx;                                                     // :79
  p.py += p.sz;
  p.height += p.sy;                                                 // :80
  if (!(p.px >= 0.0f && p.py >= 0.0f) ||                            // :83-85
      !((int)p.px < dimx - 1 && (int)p.py < dimy - 1) ||
      sqrtf(p.sx * p.sx + p.sy * p.sy + p.sz * p.sz) < 0.01) {      // :87-88
    if (A::kBudget && w.lead()) a.s->acc[3] += p.sediment;
    return SM_EXIT_OOB;
  }
  return SM_ALIVE;
}
// WindParticle::interact, wind.h:94-136 (always returns true upstream)
template <class W, class A> SM_HD int wind_interact_coop(W& w, A& a, WindP& p, const WindMidCoop& m) {
  const int SCALE = a.scale();
  const int ix = m.ix, iy = m.iy;
  const float suspension = m.suspension;
  const uint32_t transports = m.transports;
  a.fetch_a(w, 0x1FFu);                                             // the cascade around ipos needs the whole block
  Sec32* const ir = a.rec(ix, iy);
  const int nx = (int)roundf(p.px), ny = (int)roundf(p.py);         // :99
  a.target(w, nx, ny);
  int ncascade = 0;
  if (p.height <= map_height_bilinear(a, p.px, p.py) * (float)SCALE / 80.0f) {   // :102
    if (transports == p.contains) {                                 // :105
      const float len = sqrtf(p.sx * p.sx + p.sy * p.sy + p.sz * p.sz);
      const double force = len * (a.height(nx, ny) - p.height) * (float)SCALE / 80.0f *
                           (1.0f - p.sediment);                     // :107
      const double amount = suspension * force;
      w.one([&]() {
        const double h0 = A::kBudget ? rec_height(*ir) : 0.0;
        a.focus(ix, iy);
        a.s->d = col_remove(a, *ir, amount);                        // :109
        if (A::kBudget) {
          const double d = h0 - rec_height(*ir);
          a.s->acc[0] += d;
          a.cell_budget(0, ix, iy, d);
          if (amount < 0.0) a.s->acc[5] += amount;
        }
      });
      a.dirty_rec(ir);
      p.sediment += (amount - a.s->d);                              // :110
      ncascade = 1;                                                 // :112 cascade(ipos, 1)
    }
  } else if (suspension > 0.0) {                                    // :119
    const float sc = a.soil(p.contains).suspension;
    p.sediment -= sc * p.sediment;                                  // :121
    const double amount = 0.5f * sc * p.sediment;
    const uint32_t what = p.contains;
    Sec32* const nr = a.rec(nx, ny);
    w.one([&]() {
      double h0 = A::kBudget ? rec_height(*nr) : 0.0;
      a.focus(nx, ny);
      col_add(a, *nr, amount, what);                                // :123
      if (A::kBudget) {
        const double d = rec_height(*nr) - h0;
        a.s->acc[1] += d;
        a.cell_budget(1, nx, ny, d);
        h0 = rec_height(*ir);
      }
      a.focus(ix, iy);
      col_add(a, *ir, amount, what);                                // :124
      if (A::kBudget) { const double d = rec_height(*ir) - h0; a.s->acc[1] += d; a.cell_budget(1, ix, iy, d); }
    });
    a.dirty_rec(nr);
    a.dirty_rec(ir);
    ncascade = 2;                                                   // :126,129 cascade(ipos,1); cascade(npos,1)
  }
  SM_UNROLL1
  for (int q = 0; q < ncascade; q++)                                // one call site for both
    CascadeCoop<1, W, A>::run(w, a, q == 0 ? ix : nx, q == 0 ? iy : ny, 1);
  return SM_ALIVE;
}
// one move() && interact()
template <class W, class A> SM_HD int wind_step_coop(W& w, A& a, WindP& p, uint32_t amask = 0x1FFu) {
  WindMidCoop m;
  const int r = wind_move_coop(w, a, p, m, amask);
  if (r != SM_ALIVE) return r;
  return wind_interact_coop(w, a, p, m);
}
