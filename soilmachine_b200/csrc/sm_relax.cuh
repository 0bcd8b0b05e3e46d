// sm_relax.cuh -- slope relaxation over the whole map (sm_relax, DESIGN.md section 12): the per-visit logic and the
// accessors the phase kernels hand to it.
//
// A pass calls the reference's Particle::cascade(vec2(x, y), map, vp, transferloop) (particle.h:24-101, Cascade<3>) at
// every cell in a fixed phase order: with R = 1 + transferloop and P = 2R + 1, phase p = (px, py) = (p / P, p % P) for
// p = 0 .. P*P-1, inside a phase x-major over x = px, px + P, ... and y = py, py + P, ...  A cascade at c reads and
// writes only columns within Chebyshev distance R of c, and two cells of one phase are at least P apart, so the cells of
// a phase commute exactly and run all at once.
//
// Skipped visits: every cell has a stale bit, all set when the call begins.  A visit clears its own bit before it runs;
// every column it really changes (its top record's bytes differ before and after) sets the stale bits of all cells
// within R of that column, its own cell's included.  A visit at a cell whose bit is clear would read exactly what its
// previous visit read and left, so it would change nothing: it is skipped.  The marks of one phase fall on cells of
// other phases (and on the visiting cell itself), never on another cell of the same phase.
//
// Everything outside the __CUDACC__ block is SM_HD, so that the host compiles it as a test tool
// (tests/relax/host_relax.cpp).  An accessor A of sm_core.cuh used here also has a RelaxState `rs`, and
//   uint32_t* stale_word(x, y, uint32_t& bit)   the word of the owner's stale bitmap holding cell (x, y)'s bit
//   uint32_t stale_peek(const uint32_t* w)      read a word
//   void stale_set(uint32_t* w, uint32_t mask)  w |= mask (concurrently with other visits of the phase)
//   void stale_clear(uint32_t* w, uint32_t bit) w &= ~bit
// Its focus(x, y) calls relax_focus, its dirty_rec relax_dirty, its note_transfer sets rs.pending and its pool_alloc
// counts the sections it could not serve in rs.drops.
#pragma once
#include <string.h>
#include "sm_core.cuh"

SM_HD int relax_radius(int transferloop) { return 1 + transferloop; }
SM_HD int relax_period(int transferloop) { return 2 * relax_radius(transferloop) + 1; }
// the first x >= lo with x % P == px
SM_HD int relax_first(int lo, int px, int P) { return lo + ((px - lo % P) + P) % P; }

// what one thread's visits did
struct RelaxState {
  Sec32 before;                   // the record focus() saw
  int radius;                     // R
  bool pending;                   // a transfer began and has not changed a column yet
  unsigned long long changes, transfers, drops;
};
SM_HD void relax_state_init(RelaxState& s, int transferloop) {
  s.radius = relax_radius(transferloop);
  s.pending = false;
  s.changes = s.transfers = s.drops = 0;
}

SM_HD bool rec_same(const Sec32& a, const Sec32& b) {
  uint64_t u[4], v[4];
  memcpy(u, &a, sizeof(u));
  memcpy(v, &b, sizeof(v));
  return u[0] == v[0] && u[1] == v[1] && u[2] == v[2] && u[3] == v[3];
}

// the stale bits of the cells (x, y0 .. y1) of one column; they are consecutive in the owner's bitmap
template <class A> SM_HD void relax_mark_run(A& a, int x, int y0, int y1) {
  uint32_t bit;
  uint32_t* w = a.stale_word(x, y0, bit);
  int lo = SM_FFS(bit) - 1;
  int n = y1 - y0 + 1;
  while (n > 0) {
    const int k = (32 - lo < n) ? 32 - lo : n;
    const uint32_t m = (k == 32 ? 0xFFFFFFFFu : ((1u << k) - 1u)) << lo;
    a.stale_set(w, m);
    n -= k;
    lo = 0;
    w++;
  }
}
// a column changed: every cell within R of it is stale
template <class A> SM_HD void relax_mark(A& a, int x, int y) {
  const int R = a.rs.radius;
  const int xa = x - R < 0 ? 0 : x - R, xb = x + R > a.dimx() - 1 ? a.dimx() - 1 : x + R;
  const int ya = y - R < 0 ? 0 : y - R, yb = y + R > a.dimy() - 1 ? a.dimy() - 1 : y + R;
  for (int xx = xa; xx <= xb; xx++) relax_mark_run(a, xx, ya, yb);
}

// focus(x, y): the column the next col_* call changes; keep its top record
template <class A> SM_HD void relax_focus(A& a, int x, int y) { a.rs.before = *a.rec(x, y); }
// dirty_rec after that call: a column whose top record's bytes are unchanged did not change (settling == 0 gives
// remove(..., 0) and add(0); col_add ignores size <= 0)
template <class A> SM_HD void relax_dirty(A& a, const Sec32& r, int x, int y) {
  if (rec_same(r, a.rs.before)) return;
  a.rs.changes++;
  if (a.rs.pending) { a.rs.transfers++; a.rs.pending = false; }
  relax_mark(a, x, y);
}

// One visit of cell (x, y): Particle::cascade(vec2(x, y), map, vp, transferloop) when the cell is stale.  Returns
// whether it ran.
template <class A> SM_HD bool relax_visit(A& a, int x, int y, int transferloop) {
  uint32_t bit;
  uint32_t* w = a.stale_word(x, y, bit);
  if (!(a.stale_peek(w) & bit)) return false;
  a.stale_clear(w, bit);
  Cascade<3, A>::run(a, x, y, transferloop);
  return true;
}

#if defined(__CUDACC__)
#include "sm_device.cuh"

// The stale bitmaps and counter blocks of every rank (index 0 on a plain context), a trailing kernel parameter so that
// DevCtx and PeerPtrs keep their layout.  Bit (x - x0)*dimy + y of rank q's bitmap is the cell (x, y) of its strip.
// cnt[q]: visits, changed columns, transfers, pool drops, stop flag; the counts add up over the call.
#define SM_RELAX_CNT 5
struct RelaxMaps {
  uint32_t* stale[SM_MAX_RANKS];
  unsigned long long* cnt[SM_MAX_RANKS];
};

// One context: DevAccess's records and pool, with change detection and the stale bitmap.
struct RelaxDev : DevAccess {
  const RelaxMaps& m;
  RelaxState rs;
  __device__ __forceinline__ RelaxDev(const DevCtx& ctx, const SoilDev* ss, unsigned int ph, const RelaxMaps& maps,
                                      int transferloop)
      : DevAccess(ctx, ss, ph), m(maps) { relax_state_init(rs, transferloop); }
  __device__ __forceinline__ void focus(int x, int y) { relax_focus(*this, x, y); }
  __device__ __forceinline__ void dirty_rec(Sec32* r, int x, int y) { relax_dirty(*this, *r, x, y); }
  __device__ __forceinline__ void note_transfer() { rs.pending = true; }
  __device__ __forceinline__ uint32_t pool_alloc() {
    const uint32_t s = DevAccess::pool_alloc();
    rs.drops += s == SM_NIL;
    return s;
  }
  __device__ __forceinline__ uint32_t* stale_word(int x, int y, uint32_t& bit) {
    const size_t i = (size_t)x * c.dimy + y;
    bit = 1u << (i & 31);
    return m.stale[0] + (i >> 5);
  }
  __device__ __forceinline__ uint32_t stale_peek(const uint32_t* w) { return *w; }
  __device__ __forceinline__ void stale_set(uint32_t* w, uint32_t mask) { atomicOr(w, mask); }
  __device__ __forceinline__ void stale_clear(uint32_t* w, uint32_t bit) { atomicAnd(w, ~bit); }
};

// A map sharded in one process (a group): one thread per visit, every record read and written at the column's owner
// through cell_ptr<true>, pool loads, stores, allocations and frees at the owner focus() named (WinAccess<.., true>'s
// owner-pool logic), stale bits in the owner's bitmap.  No shared-memory window: rec() is the owner's record itself.
struct RelaxMulti : WinAccess<0, true> {
  typedef WinAccess<0, true> Base;
  const RelaxMaps& m;
  RelaxState rs;
  __device__ __forceinline__ RelaxMulti(const DevCtx& ctx, const SoilDev* ss, unsigned int ph, const RelaxMaps& maps,
                                        int transferloop)
      : Base(ctx, ss, ph, nullptr), m(maps) { relax_state_init(rs, transferloop); }
  __device__ __forceinline__ Sec32* rec(int x, int y) { return cell_ptr<true>(c, x, y); }
  __device__ __forceinline__ double height(int x, int y) { return rec_height(*rec(x, y)); }
  __device__ __forceinline__ uint32_t surface_of(int x, int y) { return rec_surface(*rec(x, y)); }
  __device__ __forceinline__ void query(int x, int y, double& h, uint32_t& t) {
    const Sec32* r = rec(x, y);
    h = rec_height(*r);
    t = rec_surface(*r);
  }
  __device__ __forceinline__ void cascade_prefetch(int, int) {}
  __device__ __forceinline__ void focus(int x, int y) { Base::focus(x, y); relax_focus(*this, x, y); }
  __device__ __forceinline__ void dirty_rec(Sec32* r, int x, int y) { relax_dirty(*this, *r, x, y); }
  __device__ __forceinline__ void note_transfer() { rs.pending = true; }
  __device__ __forceinline__ uint32_t pool_alloc() {
    const uint32_t s = Base::pool_alloc();
    rs.drops += s == SM_NIL;
    return s;
  }
  __device__ __forceinline__ uint32_t* stale_word(int x, int y, uint32_t& bit) {
    const int q = owner_of_x<true>(c, x);
    const size_t i = (size_t)(x - q * c.strip_w) * c.dimy + y;
    bit = 1u << (i & 31);
    return m.stale[q] + (i >> 5);
  }
  __device__ __forceinline__ uint32_t stale_peek(const uint32_t* w) { return *w; }
  __device__ __forceinline__ void stale_set(uint32_t* w, uint32_t mask) { atomicOr_system(w, mask); }
  __device__ __forceinline__ void stale_clear(uint32_t* w, uint32_t bit) { atomicAnd_system(w, ~bit); }
};
#endif
