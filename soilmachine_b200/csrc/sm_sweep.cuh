// sm_sweep.cuh -- k_sweep<KIND, MULTI>: the persistent sweep kernel with ONE WARP PER PARTICLE.
//
// Same contract as before (one cooperative launch per batch, one grid barrier per sweep, every live particle
// executes move() && interact() once per sweep, overlapping steps ordered by ascending particle index, results
// bit-identical to the reference driven in lockstep), different mapping: a particle owns a whole warp for the
// duration of its step and the step itself is lane-parallel (sm_coop.cuh).  What that buys:
//   * the dependent chain of one step is several times shorter (gathers, cascade evaluation and write-back are
//     spread over the lanes), and a sweep lasts as long as its longest chain of dependent steps;
//   * particles never share a warp, so a ready particle never waits for a neighbour lane's step and divergent
//     steps do not serialise each other;
//   * conflict detection and the wait are lane-parallel too: nine lanes walk the nine bins around the particle,
//     up to 32 blockers are polled at once.
// Included by sm_engine.cu after the bin / particle-I/O helpers.
#pragma once
#include "sm_coop.cuh"

#ifndef SM_SW_WARPS
#define SM_SW_WARPS 8        // warps (= particles in flight) per block
#endif
#ifndef SM_SW_MINBLOCKS
#define SM_SW_MINBLOCKS 3    // resident blocks per SM the kernel is compiled for (register cap)
#endif
#define SM_SW_NEAR 31        // in-range lower-index particles tracked exactly (one polling lane each)
#define SM_SW_NEARX 128      // ... by the exact schedule, which polls them in rounds of 32 (dense clusters - water
                             // collecting in a pit - are where exact footprints pay most: scripts/chain_analysis.py)

// warp policy of sm_coop.cuh on the device.  Every primitive is a full-warp synchronisation point on both
// sides: __syncwarp() orders the memory accesses of the participating lanes, so what lanes wrote before a
// phase is visible inside it and what the phase wrote is visible after it.
struct WarpDev {
  int lane;
  template <class F> __device__ __forceinline__ void each(int n, F f) {
    __syncwarp();
    if (lane < n) f(lane);
    __syncwarp();
  }
  template <class F> __device__ __forceinline__ unsigned int ballot(int n, F f) {
    __syncwarp();
    bool v = false;
    if (lane < n) v = f(lane);
    const unsigned int m = __ballot_sync(0xffffffffu, v);
    __syncwarp();
    return m;
  }
  template <class F> __device__ __forceinline__ void one(F f) {
    __syncwarp();
    if (lane == 0) f();
    __syncwarp();
  }
  __device__ __forceinline__ bool lead() const { return lane == 0; }
};

// backing store of CoopWin on the device
template <bool MULTI, bool BUDGET = false> struct DevBack {
  static constexpr bool kBudget = BUDGET;
  static constexpr bool kHydroHooks = false;
  __device__ __forceinline__ void air_mark(Sec32*, int, int) {}
  __device__ __forceinline__ void wet_mark(int, int) {}
  __device__ __forceinline__ double volume_factor() const { return c.volume_factor; }
  const DevCtx& c;
  const SoilDev* s_soils;   // shared-memory copy of the soil table
  unsigned int phase;       // sweep number mod 3: frees go to ring[phase], allocations pop ring[(phase+1)%3]
  int cur_q;                // owner rank of the column the next col_* call works on
  __device__ __forceinline__ DevBack(const DevCtx& ctx, const SoilDev* ss, unsigned int tag)
      : c(ctx), s_soils(ss), phase(tag % 3u), cur_q(0) {}
  __device__ __forceinline__ int dimx() const { return c.dimx; }
  __device__ __forceinline__ int dimy() const { return c.dimy; }
  __device__ __forceinline__ int scale() const { return c.scale; }
  __device__ __forceinline__ const SoilDev* soilp(uint32_t t) const { return &s_soils[t]; }
  __device__ __forceinline__ Sec32* cell_ptr(int x, int y) const { return ::cell_ptr<MULTI>(c, x, y); }
  __device__ __forceinline__ void focus(int x, int) { if (MULTI) cur_q = owner_of_x<true>(c, x); }
  __device__ __forceinline__ Sec32 pool_load(uint32_t i) { return MULTI ? c.peer[cur_q].pool[i] : c.pool[i]; }
  __device__ __forceinline__ void pool_store(uint32_t i, const Sec32& r) {
    if (MULTI) c.peer[cur_q].pool[i] = r; else c.pool[i] = r;
  }
  // Ticket pop from the ring that was filled two sweeps ago, else bump allocation (DESIGN.md section 3).
  // Three rings instead of two: on a sharded map the strips two ranks apart may be one sweep apart (the
  // per-sweep barrier only couples neighbouring strips) and both reach the pool of the strip between them,
  // so the ring being popped in sweep s must not be the one sweep s-1 or s+1 appends to.  The column's
  // owner holds the pool; its counters may live on another GPU (system-scope atomics).
  __device__ uint32_t pool_alloc() {
    const unsigned int pr = (phase + 1u) % 3u;
    RunCtl* const ctl = MULTI ? c.peer[cur_q].ctl : c.ctl;
    uint32_t* const ring = MULTI ? c.peer[cur_q].ringbuf[pr] : c.ringbuf[pr];
    const unsigned long long cap = MULTI ? c.peer[cur_q].pool_cap : c.pool_cap;
    PoolRing* R = &ctl->ring[pr];
    const unsigned long long t = *((volatile unsigned long long*)&R->tail);
    if (*((volatile unsigned long long*)&R->head) < t) {
      const unsigned long long h = MULTI ? atomicAdd_system(&R->head, 1ull) : atomicAdd(&R->head, 1ull);
      if (h < t) return ring[h % cap];
      if (MULTI) atomicMin_system(&R->head, t); else atomicMin(&R->head, t);
    }
    const unsigned long long bmp = MULTI ? atomicAdd_system(&ctl->bump, 1ull) : atomicAdd(&ctl->bump, 1ull);
    if (bmp < cap) return (uint32_t)bmp;
    atomicOr(&c.ctl->err, 1u << 3);   // SM_ERR_POOL
    atomicAdd(&c.ctl->drops, 1ull);
    return SM_NIL;
  }
  __device__ void pool_free(uint32_t i) {
    RunCtl* const ctl = MULTI ? c.peer[cur_q].ctl : c.ctl;
    uint32_t* const ring = MULTI ? c.peer[cur_q].ringbuf[phase] : c.ringbuf[phase];
    const unsigned long long cap = MULTI ? c.peer[cur_q].pool_cap : c.pool_cap;
    PoolRing* R = &ctl->ring[phase];
    const unsigned long long t = MULTI ? atomicAdd_system(&R->tail, 1ull) : atomicAdd(&R->tail, 1ull);
    ring[t % cap] = i;
  }
  __device__ __forceinline__ float wfreq(int i) const { return c.wfreq[i]; }
  __device__ __forceinline__ float wtrack(int i) const { return c.wtrack[i]; }
  __device__ __forceinline__ float windfreq(int i) const { return c.windfreq[i]; }
  __device__ __forceinline__ void set_wtrack(int i, float v) { c.wtrack[i] = v; }
  __device__ __forceinline__ void set_windfreq(int i, float v) { c.windfreq[i] = v; }
  __device__ __forceinline__ void note_transfer() {}
  __device__ __forceinline__ void pspeed(float px, float py, double height, float* ps) const {
    const WindField f{c.wind_v4, c.wind_nx, c.wind_ny, c.wind_nz, c.dimx, c.dimy, c.scale};
    wind_field_pspeed(f, px, py, height, ps);
  }
};

struct __align__(32) WarpSmem {
  CoopScratch cs;
  uint32_t blk[SM_SW_NEARX];   // in-range lower-index particles of this sweep (rank in bits 28-31 on a sharded map)
  uint32_t pred[12];     // per-bin predecessors (largest lower index in each of the 3x3 bins)
  uint32_t cnt;
  uint32_t m0[SM_SW_NEARX / 32];   // exact schedule: bit l = entry l can delay move() (its box can meet plus(ipos))
  uint32_t n1[SM_SW_NEARX / 32];   // exact schedule: bit l = entry l still unresolved after the wait to move
  uint32_t remote;       // exact schedule: some in-range lower-index particle is executed by another rank
  uint32_t succ;         // a higher-index particle lives in the 3x3 bins: somebody may wait for this particle's hand-off
  uint32_t blkxy[SM_SW_NEARX];   // exact schedule: packed (ipos, reach) of entry l, as in the bin node
};

#ifndef SM_PREFETCH
#define SM_PREFETCH 1
#endif
__device__ __forceinline__ float next_dy(const WaterP& p) { return p.sy; }   // speed component along map y
__device__ __forceinline__ float next_dy(const WindP& p) { return p.sz; }
template <class W, class A> __device__ __forceinline__ int do_step_coop(W& w, A& a, WaterP& p) { return water_step_coop(w, a, p); }
template <class W, class A> __device__ __forceinline__ int do_step_coop(W& w, A& a, WindP& p) { return wind_step_coop(w, a, p); }

// Conflict detection for one particle and one sweep, nine lanes = the 3x3 bins around ipos.  Two steps are
// ordered iff their published boxes can meet (|dipos|_inf <= R_A + R_B).  Sparse case: every lower-index
// particle in range gets a polling lane, plus the own-bin predecessor.  Crowded case (more than SM_SW_NEAR in
// range): the nine per-bin predecessors.  Every particle always waits for its own-bin predecessor, hence
// "X done => every lower index in X's bin done", which makes the per-bin predecessors a complete (conservative)
// blocker set however large the cluster is.  Returns this lane's wait target (SM_NIL = none).
template <int KIND, bool MULTI, bool EXACT = false>
__device__ __forceinline__ uint32_t coop_scan(const DevCtx& c, WarpSmem& ws, int lane, unsigned int tag, int pid, int ix,
                                              int iy, int R) {
  const unsigned int par = tag & 1u;
  const int G = Reach<KIND>::G;
  const int nbx = (c.dimx + G - 1) / G, nby = (c.dimy + G - 1) / G;
  if (lane == 0) { ws.cnt = 0; ws.succ = 0; if (EXACT) ws.remote = 0; }
  if (EXACT && lane < SM_SW_NEARX / 32) ws.m0[lane] = 0;
  __syncwarp();
  if (lane < 9) {
    const int cx = ix / G + lane / 3 - 1, cy = iy / G + lane % 3 - 1;
    uint32_t best = SM_NIL;
    if (cx >= 0 && cx < nbx && cy >= 0 && cy < nby) {
      const int bq = MULTI ? owner_of_x<MULTI>(c, cx * G) : 0;
      const unsigned long long* hp = MULTI ? c.peer[bq].head[par] : c.head[par];
      const unsigned long long h = *((volatile const unsigned long long*)&hp[cx * nby + cy]);
      if ((unsigned int)(h >> 32) == tag) {
        const uint2* nodes = MULTI ? c.peer[bq].node[par] : c.node[par];
        const uint32_t qtag = MULTI ? ((uint32_t)bq << 28) : 0u;
        uint32_t j = (uint32_t)h;
        while (j != SM_NIL) {
          const uint2 nd = nodes[j];
          if (j > (uint32_t)pid) ws.succ = 1u;        // (same value from every lane that sees one)
          if (j < (uint32_t)pid) {
            if (best == SM_NIL || (j | qtag) > best) best = j | qtag;
            int dx = (int)(nd.y >> 18) - ix, dy = (int)((nd.y >> 4) & 0x3FFFu) - iy;
            const int D = R + (int)(nd.y & 0xFu);
            dx = dx < 0 ? -dx : dx;
            dy = dy < 0 ? -dy : dy;
            if (dx <= D && dy <= D) {
              const unsigned int at = atomicAdd(&ws.cnt, 1u);
              if (at < (EXACT ? SM_SW_NEARX : SM_SW_NEAR)) {
                ws.blk[at] = j | qtag;
                if (EXACT) {
                  ws.blkxy[at] = nd.y;
                  // static pruning: a neighbour whose box cannot meet plus(ipos) never delays the move
                  if (Foot<KIND>::box_hits_M((int)(nd.y >> 18) - ix, (int)((nd.y >> 4) & 0x3FFFu) - iy, (int)(nd.y & 0xFu)))
                    atomicOr(&ws.m0[at >> 5], 1u << (at & 31u));
                  if (MULTI && bq != c.rank) ws.remote = 1u;
                }
              }
            }
          }
          j = nd.x;
        }
      }
    }
    ws.pred[lane] = best;
  }
  __syncwarp();
  const unsigned int cnt = ws.cnt;
  if (cnt <= SM_SW_NEAR) {
    if (lane < (int)cnt) return ws.blk[lane];
    if (lane == 31) return ws.pred[4];
    return SM_NIL;
  }
  return lane < 9 ? ws.pred[lane] : SM_NIL;
}

// spin until every lane's target has published this sweep
template <bool MULTI>
__device__ __forceinline__ void coop_wait(const DevCtx& c, unsigned int tag, uint32_t tgt) {
  bool ok = (tgt == SM_NIL);
  const unsigned int* dp = nullptr;
  bool remote = false;
  if (!ok) {
    if (MULTI) {
      const int bq = (int)(tgt >> 28);
      dp = &c.peer[bq].done[tgt & 0x0FFFFFFFu];
      remote = (bq != c.rank);      // polled over NVLink: system scope
    } else dp = &c.done[tgt];
  }
  const bool had = !ok;
  for (;;) {
    if (!ok) {
      const unsigned int v = remote ? ld_relaxed_sys_u32(dp) : ld_relaxed_u32(dp);
      ok = v >= tag;
    }
    if (__all_sync(0xffffffffu, ok)) break;
    poll_backoff();
  }
  // acquire once: the word only grows, so this load reads a value >= tag and synchronises with its release
  if (had) { if (remote) (void)ld_acquire_sys_u32(dp); else (void)ld_acquire_u32(dp); }
}

// ---- barrier across the blocks of every rank of a sharded map ---------------------------------------------
// A sweep of rank q only interacts with the strips q-1 and q+1 (halo records within +-5 cells, the bins one bin
// beyond the strip edge, particles handed over to the adjacent strip, the neighbours' pools), so the per-sweep
// barrier couples NEIGHBOURING ranks only; every SM_XSYNC_K-th sweep - and whenever a launch may end - all
// ranks meet and exchange their live-particle counts (termination is decided at those sweeps, identically on
// every rank).  Between two such sweeps strips that are d ranks apart may be up to d-1 sweeps apart.
// Protocol: every block arrives on the local counter (fence + atomic); the block that arrives LAST publishes
// (epoch << 32 | live count) with one system-scope release store per rank involved - lane q of its first warp
// serves rank q, its own rank included - and the first warp of EVERY block polls the words of the ranks
// involved in its own rank's memory (acquire), lane q polling rank q.  No leader round trip, no serial loop over
// the peers.  Words are double-buffered by epoch parity: a rank can be at most one epoch ahead of a rank it
// synchronises with.  Returns the live particles over all ranks after a global barrier (undefined otherwise).
#define SM_XSYNC_K 8
__device__ __forceinline__ unsigned int grid_barrier_x(const DevCtx& c, unsigned int& epoch, unsigned int gbase,
                                                       unsigned int local_alive_slot, bool global,
                                                       unsigned int* s_total) {
  RunCtl* ctl = c.ctl;
  __syncthreads();
  epoch++;
  const unsigned int ge = gbase + epoch;           // global epoch of this barrier (never reset)
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    unsigned int prev = 0;
    if (lane == 0) {
      __threadfence();
      prev = atomicAdd(&ctl->barrier, 1u);
      __threadfence();
    }
    prev = __shfl_sync(0xffffffffu, prev, 0);
    const int d = lane - c.rank;
    const bool involved = lane < c.nranks && (global || (d >= -1 && d <= 1));
    if (prev == epoch * gridDim.x - 1u) {
      const unsigned int mine = ld_volatile_u32(&ctl->alive_slot[local_alive_slot]);
      if (involved)
        st_release_sys_u64(&c.peer[lane].ctl->xw[ge & 1u][c.rank], ((unsigned long long)ge << 32) | mine);
    }
    unsigned int cnt = 0;
    bool ok = !involved;
    for (;;) {
      if (!ok) {
        const unsigned long long wv = ld_relaxed_sys_u64(&ctl->xw[ge & 1u][lane]);
        if ((int)((unsigned int)(wv >> 32) - ge) >= 0) { ok = true; cnt = (unsigned int)wv; }
      }
      if (__all_sync(0xffffffffu, ok)) break;
      poll_backoff();
    }
    if (involved) (void)ld_acquire_sys_u64(&ctl->xw[ge & 1u][lane]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) *s_total = cnt;
  }
  __syncthreads();
  return *s_total;
}

// ---- exact footprints ------------------------------------------------------------------------------------------
// The conservative rule orders two steps whenever their boxes (ipos +- R, R = 3 water, 3..5 wind) overlap, but a
// water step really touches F = plus(ipos) U 3x3(npos) - about 14 of the 49 cells - and a wind step
// plus(ipos) U 5x5(ipos) U 5x5(npos) (cascades around both cells with one nested re-cascade) out of up to 121; npos
// is only known after move(), so under boxes a particle can wait for a chain of 2-3 boxes that overlap while the
// footprints do not.  With EXACT a
// particle publishes three words per sweep: mv (= npos, right after move(); it only lets others SKIP a wait, so it
// needs no fence), fin (its map writes are complete; release) and done (published in own-bin index order, which
// keeps "X done => every lower index in X's bin done" and with it the crowded fallback sound).  A lower-index
// particle B in range holds A back
//   before A.move()     only while B's writes {ipos_B} U 3x3(npos_B) can meet plus(ipos_A)
//                       (B not moved yet: while B's box can),
//   before A.interact() only while F_B can meet F_A (B not moved yet: while B's box can meet F_A).
// The oracle emulation of this rule halves the longest chain per sweep at config-3 density.  Particles with more
// than SM_SW_NEARX neighbours in range, or (sharded maps) with a neighbour executed by another rank, take the
// conservative path for that sweep - waiting for `done` is always sufficient.
// Returns the step's result; fin and done are published inside.
template <class W, class A> __device__ __forceinline__ int do_move_coop(W& w, A& a, WaterP& p, WaterMidCoop& m) { return water_move_coop(w, a, p, m, SM_CW_PLUS); }
template <class W, class A> __device__ __forceinline__ int do_move_coop(W& w, A& a, WindP& p, WindMidCoop& m) { return wind_move_coop(w, a, p, m, SM_CW_PLUS); }
template <class W, class A> __device__ __forceinline__ int do_interact_coop(W& w, A& a, WaterP& p, const WaterMidCoop& m) { return water_interact_coop(w, a, p, m); }
template <class W, class A> __device__ __forceinline__ int do_interact_coop(W& w, A& a, WindP& p, const WindMidCoop& m) { return wind_interact_coop(w, a, p, m); }
template <class W, class A> __device__ __forceinline__ int do_move_coop_full(W& w, A& a, WaterP& p, WaterMidCoop& m) { return water_move_coop(w, a, p, m, 0x1FFu); }
template <class W, class A> __device__ __forceinline__ int do_move_coop_full(W& w, A& a, WindP& p, WindMidCoop& m) { return wind_move_coop(w, a, p, m, 0x1FFu); }
template <int KIND> struct MidCoopType { typedef WaterMidCoop T; };
template <> struct MidCoopType<KIND_WIND> { typedef WindMidCoop T; };

template <int KIND, bool MULTI, bool BUDGET>
__device__ __forceinline__ int sweep_exact(const DevCtx& c, WarpSmem& ws, WarpDev& w, const SoilDev* s_soils,
                                           unsigned int tag, int pid, int ix, int iy, int myR,
                                           typename PType<KIND>::T& p, bool edge) {
  const int lane = w.lane;
  const unsigned int cnt = ws.cnt;
  const uint32_t ownpred = ws.pred[4];
  // Entry base + lane of the neighbour list is this lane's in round base / 32; both waits are conjunctions over the
  // entries, so the rounds simply follow one another.
  // ---- wait to move ----
  for (unsigned int base = 0; base < cnt; base += 32u) {
    const bool mine = base + (unsigned int)lane < cnt;
    const uint32_t j = mine ? (ws.blk[base + lane] & 0x0FFFFFFFu) : 0u;   // executed by this rank (else the caller goes conservative)
    const uint32_t jxy = mine ? ws.blkxy[base + lane] : 0u;
    const int jx = (int)(jxy >> 18), jy = (int)((jxy >> 4) & 0x3FFFu);
    bool need1 = mine;                                                    // still to be resolved before interact()
    bool need0 = mine && ((ws.m0[base >> 5] >> lane) & 1u);               // ... before move()
    bool acq = false;          // this lane's neighbour was resolved by its fin word: acquire it once after the loop
    for (;;) {
      if (need0) {
        if (ld_relaxed_u32(&c.fin[j]) >= tag) { need0 = false; need1 = false; acq = true; }
        else {
          const unsigned long long v = *((volatile unsigned long long*)&c.mv[j]);
          if ((unsigned int)(v >> 32) == tag) {
            const int mx = (int)((v >> 16) & 0xFFFFu), my = (int)(v & 0xFFFFu);
            if (!Foot<KIND>::W_hits_M(jx, jy, mx, my, ix, iy)) need0 = false;
          }
        }
      }
      if (!__any_sync(0xffffffffu, need0)) break;
      poll_backoff();
    }
    if (acq) (void)ld_acquire_u32(&c.fin[j]);
    const unsigned int left = __ballot_sync(0xffffffffu, need1);
    if (lane == 0) ws.n1[base >> 5] = left;
  }
  __syncwarp();
  DevBack<MULTI, BUDGET> back(c, s_soils, tag);
  CoopWin<DevBack<MULTI, BUDGET> > a(back, &ws.cs);
  typename MidCoopType<KIND>::T mid;
  int r = do_move_coop(w, a, p, mid);
  if (r == SM_ALIVE) {
    const int nx = (int)roundf(p.px), ny = (int)roundf(p.py);
    if (lane == 0)
      *((volatile unsigned long long*)&c.mv[pid]) = ((unsigned long long)tag << 32) | ((unsigned long long)nx << 16) | (unsigned long long)ny;
    // ---- wait to interact ----
    for (unsigned int base = 0; base < cnt; base += 32u) {
      const unsigned int left = ws.n1[base >> 5];
      if (left == 0u) continue;
      bool need1 = (left >> lane) & 1u;
      const uint32_t j = need1 ? (ws.blk[base + lane] & 0x0FFFFFFFu) : 0u;
      const uint32_t jxy = need1 ? ws.blkxy[base + lane] : 0u;
      const int jx = (int)(jxy >> 18), jy = (int)((jxy >> 4) & 0x3FFFu), jR = (int)(jxy & 0xFu);
      int mx = 0, my = 0;
      bool moved = false;                                  // neighbour's npos known
      bool acq = false;
      for (;;) {
        if (need1) {
          if (ld_relaxed_u32(&c.fin[j]) >= tag) { need1 = false; acq = true; }
          else {
            if (!moved) {
              const unsigned long long v = *((volatile unsigned long long*)&c.mv[j]);
              if ((unsigned int)(v >> 32) == tag) { mx = (int)((v >> 16) & 0xFFFFu); my = (int)(v & 0xFFFFu); moved = true; }
            }
            const bool hit = moved ? Foot<KIND>::F_hits_F(ix, iy, nx, ny, jx, jy, mx, my)
                                   : Foot<KIND>::box_hits_F(ix, iy, nx, ny, jx, jy, jR);
            if (!hit) need1 = false;
          }
        }
        if (!__any_sync(0xffffffffu, need1)) break;
        poll_backoff();
      }
      if (acq) (void)ld_acquire_u32(&c.fin[j]);
    }
    r = do_interact_coop(w, a, p, mid);
    a.flush(w);
  }
  // stalled or left the map in move(): only track[] was written
  if (lane == 0) {
    const unsigned int pub = (r == SM_ALIVE) ? tag : 0xFFFFFFFFu;
    if (ws.succ) {
      // `done` in own-bin index order
      const unsigned int* dp = nullptr;
      if (ownpred != SM_NIL) dp = MULTI ? &c.peer[ownpred >> 28].done[ownpred & 0x0FFFFFFFu] : &c.done[ownpred];
      if (!(MULTI && edge) && (dp == nullptr || ld_relaxed_u32(dp) >= tag)) {
        // the predecessor has published already (the usual case): one release fence covers both words
        if (dp != nullptr) (void)ld_acquire_u32(dp);
        fence_acq_rel_gpu();
        st_relaxed_u32(&c.fin[pid], pub);
        st_relaxed_u32(&c.done[pid], pub);
      } else {
        st_release_u32(&c.fin[pid], pub);
        if (dp != nullptr) {
          while (ld_relaxed_u32(dp) < tag) poll_backoff();
          (void)ld_acquire_u32(dp);
        }
        if (MULTI && edge) st_release_sys_u32(&c.done[pid], pub);
        else st_release_u32(&c.done[pid], pub);
      }
    } else {             // no higher index in the 3x3 bins: nobody waits for fin or done (see the conservative path)
      st_volatile_u32(&c.fin[pid], pub);
      st_volatile_u32(&c.done[pid], pub);
    }
  }
  __syncwarp();
  return r;
}

// Load the live mask (W words) into shared memory, build its exclusive popcount prefix, return the number of live
// particles.  Called by every thread of the block; ends with a block barrier.
template <int NWARPS>
__device__ __forceinline__ unsigned int live_total(const unsigned int* __restrict__ mask, int W, unsigned int* s_word,
                                                   unsigned int* s_pref, unsigned int* s_wsum) {
  const int T = NWARPS * 32;
  const int cw = (W + T - 1) / T;                       // contiguous words per thread
  const int lo = threadIdx.x * cw, hi = (lo + cw < W) ? lo + cw : W;
  unsigned int local = 0;
  for (int i = lo; i < hi; i++) {
    const unsigned int wd = ld_relaxed_u32(&mask[i]);
    s_word[i] = wd;
    local += (unsigned int)__popc(wd);
  }
  unsigned int incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int v = __shfl_up_sync(0xffffffffu, incl, o);
    if ((int)(threadIdx.x & 31) >= o) incl += v;
  }
  __syncthreads();                                      // previous users of s_wsum / s_pref are done
  if ((threadIdx.x & 31) == 31) s_wsum[threadIdx.x >> 5] = incl;
  __syncthreads();
  unsigned int base = 0, total = 0;
#pragma unroll
  for (int k = 0; k < NWARPS; k++) {
    const unsigned int v = s_wsum[k];
    if (k < (int)(threadIdx.x >> 5)) base += v;
    total += v;
  }
  unsigned int run = base + incl - local;
  for (int i = lo; i < hi; i++) { s_pref[i] = run; run += (unsigned int)__popc(s_word[i]); }
  __syncthreads();
  return total;
}

template <int KIND, bool MULTI, bool BUDGET, bool EXACT>
__global__ void __launch_bounds__(SM_SW_WARPS * 32, SM_SW_MINBLOCKS) k_sweep(DevCtx c, int n, const float* __restrict__ spawn,
                                                                            int max_sweeps) {
  typedef typename PType<KIND>::T P;
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  __shared__ unsigned int s_alive, s_total, s_wsum[SM_SW_WARPS];
  __shared__ WarpSmem s_w[SM_SW_WARPS];
  extern __shared__ unsigned int s_live[];          // [0, W): this sweep's live mask, [W, 2W): exclusive popcount prefix
  const int W = (n + 31) >> 5;
  unsigned int* const s_word = s_live;
  unsigned int* const s_pref = s_live + W;
  for (int i = threadIdx.x; i < c.nsoils; i += blockDim.x) s_soils[i] = c.soils[i];
  if (threadIdx.x == 0) s_alive = 0;
  __syncthreads();

  RunCtl* ctl = c.ctl;
  unsigned int epoch = 0;
  const unsigned int tag0 = ctl->tag_base;   // constant during the launch (rewritten at the very end)
  const unsigned int gbase = MULTI ? ctl->epoch_base : 0u;
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int slot = blockIdx.x * SM_SW_WARPS + wib;
  const int nslots = gridDim.x * SM_SW_WARPS;
  WarpSmem& ws = s_w[wib];
  WarpDev w{lane};

  unsigned long long n_steps = 0, n_oob = 0, n_evap = 0, n_stall = 0;   // warp-uniform from the sweep loop on
  bool any_doa = false;

  // ---- prologue: spawn (ctor bodies water.h:13-17 / wind.h:15-20) or resume, fill the bins; one thread per particle ----
  unsigned int total_alive = 0;
  {
    unsigned int my_alive = 0;
    unsigned long long doa = 0;
    const int nthreads = gridDim.x * blockDim.x;
    for (int pid = gtid; pid < n; pid += nthreads) {
      bool alive;
      if (spawn != nullptr) {
        const float x = spawn[2 * pid], y = spawn[2 * pid + 1];
        const int sx = (int)roundf(x), sy = (int)roundf(y);
        if (MULTI && owner_of_x<MULTI>(c, sx) != c.rank) {     // another rank spawns this one
          c.alive[pid] = 0;
          if (BUDGET) for (int k = 0; k < SM_BUDGET_SLOTS; k++) c.bud[(size_t)pid * SM_BUDGET_SLOTS + k] = 0.0;
          continue;
        }
        const uint32_t contains = s_soils[rec_surface(*cell_ptr<MULTI>(c, sx, sy))].transports;
        if (KIND == KIND_WATER) {
          WaterP q{x, y, 0.0f, 0.0f, 1.0, 0.0, contains};
          store_particle(c, pid, q);
          alive = true;
        } else {
          WindP q{x, y, -2.0f, 0.0f, 1.0f, 0.0, 0.0, contains};
          store_particle(c, pid, q);
          // wind.h:56-57: a particle whose load cannot be suspended dies in its first move() without
          // touching anything
          alive = !(s_soils[contains].suspension == 0.0);
          if (!alive) { doa++; any_doa = true; }
        }
        c.alive[pid] = alive ? 1 : 0;
        c.done[pid] = alive ? (tag0 - 1u) : 0xFFFFFFFFu;
        if (EXACT) c.fin[pid] = alive ? (tag0 - 1u) : 0xFFFFFFFFu;
        if (BUDGET) for (int k = 0; k < SM_BUDGET_SLOTS; k++) c.bud[(size_t)pid * SM_BUDGET_SLOTS + k] = 0.0;
      } else {
        alive = c.alive[pid] != 0;
      }
      if (alive) {
        P q;
        load_particle(c, pid, q);
        bin_insert<KIND, MULTI>(c, tag0, pid, (int)roundf(q.px), (int)roundf(q.py), particle_reach(q), c.rank);
        atomicOr(&c.lmask[tag0 % 3u][pid >> 5], 1u << (pid & 31));     // the masks were zeroed by the host
        my_alive++;
      }
    }
    if (doa) atomicAdd(&ctl->exit_oob, doa);
    if (my_alive) atomicAdd(&s_alive, my_alive);
    __syncthreads();
    if (threadIdx.x == 0) {
      if (s_alive) atomicAdd(&ctl->alive_slot[0], s_alive);
      s_alive = 0;
    }
    if (MULTI) total_alive = grid_barrier_x(c, epoch, gbase, 0u, true, &s_total);
    else grid_barrier(&ctl->barrier, epoch);
  }
  // neighbour-only barriers need the bins a rank's neighbours scan and the bins a rank two strips away inserts
  // into to be different ones: at least three bins per strip
  const bool xnb = MULTI && c.strip_w >= 3 * Reach<KIND>::G;
  bool xglobal = true;          // was the barrier that opened this sweep a global one (total_alive valid)?
  int last_active = -1;         // last sweep in which this warp executed a particle

  int s = 0;
  for (;; s++) {
    const unsigned int tag = tag0 + (unsigned int)s;
    if (max_sweeps >= 0 && s >= max_sweeps) {
      if (!MULTI) total_alive = live_total<SM_SW_WARPS>(c.lmask[tag % 3u], W, s_word, s_pref, s_wsum);
      break;
    }
    // ---- who is alive, in index order ------------------------------------------------------------------------
    // The live particles of this rank are the set bits of lmask[tag % 3] (written during the previous sweep,
    // complete since the barrier).  Every block loads the mask and its exclusive popcount prefix into shared
    // memory; the warp with grid-wide index g then runs the live particles of RANK g, g + nslots, g + 2 nslots, ...
    // - ascending index within a warp (no wait can cycle), and every warp gets the same share whatever the pattern
    // of deaths is.  (With a fixed particle -> warp map the warp holding the most survivors set the pace of the
    // sweep: 5-6 of its 7 particles where the average is under 2.)
    const unsigned int live = live_total<SM_SW_WARPS>(c.lmask[tag % 3u], W, s_word, s_pref, s_wsum);
    if (!MULTI) total_alive = live;
    if ((!MULTI || xglobal) && total_alive == 0) break;
    {   // the mask two sweeps ahead becomes the survivors' mask of the next sweep: clear it now
      unsigned int* const z = c.lmask[(tag + 2u) % 3u];
      for (int i = gtid; i < W; i += gridDim.x * blockDim.x) z[i] = 0u;
    }
    if (gtid == 0) {
      if (MULTI) st_volatile_u32(&ctl->alive_slot[(s + 2) % 3], 0u);
      st_volatile_u32(&ctl->ticket[(tag + 2u) % 3u], 0u);
    }

    unsigned int my_alive = 0;
#ifdef SM_PROFILE
    unsigned long long prof_warp = 0;
    if (gtid == 0 && s < 16380) c.dbg[8 * s + 0] = live;
#endif
    {
    // Rank g belongs to warp g; the ranks beyond the first nslots are claimed one at a time, in order, by whichever
    // warp is free (a warp stuck in a long step does not hold up the particles a fixed map would queue behind it).
    // Ranks are handed out in ascending order and a holder only ever waits for lower ranks, which are done or held
    // by a running warp: no wait can cycle.
    for (unsigned int rank = (unsigned int)slot; rank < live;) {
      // rank -> particle: the word whose prefix range holds it, then the (rank - prefix)-th set bit of that word
      int lo = 0, hi = W - 1;
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_pref[mid] <= rank) lo = mid; else hi = mid - 1;
      }
      const int pid = (lo << 5) + (int)__fns(s_word[lo], 0u, (int)(rank - s_pref[lo]) + 1);
      last_active = s;
#ifdef SM_PROFILE
      const long long pc0 = clock64();
      if (lane == 0 && s < 16380) {
        unsigned long long gt; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
        atomicMax(&c.dbg[8 * s + 6], ~gt);             // max of the complement = earliest start
      }
#endif
      P p;
      load_particle(c, pid, p);
      const int ix = (int)roundf(p.px), iy = (int)roundf(p.py);
      const int myR = particle_reach(p);
      const uint32_t tgt = coop_scan<KIND, MULTI, EXACT>(c, ws, lane, tag, pid, ix, iy, myR);
#ifdef SM_PROFILE
      const long long pc1 = clock64();
      long long pc2 = pc1;
#endif
      // sharded map: only particles within two bins of a strip edge can have touched a peer's records or be polled
      // from another rank: they release at system scope, the interior ones at gpu scope
      bool edge = false;
      if (MULTI) {
        const int xlo = c.rank * c.strip_w, xhi = xlo + c.strip_w;
        edge = (ix < xlo + 32 && c.rank > 0) || (ix >= xhi - 32 && c.rank < c.nranks - 1);
      }
      int r = SM_ALIVE;
      bool exact_now = false;
      if constexpr (EXACT) {
        // (also for a particle with nothing in range: its mv word is what lets the particles behind it skip waits -
        // sending those down the conservative path makes the particles behind it wait longer)
        exact_now = ws.cnt <= SM_SW_NEARX && !(MULTI && ws.remote);
        if (exact_now) r = sweep_exact<KIND, MULTI, BUDGET>(c, ws, w, s_soils, tag, pid, ix, iy, myR, p, edge);
      }
      if (!exact_now) {
        coop_wait<MULTI>(c, tag, tgt);
#ifdef SM_PROFILE
        pc2 = clock64();
#endif
        DevBack<MULTI, BUDGET> back(c, s_soils, tag);
        CoopWin<DevBack<MULTI, BUDGET> > a(back, &ws.cs);
#ifdef SM_PROFILE
        long long pcm, pci;
        {
          typename MidCoopType<KIND>::T mid;
          r = do_move_coop_full(w, a, p, mid);
          pcm = clock64();
          if (r == SM_ALIVE) r = do_interact_coop(w, a, p, mid);
          pci = clock64();
        }
#else
        r = do_step_coop(w, a, p);
#endif
        // hand-off first: the map writes are all the successors of this step wait for
        a.flush(w);
        if (lane == 0) {
          const unsigned int pub = (r == SM_ALIVE) ? tag : 0xFFFFFFFFu;
          if (ws.succ) {
            if (EXACT && !(MULTI && edge)) {      // one release fence for both words
              fence_acq_rel_gpu();
              st_relaxed_u32(&c.fin[pid], pub);
              st_relaxed_u32(&c.done[pid], pub);
            } else {
              if (EXACT) st_release_u32(&c.fin[pid], pub);
              if (MULTI && edge) st_release_sys_u32(&c.done[pid], pub);
              else st_release_u32(&c.done[pid], pub);
            }
          } else {
            // Nobody can be waiting for this hand-off: a waiter lists particles of its own 3x3 bins, so it would
            // sit in ours, and no higher index does.  The release fence (the single most expensive instruction of
            // a step: it waits for every write-back to be acknowledged) is left to the sweep barrier.
            if (EXACT) st_volatile_u32(&c.fin[pid], pub);
            st_volatile_u32(&c.done[pid], pub);
          }
        }
#ifdef SM_PROFILE
        if (lane == 0) {   // phase sums of the conservative path, row 16383 of the debug buffer
          const long long pcp = clock64();
          unsigned long long* const ph = c.dbg + 8 * 16383;
          atomicAdd(&ph[0], (unsigned long long)(pc1 - pc0));
          atomicAdd(&ph[1], (unsigned long long)(pc2 - pc1));
          atomicAdd(&ph[2], (unsigned long long)(pcm - pc2));
          atomicAdd(&ph[3], (unsigned long long)(pci - pcm));
          atomicAdd(&ph[4], (unsigned long long)(pcp - pci));
          atomicAdd(&ph[5], 1ull);
          if (ws.succ) { atomicAdd(&ph[6], (unsigned long long)(pcp - pci)); atomicAdd(&ph[7], 1ull); }
        }
#endif
      }
      const int jx = (int)roundf(p.px), jy = (int)roundf(p.py);
      if (lane == 0) {
        // own state and next sweep's bins are only needed after the grid barrier
        if (BUDGET) {
          // the step's six sums join the particle's totals; the totals travel with a particle that changes strips
          // (exactly one rank holds them), so the final sum per particle is in step order on any number of ranks
          const int bq = (MULTI && r == SM_ALIVE) ? owner_of_x<MULTI>(c, jx) : c.rank;
          double* const dst = (MULTI && bq != c.rank) ? c.peer[bq].bud : c.bud;
          for (int k = 0; k < SM_BUDGET_SLOTS; k++) {
            const size_t at = (size_t)pid * SM_BUDGET_SLOTS + k;
            const double tot = c.bud[at] + ws.cs.acc[k];
            if (MULTI && bq != c.rank) c.bud[at] = 0.0;
            dst[at] = tot;
          }
        }
        if (r == SM_ALIVE) {
          int ddx = jx - ix, ddy = jy - iy;
          ddx = ddx < 0 ? -ddx : ddx; ddy = ddy < 0 ? -ddy : ddy;
          const int lim = myR - Reach<KIND>::RING;      // the step promised to stay within ipos +- lim
          if (ddx > lim || ddy > lim) atomicOr(&ctl->err, 1u << 4);  // SM_ERR_REACH
          const int nq = owner_of_x<MULTI>(c, jx);
          if (MULTI && nq != c.rank) {
            // the particle leaves this strip: hand it to the new owner (its arrays, its bins)
            DevCtx o = c;   // view of the owner's particle arrays
            o.pa = c.peer[nq].pa; o.pb = c.peer[nq].pb; o.pc = c.peer[nq].pc;
            store_particle(o, pid, p);
            c.peer[nq].done[pid] = tag;            // it has completed this sweep, wherever it is asked
            if (EXACT) c.peer[nq].fin[pid] = tag;
            c.peer[nq].alive[pid] = 1;
            c.alive[pid] = 0;
            atomicOr_system(&c.peer[nq].lmask[(tag + 1u) % 3u][pid >> 5], 1u << (pid & 31));   // runnable there next sweep
          } else {
            store_particle(c, pid, p);
            atomicOr(&c.lmask[(tag + 1u) % 3u][pid >> 5], 1u << (pid & 31));
          }
          bin_insert<KIND, MULTI>(c, tag + 1u, pid, jx, jy, particle_reach(p), nq);
        } else {
          store_particle(c, pid, p);
          c.alive[pid] = 0;
        }
      }
#if SM_PREFETCH
      // next sweep's records towards L2 while this sweep finishes: the 3x3 blocks around the next ipos and around
      // the position the current speed predicts after it (a wind particle covers fresh terrain every sweep; the
      // config-3 map is ten times the H100's 50 MB L2)
      if (r == SM_ALIVE && lane < 18) {
        const int ox = lane < 9 ? jx : (int)roundf(p.px + p.sx);
        const int oy = lane < 9 ? jy : (int)roundf(p.py + next_dy(p));
        const int k = lane < 9 ? lane : lane - 9;
        const int x = ox + k / 3 - 1, y = oy + k % 3 - 1;
        if (x >= 0 && y >= 0 && x < c.dimx && y < c.dimy && (!MULTI || owner_of_x<MULTI>(c, x) == c.rank))
          prefetch_l2(cell_ptr<MULTI>(c, x, y));
      }
#endif
#ifdef SM_PROFILE
      {
        const long long pc3 = clock64();
        prof_warp += (unsigned long long)(pc3 - pc0);
        if (lane == 0 && s < 16380) {
          atomicMax(&c.dbg[8 * s + 1], (unsigned long long)(pc3 - pc2));
          atomicMax(&c.dbg[8 * s + 2], (unsigned long long)(pc2 - pc1));
          atomicAdd(&c.dbg[8 * s + 4], (unsigned long long)(pc3 - pc2));
          atomicAdd(&c.dbg[8 * s + 5], 1ull);
        }
      }
#endif
      if (r == SM_ALIVE) { n_steps++; my_alive++; }
      else if (r == SM_EXIT_OOB) n_oob++;
      else if (r == SM_EXIT_STALL) n_stall++;
      else { n_steps++; n_evap++; }
      __syncwarp();
      // next rank: only when there are more live particles than warps
      if (live <= (unsigned int)nslots) break;
      unsigned int nr = 0;
      if (lane == 0) nr = (unsigned int)nslots + atomicAdd(&ctl->ticket[tag % 3u], 1u);
      rank = __shfl_sync(0xffffffffu, nr, 0);
    }
    }
#ifdef SM_PROFILE
    if (lane == 0 && s < 16380 && prof_warp) {
      atomicMax(&c.dbg[8 * s + 3], prof_warp);
      unsigned long long gt; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
      atomicMax(&c.dbg[8 * s + 7], gt);
    }
#endif
    if (MULTI) {     // the cross-rank barrier carries this rank's survivor count
      if (lane == 0 && my_alive) atomicAdd(&s_alive, my_alive);
      __syncthreads();
      if (threadIdx.x == 0) {
        if (s_alive) atomicAdd(&ctl->alive_slot[(s + 1) % 3], s_alive);
        s_alive = 0;
      }
    }
    if (MULTI) {
      xglobal = !xnb || ((s + 1) % SM_XSYNC_K == 0) || (max_sweeps >= 0 && s + 1 >= max_sweeps);
      total_alive = grid_barrier_x(c, epoch, gbase, (unsigned int)((s + 1) % 3), xglobal, &s_total);
    } else grid_barrier(&ctl->barrier, epoch);
  }

  // ---- epilogue ----
  if (lane == 0) {
    if (n_steps) atomicAdd(&ctl->steps, n_steps);
    if (n_oob) atomicAdd(&ctl->exit_oob, n_oob);
    if (n_evap) atomicAdd(&ctl->exit_evap, n_evap);
    if (n_stall) atomicAdd(&ctl->exit_stall, n_stall);
  }
  // tag_base was read by every block before its first barrier; barrier/alive_slot are reset by the host
  // before the next launch
  if (any_doa) atomicMax(&ctl->sweeps, 1ull);
  // sharded map: termination is noticed at the next global barrier, up to SM_XSYNC_K - 1 empty sweeps late; the
  // sweep count of the batch is the last sweep in which any rank executed a particle (the host takes the max)
  if (MULTI && lane == 0 && last_active >= 0) atomicMax(&ctl->sweeps, (unsigned long long)(last_active + 1));
  if (gtid == 0) {
    if (!MULTI) atomicMax(&ctl->sweeps, (unsigned long long)s);
    ctl->alive = total_alive;
    ctl->tag_base = tag0 + (unsigned int)s + 2u;
    if (MULTI) ctl->epoch_base = gbase + epoch;
  }
}
