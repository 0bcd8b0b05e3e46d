// sm_engine.cu -- sm_90a kernels and the C ABI of include/soilmachine_b200.h.
//
// Hot path = k_run<KIND>: ONE persistent, co-resident kernel per particle batch.  Every sweep each
// live particle executes move()+interact() (sm_core.cuh) exactly once; particles whose conflict
// boxes overlap are serialised in ascending particle index by a dataflow wait (a particle spins
// until every lower-index particle within reach has published the current sweep tag), so the
// result is bit-identical to the reference functions driven sweep by sweep in index order
// (oracle lockstep mode).  One grid barrier per sweep; no kernel launch per sweep.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <algorithm>
#include "../../include/soilmachine_b200.h"
#include "../../include/soilmachine/soilfile.hpp"
#include "sm_device.cuh"
#include "sm_noise.cuh"
#include "sm_hydro.cuh"
#include "sm_lbm.cuh"

#define KIND_WATER 0
#define KIND_WIND 1

// conflict reach (SURVEY.md Appendix A.6): a water step stays within ipos+-3, a wind step within
// ipos+-5, so two steps commute unless |dipos|_inf <= 6 (water) / 10 (wind).  Bin edge >= reach*2
// keeps every possible blocker inside the 3x3 bins around a particle.
template <int KIND> struct Reach {
  static constexpr int D = (KIND == KIND_WATER) ? 6 : 10;       // largest possible sum of two reaches
  static constexpr int G = (KIND == KIND_WATER) ? 8 : 16;
  static constexpr int STEP = (KIND == KIND_WATER) ? 2 : 3;     // max |npos - ipos|_inf of any step
  static constexpr int RING = (KIND == KIND_WATER) ? 1 : 2;     // cells the cascade reaches beyond npos
};

// Footprint half-width R of the NEXT step of a particle: everything the step reads or writes lies in
// ipos +- R.  Water: |speed| = sqrt(2) after normalisation => npos within ipos+-2, cascade 3x3 => R = 3.
// Wind: the new horizontal speed is 0.8*m + 0.2*pspeed with |m| <= |speed| in both branches of wind.h:73-78
// (gravity only changes y; contact: m = 0.2 s - 0.8 s_tangential), so each component moves by at most
// rho = 0.8*|speed| + 0.4 and npos lies within ipos +- floor(1 + rho); cascade(.,1) with one nested
// re-cascade reaches 2 further (SURVEY.md A.6).  Slow particles therefore claim +-3 instead of +-5.
__device__ __forceinline__ int particle_reach(const WaterP&) { return 3; }
__device__ __forceinline__ int particle_reach(const WindP& p) {
  const float len = sqrtf(p.sx * p.sx + p.sy * p.sy + p.sz * p.sz);
  int r = (int)floorf(1.0f + 0.8f * len + 0.4f + 0.01f);
  r = r < 1 ? 1 : (r > 3 ? 3 : r);          // NaN speed -> r = 1; the step then dies out of bounds
  return r + 2;
}
#define SM_PACK_NODE(x, y, R) (((uint32_t)(x) << 18) | ((uint32_t)(y) << 4) | (uint32_t)(R))
#define SM_MIN_BIN 8
#ifndef SM_BLOCK
#define SM_BLOCK 128   // threads per block of the sweep kernel
#endif
#ifndef SM_MINBLOCKS
#define SM_MINBLOCKS 3  // resident blocks per SM the sweep kernels are compiled for (register cap)
#endif
#define SM_SWEEPS_NONE 0x40000000   // internal: run the prologue only
#ifndef SM_DEFAULT_EXACT
#define SM_DEFAULT_EXACT 1             // warp kernel: exact footprints for water batches (bit 0: shorter dependency
                                       // chains in dense water clusters), bit 1 = wind
#endif
#ifndef SM_DEFAULT_COOP
#define SM_DEFAULT_COOP true           // k_sweep (warp per particle); SM_KERNEL=thread selects the round-1 kernels
#endif
#define SM_DONE_FLOODED 0xFFFFFFFEu  // done[] of a dead particle whose flood() has run (0xFFFFFFFF = dead)

// ---------------------------------------------------------------------------------------------
// bins
// ---------------------------------------------------------------------------------------------
template <int KIND, bool MULTI = false>
__device__ __forceinline__ void bin_insert(const DevCtx& c, unsigned int tag, int pid, int ix, int iy, int R, int q = 0) {
  // q = rank that owns the column x = ix (the bins, like the particle, live with the owner)
  const unsigned int par = tag & 1u;
  const int G = Reach<KIND>::G;
  const int nby = (c.dimy + G - 1) / G;
  const int b = (ix / G) * nby + (iy / G);
  unsigned long long* head = MULTI ? c.peer[q].head[par] : c.head[par];
  uint2* node = MULTI ? c.peer[q].node[par] : c.node[par];
  // a sharded map's bin heads are also updated from other GPUs (particles handed over): system scope
  const unsigned long long ent = ((unsigned long long)tag << 32) | (unsigned long long)(uint32_t)pid;
  unsigned long long old = MULTI ? atomicExch_system(&head[b], ent) : atomicExch(&head[b], ent);
  node[pid] = make_uint2(((unsigned int)(old >> 32) == tag) ? (uint32_t)old : SM_NIL, SM_PACK_NODE(ix, iy, R));
}

// Conflict detection for one particle and one sweep.  Lists were completed before the grid barrier
// that opened this sweep.  scan_blockers walks the 3x3 bins once (non-blocking) and returns at most 9
// particle indices whose completion of sweep `tag` implies that EVERY lower-index particle with an
// overlapping conflict box has completed it:
//   sparse case : the (<= K) lower-index particles really in range, plus the own-bin predecessor;
//   crowded case: the 9 per-bin predecessors (largest lower index in each bin, at any distance).
// Every particle always waits for its own-bin predecessor, hence "X done" implies "every lower index
// in X's bin is done", which makes the per-bin predecessors a complete (conservative) blocker set and
// the hand-off from the last blocker to this particle O(1).
// Sharded maps: a neighbouring bin may belong to another rank; list entries carry that rank in bits 28-31
// (the blocker's `done` word lives with the rank that executes it this sweep = the owner of its bin).
template <int KIND, bool MULTI = false>
__device__ __forceinline__ unsigned int scan_blockers(const DevCtx& c, unsigned int tag, int pid, int ix, int iy,
                                                      int R, uint32_t (&list)[9]) {
  const unsigned int par = tag & 1u;
  const int G = Reach<KIND>::G;
  const int nbx = (c.dimx + G - 1) / G, nby = (c.dimy + G - 1) / G;
  const int bx = ix / G, by = iy / G;
  unsigned long long heads[9];
#pragma unroll
  for (int k = 0; k < 9; k++) {
    const int cx = bx + k / 3 - 1, cy = by + k % 3 - 1;
    const unsigned long long* hp = MULTI ? c.peer[owner_of_x<MULTI>(c, (cx < 0 ? 0 : cx) * G)].head[par] : c.head[par];
    heads[k] = (cx >= 0 && cx < nbx && cy >= 0 && cy < nby)
                   ? *((volatile const unsigned long long*)&hp[cx * nby + cy]) : 0ull;
  }
  const int K = 6;
  uint32_t near_[K];
  uint32_t pred[9];
  int nnear = 0;
  bool crowded = false;
#pragma unroll
  for (int q = 0; q < K; q++) near_[q] = SM_NIL;
#pragma unroll
  for (int k = 0; k < 9; k++) {
    pred[k] = SM_NIL;
    const unsigned long long h = heads[k];
    if ((unsigned int)(h >> 32) != tag) continue;
    uint32_t j = (uint32_t)h;
    uint32_t best = SM_NIL;
    const int bq = MULTI ? owner_of_x<MULTI>(c, (bx + k / 3 - 1) * G) : 0;
    const uint2* nodes = MULTI ? c.peer[bq].node[par] : c.node[par];
    const uint32_t qtag = MULTI ? ((uint32_t)bq << 28) : 0u;
    while (j != SM_NIL) {
      const uint2 nd = nodes[j];
      if (j < (uint32_t)pid) {
        if (best == SM_NIL || (j | qtag) > best) best = j | qtag;
        int dx = (int)(nd.y >> 18) - ix, dy = (int)((nd.y >> 4) & 0x3FFFu) - iy;
        const int D = R + (int)(nd.y & 0xFu);       // the two footprints can meet iff |d| <= R_A + R_B
        dx = dx < 0 ? -dx : dx;
        dy = dy < 0 ? -dy : dy;
        if (dx <= D && dy <= D) {
          if (nnear < K) {
#pragma unroll
            for (int q = 0; q < K; q++) if (q == nnear) near_[q] = j | qtag;
            nnear++;
          } else crowded = true;
        }
      }
      j = nd.x;
    }
    pred[k] = best;
  }
  unsigned int mask = 0;
#pragma unroll
  for (int k = 0; k < 9; k++) {
    list[k] = crowded ? pred[k] : (k < K ? near_[k] : (k == K ? pred[4] : SM_NIL));
    if (list[k] != SM_NIL) mask |= 1u << k;
  }
  return mask;
}

// poll the still-unfinished blockers once; returns the mask of those not yet done
template <bool MULTI = false>
__device__ __forceinline__ unsigned int poll_blockers(const DevCtx& c, unsigned int tag, const uint32_t (&list)[9],
                                                      unsigned int mask) {
#pragma unroll
  for (int k = 0; k < 9; k++) {
    if ((mask >> k) & 1u) {
      if (MULTI) {
        // a blocker on another rank is polled over NVLink at system scope, a local one at gpu scope
        const int bq = (int)(list[k] >> 28);
        const unsigned int* dp = &c.peer[bq].done[list[k] & 0x0FFFFFFFu];
        const unsigned int v = (bq == c.rank) ? ld_acquire_u32(dp) : ld_acquire_sys_u32(dp);
        if (v >= tag) mask &= ~(1u << k);
      } else {
#ifdef SM_ACQREL
        if (ld_acquire_u32(&c.done[list[k]]) >= tag) mask &= ~(1u << k);
#else
        if (ld_volatile_u32(&c.done[list[k]]) >= tag) mask &= ~(1u << k);
#endif
      }
    }
  }
  return mask;
}

// ---------------------------------------------------------------------------------------------
// particle state I/O
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_particle(const DevCtx& c, int pid, WaterP& p) {
  float4 a = c.pa[pid]; double2 b = c.pb[pid]; uint2 d = c.pc[pid];
  p.px = a.x; p.py = a.y; p.sx = a.z; p.sy = a.w; p.volume = b.x; p.sediment = b.y; p.contains = d.x;
}
__device__ __forceinline__ void store_particle(const DevCtx& c, int pid, const WaterP& p) {
  c.pa[pid] = make_float4(p.px, p.py, p.sx, p.sy);
  c.pb[pid] = make_double2(p.volume, p.sediment);
  c.pc[pid] = make_uint2(p.contains, 0u);
}
__device__ __forceinline__ void load_particle(const DevCtx& c, int pid, WindP& p) {
  float4 a = c.pa[pid]; double2 b = c.pb[pid]; uint2 d = c.pc[pid];
  p.px = a.x; p.py = a.y; p.sx = a.z; p.sy = a.w; p.sediment = b.x; p.height = b.y;
  p.contains = d.x; p.sz = __uint_as_float(d.y);
}
__device__ __forceinline__ void store_particle(const DevCtx& c, int pid, const WindP& p) {
  c.pa[pid] = make_float4(p.px, p.py, p.sx, p.sy);
  c.pb[pid] = make_double2(p.sediment, p.height);
  c.pc[pid] = make_uint2(p.contains, __float_as_uint(p.sz));
}
template <int KIND> struct PType { typedef WaterP T; };
template <> struct PType<KIND_WIND> { typedef WindP T; };

template <class A> __device__ __forceinline__ int do_step(A& a, WaterP& p) { return water_step(a, p); }
template <class A> __device__ __forceinline__ int do_step(A& a, WindP& p) { return wind_step(a, p); }

// ---------------------------------------------------------------------------------------------
// the persistent sweep kernel
// ---------------------------------------------------------------------------------------------
#ifdef SM_PROFILE
__device__ __forceinline__ void ctl_marks(RunCtl* ctl, const unsigned long long* m) {
  for (int i = 1; i < 8; i++) if (m[i]) atomicAdd(&ctl->marks[i], m[i]);
}
#endif
// MULTI = the map is sharded by x-strips over several ranks (GPUs, or contexts sharing one GPU): a
// rank executes the particles whose ipos lies in its strip, reads/writes halo records, bins and `done`
// words of its neighbours through peer pointers, hands a particle that leaves the strip over to the new
// owner (state, bin entry and alive flag are written into the owner's arrays before the barrier) and
// synchronises sweeps with the cross-rank barrier.  The canonical order is unchanged, so an N-rank run
// is bit-identical to the 1-rank run.
template <int KIND, bool MULTI>
__global__ void __launch_bounds__(SM_BLOCK, SM_MINBLOCKS) k_run(DevCtx c, int n, const float* __restrict__ spawn,
                                            int max_sweeps, int lshift) {
  typedef typename PType<KIND>::T P;
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  __shared__ unsigned int s_alive;
  extern __shared__ __align__(32) unsigned char s_win[];   // (blockDim.x >> lshift) windows
  for (int i = threadIdx.x; i < c.nsoils; i += blockDim.x) s_soils[i] = c.soils[i];
  if (threadIdx.x == 0) s_alive = 0;
  __syncthreads();
  Sec32* my_win = (Sec32*)(s_win + (size_t)(threadIdx.x >> lshift) * SM_WIN_BYTES);

  RunCtl* ctl = c.ctl;
  unsigned int epoch = 0;
  const unsigned int tag0 = ctl->tag_base;   // constant during the launch (rewritten at the very end)
  const unsigned int gbase = MULTI ? ctl->epoch_base : 0u;
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const bool leader = (gtid & ((1 << lshift) - 1)) == 0;
  const int slot = gtid >> lshift;
  const int nslots = (gridDim.x * blockDim.x) >> lshift;
  const int trips = (n + nslots - 1) / nslots;

  unsigned long long n_steps = 0, n_oob = 0, n_evap = 0, n_stall = 0;
  bool any_doa = false;
  SM_PROF_DECL

  // ---- prologue: spawn (ctor bodies water.h:13-17 / wind.h:15-20) or resume, fill the bins ----
  unsigned int total_alive = 0;
  {
    unsigned int my_alive = 0;
    if (leader) {
      for (int pid = slot; pid < n; pid += nslots) {
        bool alive;
        if (spawn != nullptr) {
          const float x = spawn[2 * pid], y = spawn[2 * pid + 1];
          const int sx = (int)roundf(x), sy = (int)roundf(y);
          if (MULTI && owner_of_x<MULTI>(c, sx) != c.rank) {     // another rank spawns this one
            c.alive[pid] = 0;
            continue;
          }
          const uint32_t contains = s_soils[rec_surface(*cell_ptr<MULTI>(c, sx, sy))].transports;
          if (KIND == KIND_WATER) {
            WaterP w{x, y, 0.0f, 0.0f, 1.0, 0.0, contains};
            store_particle(c, pid, w);
            alive = true;
          } else {
            WindP w{x, y, -2.0f, 0.0f, 1.0f, 0.0, 0.0, contains};
            store_particle(c, pid, w);
            // wind.h:56-57: a particle whose load cannot be suspended dies in its first move()
            // without touching anything
            alive = !(s_soils[contains].suspension == 0.0);
            if (!alive) { n_oob++; any_doa = true; }
          }
          c.alive[pid] = alive ? 1 : 0;
          c.done[pid] = alive ? (tag0 - 1u) : 0xFFFFFFFFu;
        } else {
          alive = c.alive[pid] != 0;
        }
        if (alive) {
          P q;
          load_particle(c, pid, q);
          bin_insert<KIND, MULTI>(c, tag0, pid, (int)roundf(q.px), (int)roundf(q.py), particle_reach(q), c.rank);
          my_alive++;
        }
      }
    }
    if (my_alive) atomicAdd(&s_alive, my_alive);
    __syncthreads();
    if (threadIdx.x == 0) {
      if (s_alive) atomicAdd(&ctl->alive_slot[0], s_alive);
      s_alive = 0;
    }
    if (MULTI) total_alive = grid_barrier_multi(c, epoch, gbase, 0u);
    else grid_barrier(&ctl->barrier, epoch);
  }

  int s = 0;
  for (;; s++) {
    const unsigned int tag = tag0 + (unsigned int)s;
    if (!MULTI) total_alive = ld_volatile_u32(&ctl->alive_slot[s % 3]);
    if (total_alive == 0 || (max_sweeps >= 0 && s >= max_sweeps)) break;
    if (gtid == 0) st_volatile_u32(&ctl->alive_slot[(s + 2) % 3], 0u);
#ifdef SM_PROFILE
    if (gtid == 0 && s < 16384 && c.dbg) { c.dbg[2 * s] = (unsigned long long)clock64(); c.dbg[2 * s + 1] = total_alive; }
#endif

    unsigned int my_alive = 0;
    SM_PROF(0)   // barrier exit -> loop top
    // Warp-converged rounds: every lane scans its blockers once, then the warp loops - each round
    // the lanes whose blockers have all published this sweep execute their particle-step TOGETHER
    // (SIMT), the others poll again.
    for (int trip = 0; trip < trips; trip++) {
      const int pid = slot + trip * nslots;
      const bool has = leader && pid < n && c.alive[pid] != 0;
      P p;
      int ix = 0, iy = 0, myR = 0;
      uint32_t list[9];
      unsigned int waitmask = 0;
      if (has) {
        load_particle(c, pid, p);
        ix = (int)roundf(p.px); iy = (int)roundf(p.py);
        SM_PROF(1)   // state load
        myR = particle_reach(p);
        waitmask = scan_blockers<KIND, MULTI>(c, tag, pid, ix, iy, myR, list);
        SM_PROF(2)   // blocker scan
      }
      bool pending = has;
      for (;;) {
        if (pending && waitmask) waitmask = poll_blockers<MULTI>(c, tag, list, waitmask);
        const bool ready = pending && waitmask == 0;
        if (__ballot_sync(0xffffffffu, pending) == 0u) break;
#ifdef SM_NOSLEEP
        if (__ballot_sync(0xffffffffu, ready) == 0u) continue;
#else
        if (__ballot_sync(0xffffffffu, ready) == 0u) { __nanosleep(32); continue; }
#endif
        if (ready) {
          SM_PROF(12)  // waiting for blockers
#ifndef SM_ACQREL
          __threadfence();
#endif
          SM_PROF(3)   // acquire fence
          WinAccess<KIND, MULTI> a(c, s_soils, tag, my_win);
          const int r = do_step(a, p);
#ifdef SM_PROFILE
          { long long t_ = clock64();
            if (a.t_target1) { prof_[8] += a.t_begin - pt_; prof_[9] += a.t_target0 - a.t_begin;
                               prof_[10] += a.t_target1 - a.t_target0; prof_[11] += t_ - a.t_target1;
                               ctl_marks(ctl, a.t_mark); } }
#endif
#ifdef SM_PROFILE
          { const unsigned long long dt_ = (unsigned long long)(clock64() - pt_);   // step duration (pt_ = after acquire)
            if (dt_ > 20000ull) atomicAdd(&ctl->marks[0], 1ull);
            if (dt_ > 40000ull) { atomicAdd(&ctl->marks[7], 1ull); atomicAdd(&ctl->prof[13], (unsigned long long)a.n_transfers);
                                  atomicAdd(&ctl->prof[14], dt_); }
            atomicAdd(&ctl->prof[12], (unsigned long long)a.n_transfers);
            atomicMax(&ctl->prof[15], dt_); }
#endif
          SM_PROF(4)   // step
          // hand-off first: the map writes are all the successors of this step wait for
          a.flush();
          if (MULTI) {
            // only particles within two bins of a strip edge can have touched a peer's records or be
            // polled from another rank: they release at system scope, the interior ones at gpu scope
            const int xlo = c.rank * c.strip_w, xhi = xlo + c.strip_w;
            const bool edge = (ix < xlo + 32 && c.rank > 0) || (ix >= xhi - 32 && c.rank < c.nranks - 1);
            if (edge) st_release_sys_u32(&c.done[pid], r == SM_ALIVE ? tag : 0xFFFFFFFFu);
            else st_release_u32(&c.done[pid], r == SM_ALIVE ? tag : 0xFFFFFFFFu);
          } else {
#ifdef SM_ACQREL
            st_release_u32(&c.done[pid], r == SM_ALIVE ? tag : 0xFFFFFFFFu);
#else
            __threadfence();
            st_volatile_u32(&c.done[pid], r == SM_ALIVE ? tag : 0xFFFFFFFFu);
#endif
          }
          SM_PROF(6)   // write-back + release fence + publish
          // own state and next sweep's bins are only needed after the grid barrier
          if (r == SM_ALIVE) {
            n_steps++;
            const int jx = (int)roundf(p.px), jy = (int)roundf(p.py);
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
              c.peer[nq].alive[pid] = 1;
              c.alive[pid] = 0;
            } else {
              store_particle(c, pid, p);
            }
            bin_insert<KIND, MULTI>(c, tag + 1u, pid, jx, jy, particle_reach(p), nq);
            my_alive++;
          } else {
            store_particle(c, pid, p);
            c.alive[pid] = 0;
            if (r == SM_EXIT_OOB) n_oob++;
            else if (r == SM_EXIT_STALL) n_stall++;
            else { n_steps++; n_evap++; }
          }
          SM_PROF(5)   // state store + bin insert
          pending = false;
        }
        __syncwarp();
      }
    }
    if (my_alive) atomicAdd(&s_alive, my_alive);
    __syncthreads();
    if (threadIdx.x == 0) {
      if (s_alive) atomicAdd(&ctl->alive_slot[(s + 1) % 3], s_alive);
      s_alive = 0;
    }
    if (MULTI) total_alive = grid_barrier_multi(c, epoch, gbase, (unsigned int)((s + 1) % 3));
    else grid_barrier(&ctl->barrier, epoch);
    SM_PROF(7)   // grid barrier
  }
  if (leader && slot < n) SM_PROF_FLUSH(ctl)

  // ---- epilogue ----
  if (n_steps) atomicAdd(&ctl->steps, n_steps);
  if (n_oob) atomicAdd(&ctl->exit_oob, n_oob);
  if (n_evap) atomicAdd(&ctl->exit_evap, n_evap);
  if (n_stall) atomicAdd(&ctl->exit_stall, n_stall);
  // tag_base was read by every block before its first barrier; barrier/alive_slot are reset by the
  // host before the next launch
  if (any_doa) atomicMax(&ctl->sweeps, 1ull);
  if (gtid == 0) {
    atomicMax(&ctl->sweeps, (unsigned long long)s);
    ctl->alive = total_alive;
    ctl->tag_base = tag0 + (unsigned int)s + 2u;
    if (MULTI) ctl->epoch_base = gbase + epoch;
  }
}

// ---------------------------------------------------------------------------------------------
// k_run_exact: water batches with EXACT footprints (single rank).
//
// k_run orders two steps whenever their conservative boxes (ipos +- 3) overlap.  The cells a water step
// really touches are F = plus(ipos) U 3x3(npos) - about 14 of the 49 - but npos is only known after
// move().  Here the step is split: a particle publishes mv = npos right after move(), its map writes
// with fin, and a lower-index particle B only holds A back
//   before A.move()     if B's writes W_B = {ipos_B} U 3x3(npos_B) can meet plus(ipos_A)
//                       (while B has not moved yet: if B's box can meet plus(ipos_A)),
//   before A.interact() if F_B can meet F_A (while B has not moved yet: if B's box can meet F_A).
// The oracle emulation of this rule halves the longest chain per sweep (32.7 -> 16.1 at config-3
// density).  Particles with more than KX in-range lower-index neighbours fall back to the per-bin
// predecessor rule of k_run; to keep that rule sound every particle publishes `done` only after its
// own-bin predecessor's `done` (so "X done => every lower index in X's bin done" still holds), while
// exact waiters look at `fin`.
#define SM_KX 128            // in-range lower-index neighbours tracked exactly (ids in shared memory)
#define SM_KXW (SM_KX / 64)
#include "sm_foot.cuh"
template <int KIND> struct MidType { typedef WaterMid T; };
template <> struct MidType<KIND_WIND> { typedef WindMid T; };
template <class A> __device__ __forceinline__ int do_move(A& a, WaterP& p, WaterMid& m) { return water_move(a, p, m); }
template <class A> __device__ __forceinline__ int do_move(A& a, WindP& p, WindMid& m) { return wind_move(a, p, m); }
template <class A> __device__ __forceinline__ int do_interact(A& a, WaterP& p, const WaterMid& m) { return water_interact(a, p, m); }
template <class A> __device__ __forceinline__ int do_interact(A& a, WindP& p, const WindMid& m) { return wind_interact(a, p, m); }

#include "sm_sweep.cuh"
#include "sm_hydro_coop.cuh"

template <int KIND>
__global__ void __launch_bounds__(SM_BLOCK, SM_MINBLOCKS) k_run_exact(DevCtx c, int n, const float* __restrict__ spawn,
                                                                      int max_sweeps, int lshift) {
  typedef typename PType<KIND>::T P;
  typedef typename MidType<KIND>::T Mid;
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  __shared__ unsigned int s_alive;
  extern __shared__ __align__(32) unsigned char s_win[];   // per slot: window, then KX ids, then KX packed ipos
  for (int i = threadIdx.x; i < c.nsoils; i += blockDim.x) s_soils[i] = c.soils[i];
  if (threadIdx.x == 0) s_alive = 0;
  __syncthreads();
  const size_t slot_bytes = SM_WIN_BYTES + SM_KX * sizeof(uint32_t);
  unsigned char* my_smem = s_win + (size_t)(threadIdx.x >> lshift) * slot_bytes;
  Sec32* my_win = (Sec32*)my_smem;
  uint32_t* blk = (uint32_t*)(my_smem + SM_WIN_BYTES);

  RunCtl* ctl = c.ctl;
  unsigned int epoch = 0;
  const unsigned int tag0 = ctl->tag_base;
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const bool leader = (gtid & ((1 << lshift) - 1)) == 0;
  const int slot = gtid >> lshift;
  const int nslots = (gridDim.x * blockDim.x) >> lshift;
  const int trips = (n + nslots - 1) / nslots;
  const int G = Reach<KIND>::G;
  const int nbx = (c.dimx + G - 1) / G, nby = (c.dimy + G - 1) / G;

  unsigned long long n_steps = 0, n_oob = 0, n_evap = 0, n_stall = 0;
  bool any_doa = false;

  // ---- prologue ----
  {
    unsigned int my_alive = 0;
    if (leader) {
      for (int pid = slot; pid < n; pid += nslots) {
        bool alive;
        if (spawn != nullptr) {
          const float x = spawn[2 * pid], y = spawn[2 * pid + 1];
          const uint32_t contains = s_soils[rec_surface(c.top[(size_t)(int)roundf(x) * c.dimy + (int)roundf(y)])].transports;
          if (KIND == KIND_WATER) {
            WaterP w{x, y, 0.0f, 0.0f, 1.0, 0.0, contains};
            store_particle(c, pid, w);
            alive = true;
          } else {
            WindP w{x, y, -2.0f, 0.0f, 1.0f, 0.0, 0.0, contains};
            store_particle(c, pid, w);
            alive = !(s_soils[contains].suspension == 0.0);     // wind.h:56-57
            if (!alive) { n_oob++; any_doa = true; }
          }
          c.alive[pid] = alive ? 1 : 0;
          c.done[pid] = alive ? (tag0 - 1u) : 0xFFFFFFFFu;
          c.fin[pid] = alive ? (tag0 - 1u) : 0xFFFFFFFFu;
        } else {
          alive = c.alive[pid] != 0;
        }
        if (alive) {
          P q;
          load_particle(c, pid, q);
          bin_insert<KIND, false>(c, tag0, pid, (int)roundf(q.px), (int)roundf(q.py), particle_reach(q));
          my_alive++;
        }
      }
    }
    if (my_alive) atomicAdd(&s_alive, my_alive);
    __syncthreads();
    if (threadIdx.x == 0) {
      if (s_alive) atomicAdd(&ctl->alive_slot[0], s_alive);
      s_alive = 0;
    }
    grid_barrier(&ctl->barrier, epoch);
  }

  int s = 0;
  unsigned int total_alive = 0;
  for (;; s++) {
    const unsigned int tag = tag0 + (unsigned int)s;
    const unsigned int par = tag & 1u;
    total_alive = ld_volatile_u32(&ctl->alive_slot[s % 3]);
    if (total_alive == 0 || (max_sweeps >= 0 && s >= max_sweeps)) break;
    if (gtid == 0) st_volatile_u32(&ctl->alive_slot[(s + 2) % 3], 0u);

    unsigned int my_alive = 0;
    for (int trip = 0; trip < trips; trip++) {
      const int pid = slot + trip * nslots;
      const bool has = leader && pid < n && c.alive[pid] != 0;
      P p;
      Mid mid;
      WinAccess<KIND, false> a(c, s_soils, tag, my_win);
      int ix = 0, iy = 0, nx = 0, ny = 0, nl = 0, myR = 0;
      uint32_t ownpred = SM_NIL;          // largest lower index in my own bin
      uint32_t pred[9];                   // crowded fallback: per-bin predecessors
      unsigned long long un0[SM_KXW], un1[SM_KXW];   // exact mode: unresolved list entries for move / interact
#pragma unroll
      for (int w = 0; w < SM_KXW; w++) { un0[w] = 0; un1[w] = 0; }
      unsigned int pm = 0;                // crowded mode: per-bin predecessors not yet `done`
      bool crowded = false;
      int stage = 3;                      // 0 wait-to-move, 1 wait-to-interact, 2 wait-to-publish-done, 3 complete
      int result = SM_ALIVE;
      if (has) {
        load_particle(c, pid, p);
        ix = (int)roundf(p.px); iy = (int)roundf(p.py);
        myR = particle_reach(p);
        stage = 0;
        // ---- scan: in-range lower indices (exact list) and per-bin predecessors (fallback) ----
        const int bx = ix / G, by = iy / G;
#pragma unroll
        for (int k = 0; k < 9; k++) {
          pred[k] = SM_NIL;
          const int cx = bx + k / 3 - 1, cy = by + k % 3 - 1;
          if (cx < 0 || cx >= nbx || cy < 0 || cy >= nby) continue;
          const unsigned long long h = *((volatile unsigned long long*)&c.head[par][cx * nby + cy]);
          if ((unsigned int)(h >> 32) != tag) continue;
          uint32_t j = (uint32_t)h, best = SM_NIL;
          while (j != SM_NIL) {
            const uint2 nd = c.node[par][j];
            if (j < (uint32_t)pid) {
              if (best == SM_NIL || j > best) best = j;
              const int jx = (int)(nd.y >> 18), jy = (int)((nd.y >> 4) & 0x3FFFu);
              const int jR = (int)(nd.y & 0xFu);
              if (Foot<KIND>::in_range(jx - ix, jy - iy, myR, jR)) {
                if (nl < SM_KX) {
                  blk[nl] = j;
                  // static pruning: a neighbour whose box cannot meet plus(ipos) never delays the move
                  const bool m0 = Foot<KIND>::box_hits_M(jx - ix, jy - iy, jR);
#pragma unroll
                  for (int w = 0; w < SM_KXW; w++) {
                    if ((nl >> 6) == w) { un1[w] |= 1ull << (nl & 63); if (m0) un0[w] |= 1ull << (nl & 63); }
                  }
                  nl++;
                } else crowded = true;
              }
            }
            j = nd.x;
          }
          pred[k] = best;
        }
        ownpred = pred[4];
        if (crowded) {
#pragma unroll
          for (int k = 0; k < 9; k++) if (pred[k] != SM_NIL) pm |= 1u << k;
        }
      }

      for (;;) {
        // ---- readiness of this lane's next stage ----
        bool ready = false;
        if (stage == 0) {
          if (crowded) {
#pragma unroll
            for (int k = 0; k < 9; k++)
              if (((pm >> k) & 1u) && ld_acquire_u32(&c.done[pred[k]]) >= tag) pm &= ~(1u << k);
            ready = (pm == 0);
          } else {
            bool all0 = true;
#pragma unroll
            for (int w = 0; w < SM_KXW; w++) {
              unsigned long long m = un0[w];
              while (m) {
                const int b = __ffsll((long long)m) - 1; m &= m - 1;
                const uint32_t j = blk[w * 64 + b];
                if (ld_acquire_u32(&c.fin[j]) >= tag) { un0[w] &= ~(1ull << b); un1[w] &= ~(1ull << b); continue; }
                const unsigned long long v = *((volatile unsigned long long*)&c.mv[j]);
                if ((unsigned int)(v >> 32) == tag) {
                  const uint32_t xy = c.node[par][j].y;
                  const int jx = (int)(xy >> 18), jy = (int)((xy >> 4) & 0x3FFFu);
                  const int mx = (int)((v >> 16) & 0xFFFFu), my = (int)(v & 0xFFFFu);
                  // what B writes against plus(ipos_A)
                  const bool hit = Foot<KIND>::W_hits_M(jx, jy, mx, my, ix, iy);
                  if (!hit) un0[w] &= ~(1ull << b);
                }
              }
              if (un0[w]) all0 = false;
            }
            ready = all0;
          }
        } else if (stage == 1) {
          if (crowded) ready = true;
          else {
            bool all1 = true;
#pragma unroll
            for (int w = 0; w < SM_KXW; w++) {
              unsigned long long m = un1[w];
              while (m) {
                const int b = __ffsll((long long)m) - 1; m &= m - 1;
                const uint32_t j = blk[w * 64 + b];
                if (ld_acquire_u32(&c.fin[j]) >= tag) { un1[w] &= ~(1ull << b); continue; }
                const uint32_t xy = c.node[par][j].y;
                const int jx = (int)(xy >> 18), jy = (int)((xy >> 4) & 0x3FFFu);
                const unsigned long long v = *((volatile unsigned long long*)&c.mv[j]);
                bool hit;
                if ((unsigned int)(v >> 32) == tag) {
                  const int mx = (int)((v >> 16) & 0xFFFFu), my = (int)(v & 0xFFFFu);
                  hit = Foot<KIND>::F_hits_F(ix, iy, nx, ny, jx, jy, mx, my);
                } else {
                  // B has not moved yet: its footprint lies in ipos_B +- R_B
                  hit = Foot<KIND>::box_hits_F(ix, iy, nx, ny, jx, jy, (int)(xy & 0xFu));
                }
                if (!hit) un1[w] &= ~(1ull << b);
              }
              if (un1[w]) all1 = false;
            }
            ready = all1;
          }
        } else if (stage == 2) {
          ready = (ownpred == SM_NIL) || (ld_acquire_u32(&c.done[ownpred]) >= tag);
        }
        if (__ballot_sync(0xffffffffu, stage != 3) == 0u) break;
        if (__ballot_sync(0xffffffffu, ready) == 0u) { __nanosleep(32); continue; }

        // ---- move ----
        if (stage == 0 && ready) {
          result = do_move(a, p, mid);
          if (result == SM_ALIVE) {
            nx = (int)roundf(p.px); ny = (int)roundf(p.py);
            *((volatile unsigned long long*)&c.mv[pid]) = ((unsigned long long)tag << 32) | ((unsigned long long)nx << 16) | (unsigned long long)ny;
            if (iabs_(nx - ix) > myR - Reach<KIND>::RING || iabs_(ny - iy) > myR - Reach<KIND>::RING)
              atomicOr(&ctl->err, 1u << 4);   // SM_ERR_REACH
            stage = 1;
          } else {
            // stalled or left the map: only track[] was written
            st_release_u32(&c.fin[pid], 0xFFFFFFFFu);
            store_particle(c, pid, p);
            c.alive[pid] = 0;
            if (result == SM_EXIT_STALL) n_stall++; else n_oob++;
            stage = 2;
          }
          ready = false;
        }
        __syncwarp();
        // ---- interact ----
        if (stage == 1 && ready) {
          result = do_interact(a, p, mid);
          a.flush();
          st_release_u32(&c.fin[pid], result == SM_ALIVE ? tag : 0xFFFFFFFFu);
          store_particle(c, pid, p);
          n_steps++;
          if (result == SM_ALIVE) {
            bin_insert<KIND, false>(c, tag + 1u, pid, nx, ny, particle_reach(p));
            my_alive++;
          } else {
            c.alive[pid] = 0;
            n_evap++;
          }
          stage = 2;
          ready = false;
        }
        __syncwarp();
        // ---- publish `done` in own-bin index order ----
        if (stage == 2 && ready) {
          st_release_u32(&c.done[pid], result == SM_ALIVE ? tag : 0xFFFFFFFFu);
          stage = 3;
        }
        __syncwarp();
      }
    }
    if (my_alive) atomicAdd(&s_alive, my_alive);
    __syncthreads();
    if (threadIdx.x == 0) {
      if (s_alive) atomicAdd(&ctl->alive_slot[(s + 1) % 3], s_alive);
      s_alive = 0;
    }
    grid_barrier(&ctl->barrier, epoch);
  }

  if (n_steps) atomicAdd(&ctl->steps, n_steps);
  if (n_oob) atomicAdd(&ctl->exit_oob, n_oob);
  if (n_evap) atomicAdd(&ctl->exit_evap, n_evap);
  if (n_stall) atomicAdd(&ctl->exit_stall, n_stall);
  if (any_doa) atomicMax(&ctl->sweeps, 1ull);
  if (gtid == 0) {
    atomicMax(&ctl->sweeps, (unsigned long long)s);
    ctl->alive = total_alive;
    ctl->tag_base = tag0 + (unsigned int)s + 2u;
  }
}

// ---------------------------------------------------------------------------------------------
// full-grid and utility kernels
// ---------------------------------------------------------------------------------------------
// mapfrequency + resetfrequency, water.h:353-365 (one fused pass: 16 B per cell)
__global__ void k_frequency_update(float* __restrict__ freq, float* __restrict__ track, size_t n) {
  const float lrate = 0.01f, K = 50.0f;
  // 16-byte vectors over the bulk (cudaMalloc'd arrays are 256-byte aligned), scalars over the tail
  const size_t n4 = n / 4;
  float4* f4 = (float4*)freq;
  float4* t4 = (float4*)track;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    const float4 t = t4[i];
    float4 f = f4[i];
    f.x = (1.0f - lrate) * f.x + lrate * K * t.x / (1.0f + K * t.x);
    f.y = (1.0f - lrate) * f.y + lrate * K * t.y / (1.0f + K * t.y);
    f.z = (1.0f - lrate) * f.z + lrate * K * t.z / (1.0f + K * t.z);
    f.w = (1.0f - lrate) * f.w + lrate * K * t.w / (1.0f + K * t.w);
    f4[i] = f;
    t4[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  }
  for (size_t i = n4 * 4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float t = track[i];
    freq[i] = (1.0f - lrate) * freq[i] + lrate * K * t / (1.0f + K * t);
    track[i] = 0.0f;
  }
}

__global__ void k_heights(const Sec32* __restrict__ top, double* __restrict__ out, int32_t* __restrict__ surf,
                          size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const Sec32 r = top[i];
    if (out) out[i] = rec_height(r);
    if (surf) surf[i] = (int32_t)rec_surface(r);
  }
}

// deterministic sum: fixed chunking, fixed in-block tree; second pass sums the partials in order
#define SUM_BLOCKS 1024
__global__ void k_height_sum1(const Sec32* __restrict__ top, size_t n, double* __restrict__ partial) {
  __shared__ double sh[256];
  const size_t chunk = (n + SUM_BLOCKS - 1) / SUM_BLOCKS;
  const size_t lo = (size_t)blockIdx.x * chunk, hi = (lo + chunk < n) ? lo + chunk : n;
  double acc = 0.0;
  for (size_t i = lo + threadIdx.x; i < hi; i += 256) acc += rec_height(top[i]);
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s2 = 128; s2 > 0; s2 >>= 1) {
    if (threadIdx.x < s2) sh[threadIdx.x] += sh[threadIdx.x + s2];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = sh[0];
}
__global__ void k_height_sum2(const double* __restrict__ partial, double* __restrict__ out) {
  __shared__ double sh[SUM_BLOCKS];
  for (int i = threadIdx.x; i < SUM_BLOCKS; i += blockDim.x) sh[i] = partial[i];
  __syncthreads();
  for (int s2 = SUM_BLOCKS / 2; s2 > 0; s2 >>= 1) {
    for (int i = threadIdx.x; i < s2; i += blockDim.x) sh[i] += sh[i + s2];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sh[0];
}

// Position-sensitive checksum of every section of every column of this rank's strip (parity evidence for runs
// too large to download: equal checksums on 1, 2, 4, 8 GPUs, equal to the oracle's columns hashed by
// soilmachine_b200/checksum.py).  Each section contributes mix(cell, depth from the top, size, floor,
// saturation, type); contributions are summed modulo 2^64, so the sum over the strips of a sharded map is the
// checksum of the whole map and the order of summation does not matter.
__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {   // splitmix64 finaliser
  z ^= z >> 30; z *= 0xbf58476d1ce4e5b9ull;
  z ^= z >> 27; z *= 0x94d049bb133111ebull;
  z ^= z >> 31;
  return z;
}
__device__ __forceinline__ unsigned long long section_hash(unsigned long long cell, unsigned int depth, const Sec32& r) {
  unsigned long long h = mix64(cell * 0x9e3779b97f4a7c15ull + depth);
  h = mix64(h ^ (unsigned long long)__double_as_longlong(r.size));
  h = mix64(h ^ (unsigned long long)__double_as_longlong(r.floor));
  h = mix64(h ^ (unsigned long long)__double_as_longlong(r.saturation));
  return mix64(h ^ (unsigned long long)r.type);
}
__global__ void __launch_bounds__(256) k_checksum(DevCtx c, unsigned long long* __restrict__ out) {
  __shared__ unsigned long long sh[256];
  const int x0 = c.rank * c.strip_w;
  const int x1 = (x0 + c.strip_w < c.dimx) ? x0 + c.strip_w : c.dimx;
  const size_t cells = (size_t)(x1 - x0) * c.dimy;
  const unsigned long long base = (unsigned long long)x0 * c.dimy;        // global index of this strip's first cell
  unsigned long long acc = 0;
  for (size_t cell = (size_t)blockIdx.x * blockDim.x + threadIdx.x; cell < cells; cell += (size_t)gridDim.x * blockDim.x) {
    Sec32 r = c.top[cell];
    if (r.type == SM_EMPTY) continue;
    unsigned int depth = 0;
    for (;;) {
      acc += section_hash(base + cell, depth++, r);
      if (r.below == SM_NIL) break;
      r = c.pool[r.below];
    }
  }
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s2 = 128; s2 > 0; s2 >>= 1) {
    if (threadIdx.x < s2) sh[threadIdx.x] += sh[threadIdx.x + s2];
    __syncthreads();
  }
  if (threadIdx.x == 0) atomicAdd(out, sh[0]);
}

// Layermap::initialize, layermap.h:163-216: one thread per cell replays add() for every layer
#define SM_MAX_LAYERS 16
struct LayerSet { LayerDev L[SM_MAX_LAYERS]; int zslice[SM_MAX_LAYERS]; int n; };
__global__ void k_initialize(DevCtx c, LayerSet ls) {
  DevAccess a(c, nullptr, 0u);
  const int x0 = c.rank * c.strip_w;
  const int x1 = (x0 + c.strip_w < c.dimx) ? x0 + c.strip_w : c.dimx;
  const size_t cells = (size_t)(x1 - x0) * c.dimy;                 // this rank's strip
  for (size_t cell = (size_t)blockIdx.x * blockDim.x + threadIdx.x; cell < cells;
       cell += (size_t)gridDim.x * blockDim.x) {
    const int i = x0 + (int)(cell / c.dimy), j = (int)(cell % c.dimy);
    Sec32 r;
    rec_set_empty(r);
    for (int l = 0; l < ls.n; l++) {
      const double h = layer_value(ls.L[l], i, j, ls.zslice[l], c.dimx, c.dimy);
      col_add(a, r, h, ls.L[l].type);
    }
    c.top[cell] = r;
  }
}

// Layermap::update(ivec2, Vertexpool&), layermap.h:475-549, for every cell: the mesh the renderer and
// the PNG exporters read.  HBM-bound: per cell one 32-byte top record (+4 neighbours, L2-resident rows)
// in, one 44-byte vertex out.
struct MeshMap {   // read-only accessor for map_normal(): heights through the read-only (nc) path
  const DevCtx& c;
  struct H { double size, floor; uint32_t type; };
  __device__ __forceinline__ int dimx() const { return c.dimx; }
  __device__ __forceinline__ int dimy() const { return c.dimy; }
  __device__ __forceinline__ int scale() const { return c.scale; }
};
__device__ __forceinline__ Sec32 ldg_rec(const Sec32* p) {
  const double2 a = __ldg((const double2*)p);
  const double2 b = __ldg(((const double2*)p) + 1);
  Sec32 r;
  r.size = a.x; r.floor = a.y; r.saturation = b.x;
  const unsigned long long w = (unsigned long long)__double_as_longlong(b.y);
  r.type = (uint32_t)w; r.below = (uint32_t)(w >> 32);
  return r;
}
struct MeshAccess {   // adapts MeshMap to the accessor interface map_normal() expects
  const DevCtx& c;
  Sec32 tmp;
  __device__ __forceinline__ int dimx() const { return c.dimx; }
  __device__ __forceinline__ int dimy() const { return c.dimy; }
  __device__ __forceinline__ int scale() const { return c.scale; }
  __device__ __forceinline__ const Sec32* rec(int x, int y) { tmp = ldg_rec(&c.top[(size_t)x * c.dimy + y]); return &tmp; }
  __device__ __forceinline__ double height(int x, int y) { return rec_height(*rec(x, y)); }
};
#define MESH_BLOCK 256
__global__ void __launch_bounds__(MESH_BLOCK) k_mesh(DevCtx c, int slice, const float4* __restrict__ colors,
                                                     float* __restrict__ verts) {
  __shared__ __align__(16) float s_v[MESH_BLOCK * 11];   // staged so the 44-byte vertices leave as 16-byte rows
  const size_t cells = (size_t)c.dimx * c.dimy;
  const float plane = (float)slice / (float)c.scale;             // (float)SLICE/(float)SCALE
  for (size_t base = (size_t)blockIdx.x * MESH_BLOCK; base < cells; base += (size_t)gridDim.x * MESH_BLOCK) {
    const size_t cell = base + threadIdx.x;
    if (cell < cells) {
      const int x = (int)(cell / c.dimy), y = (int)(cell % c.dimy);
      Sec32 r = ldg_rec(&c.top[cell]);
      bool none = (r.type == SM_EMPTY);
      while (!none && r.floor > plane) {                            // :478-479 walk down to the slice plane
        if (r.below == SM_NIL) none = true;
        else r = ldg_rec(&c.pool[r.below]);
      }
      float px = (float)x, py, pz = (float)y, nx = 0.f, ny = 1.f, nz = 0.f;
      float4 col;
      int index;
      if (none) {                                                   // :481-488
        py = 0.f; col = colors[0]; index = 0;
      } else if (r.floor + r.size > plane) {                        // :490-510 cut by the plane
        py = (float)slice;
        if (r.floor + r.size * r.saturation > plane) {
          const float4 a = colors[0], b = colors[r.type];
          col = make_float4((float)((double)a.x * (1.0 - 0.6) + (double)b.x * 0.6), (float)((double)a.y * (1.0 - 0.6) + (double)b.y * 0.6),
                            (float)((double)a.z * (1.0 - 0.6) + (double)b.z * 0.6), (float)((double)a.w * (1.0 - 0.6) + (double)b.w * 0.6));
          index = 0;
        } else { col = colors[r.type]; index = (int)r.type; }
      } else {                                                      // :512-530 the surface itself
        py = (float)(c.scale * (r.floor + r.size));
        MeshAccess m{c, Sec32{}};
        const sm_f3 n = map_normal(m, x, y);
        nx = n.x; ny = n.y; nz = n.z;
        col = colors[r.type]; index = (int)r.type;
      }
      float* v = s_v + threadIdx.x * 11;
      v[0] = px; v[1] = py; v[2] = pz; v[3] = nx; v[4] = ny; v[5] = nz;
      v[6] = col.x; v[7] = col.y; v[8] = col.z; v[9] = col.w; v[10] = (float)index;
    }
    __syncthreads();
    const size_t nvalid = (cells - base < MESH_BLOCK) ? (cells - base) : MESH_BLOCK;
    const size_t nfl = nvalid * 11;
    float* dst = verts + base * 11;                                 // base*44 bytes: 16-byte aligned (MESH_BLOCK*44 % 16 == 0)
    for (size_t i = threadIdx.x * 4; i < nfl; i += MESH_BLOCK * 4) {
      if (i + 4 <= nfl) *((float4*)(dst + i)) = *((const float4*)(s_v + i));
      else for (size_t k = i; k < nfl; k++) dst[k] = s_v[k];
    }
    __syncthreads();
  }
}
// exportheight / exportcolor, io.h:234-252
__global__ void k_export(const float* __restrict__ verts, size_t cells, int scale, float* __restrict__ height,
                         float* __restrict__ bgra) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (size_t)gridDim.x * blockDim.x) {
    const float* v = verts + i * 11;
    if (height) height[i] = (float)(v[1] / scale / sqrt(2.0));
    if (bgra) { bgra[4 * i] = v[8]; bgra[4 * i + 1] = v[7]; bgra[4 * i + 2] = v[6]; bgra[4 * i + 3] = 1.0f; }
  }
}

// single-cell operations for the facade's legacy Layermap calls: op 0 add, 1 remove, 2 cascade,
// 3 query (height, surface, normal), 4 bilinear height
struct CellOp { int op; int x, y; float fx, fy; double v; int t; };
struct CellRes { double d; int32_t surface; float n[3]; };
__global__ void k_cell_op(DevCtx c, CellOp o, CellRes* res) {
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  for (int i = 0; i < c.nsoils; i++) s_soils[i] = c.soils[i];
  DevAccess a(c, s_soils, 0u);
  CellRes r{0.0, 0, {0.f, 0.f, 0.f}};
  if (o.op == 0) col_add(a, *a.rec(o.x, o.y), o.v, (uint32_t)o.t);
  else if (o.op == 1) r.d = col_remove(a, *a.rec(o.x, o.y), o.v);
  else if (o.op == 2) Cascade<3, DevAccess>::run(a, (int)roundf(o.fx), (int)roundf(o.fy), o.t);
  else if (o.op == 3) {
    r.d = map_height(a, o.x, o.y);
    r.surface = (int32_t)rec_surface(*a.rec(o.x, o.y));
    sm_f3 n = map_normal(a, o.x, o.y);
    r.n[0] = n.x; r.n[1] = n.y; r.n[2] = n.z;
  } else if (o.op == 4) r.d = map_height_bilinear(a, o.fx, o.fy);
  else if (o.op == 5) hydro_seep_cell(a, o.x, o.y);                 // WaterParticle::seep(vec2,...), water.h:285-333
  else if (o.op == 6) {                                             // WaterParticle::cascade(vec2,...,spill), water.h:151-283
    HydroCount hc{};
    WFrame st[SM_WSTACK];
    int sp = 0;
    hydro_push(a, st, sp, o.x, o.y, o.t, hc);
    hydro_drain(a, st, sp, hc);
  }
  *res = r;
}
// one whole column, bottom -> top, for the facade's Layermap::top(ivec2) (layermap.h:150-152)
__global__ void k_cell_column(DevCtx c, int x, int y, int cap, int* n_out, Sec32* out) {
  Sec32 r = c.top[(size_t)x * c.dimy + y];
  int n = 0;
  if (r.type != SM_EMPTY) {
    for (;;) {
      if (n < cap) out[n] = r;
      n++;
      if (r.below == SM_NIL) break;
      r = c.pool[r.below];
    }
  }
  *n_out = n;       // top first; the host reverses
}


// ---------------------------------------------------------------------------------------------
// pooling hydrology (sm_hydro.cuh): flood phase and the per-frame seep pass
// ---------------------------------------------------------------------------------------------
// Both are sequential by definition: the flood of particle i sees the map the floods of all
// lower-indexed particles left behind, nested particles included (water.h:123-145,252-256), and the seep
// pass visits the cells in x-major order with the same nesting (water.h:335-343).  One thread executes them;
// what the device adds is (a) a full-grid classification that reduces the 16.8 M-cell scan of the seep pass
// to the few cells where water is, and (b) a software-managed record cache in shared memory, because the
// executor works on a handful of neighbouring cells over and over and a shared-memory hit costs a tenth of
// an L2 round trip.
//
// The cache is direct-mapped on (x mod 64, y mod 64): all cells of any 64 x 64 window have distinct lines,
// and the core never holds record pointers that are further apart than one particle step (a few cells), so
// a pointer handed out by rec() cannot be evicted while it is in use.  Lines are written back when they are
// replaced and when the kernel ends.  Buried sections (pool) and the frequency maps are accessed in place.
#define SM_HC_EDGE 64
#define SM_HC_LINES (SM_HC_EDGE * SM_HC_EDGE)
#define SM_HC_FREE 256    // private free list of pool slots (the executor is the only thread touching the pool)
#define SM_HC_BYTES (SM_HC_LINES * (int)sizeof(Sec32) + SM_HC_LINES * 8 + SM_HC_FREE * 4)

struct HydroAccess : DevAccess {
  Sec32* s_rec;          // SM_HC_LINES records
  uint32_t* s_tag;       // cell index held by each line, SM_NIL = none
  uint32_t* s_mark;      // cell whose 3x3 block this line last flagged in the active index (marks are never cleared)
  uint32_t* s_free;      // pool slots freed by this kernel, reused before the shared rings are touched
  int nfree;
  ActiveMap act;
  bool marking;
  __device__ __forceinline__ HydroAccess(const DevCtx& ctx, const SoilDev* ss, Sec32* sr, uint32_t* st, const ActiveMap& am, bool mk)
      : DevAccess(ctx, ss, 0u), s_rec(sr), s_tag(st), s_mark(st + SM_HC_LINES), s_free(st + 2 * SM_HC_LINES), nfree(0),
        act(am), marking(mk) {}
  __device__ __forceinline__ uint32_t pool_alloc() {
    if (nfree > 0) return s_free[--nfree];
    return DevAccess::pool_alloc();
  }
  __device__ __forceinline__ void pool_free(uint32_t i) {
    if (nfree < SM_HC_FREE) s_free[nfree++] = i;
    else DevAccess::pool_free(i);
  }
  __device__ __forceinline__ Sec32* rec(int x, int y) {
    const uint32_t cell = (uint32_t)x * (uint32_t)c.dimy + (uint32_t)y;
    const int line = (x & (SM_HC_EDGE - 1)) * SM_HC_EDGE + (y & (SM_HC_EDGE - 1));
    const uint32_t held = s_tag[line];
    if (held != cell) {
      if (held != SM_NIL) c.top[held] = s_rec[line];
      s_rec[line] = c.top[cell];
      s_tag[line] = cell;
    }
    return &s_rec[line];
  }
  __device__ __forceinline__ double height(int x, int y) { return rec_height(*rec(x, y)); }
  __device__ __forceinline__ uint32_t surface_of(int x, int y) { return rec_surface(*rec(x, y)); }
  __device__ __forceinline__ void query(int x, int y, double& h, uint32_t& t) { const Sec32* r = rec(x, y); h = rec_height(*r); t = rec_surface(*r); }
  __device__ __forceinline__ void dirty_rec(Sec32* r, int x, int y) {
    if (marking && r->type == SM_AIR) {
      const int line = (int)(r - s_rec);             // r always comes from rec()
      const uint32_t cell = s_tag[line];
      if (s_mark[line] != cell) {
        active_mark_block(act, x, y, c.dimx, c.dimy);
        s_mark[line] = cell;
      }
    }
  }
  __device__ __forceinline__ void dirty(int x, int y) { dirty_rec(rec(x, y), x, y); }
  __device__ __forceinline__ void wet_mark(int x, int y) {
    if (marking) active_set(act, (unsigned long long)x * c.dimy + y);
  }
  __device__ void flush() {
    for (int line = 0; line < SM_HC_LINES; line++) {
      const uint32_t held = s_tag[line];
      if (held != SM_NIL) c.top[held] = s_rec[line];
    }
    while (nfree > 0) DevAccess::pool_free(s_free[--nfree]);
  }
};

__device__ __forceinline__ void hydro_smem_init(unsigned char* smem, Sec32*& s_rec, uint32_t*& s_tag, SoilDev* s_soils, const DevCtx& c) {
  s_rec = reinterpret_cast<Sec32*>(smem);
  s_tag = reinterpret_cast<uint32_t*>(smem + SM_HC_LINES * sizeof(Sec32));
  for (int i = threadIdx.x; i < 2 * SM_HC_LINES; i += blockDim.x) s_tag[i] = SM_NIL;   // tags and marks
  for (int i = threadIdx.x; i < c.nsoils; i += blockDim.x) s_soils[i] = c.soils[i];
  __syncthreads();
}
__device__ __forceinline__ void hydro_count_out(HydroCount* out, const HydroCount& hc) {
  out->floods = hc.floods; out->nested = hc.nested; out->nested_steps = hc.nested_steps;
  out->transfers = hc.transfers; out->cells = hc.cells; out->overflow = hc.overflow;
}

// flood() of every finished particle of the last water batch, ascending index (SoilMachine.cpp:292-296).
// The warp scans the batch 32 particles at a time; lane 0 executes the floods the ballot found.
__global__ void __launch_bounds__(32) k_hydro_flood(DevCtx c, int n, HydroCount* out) {
  extern __shared__ __align__(32) unsigned char hy_smem[];
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  Sec32* s_rec; uint32_t* s_tag;
  hydro_smem_init(hy_smem, s_rec, s_tag, s_soils, c);
  ActiveMap none{};
  HydroAccess a(c, s_soils, s_rec, s_tag, none, false);
  HydroCount hc{};
  const int lane = threadIdx.x;
  for (int base = 0; base < n; base += 32) {
    const int i = base + lane;
    bool cand = false;
    // a particle floods exactly once (upstream: flood() ends the particle): flooded ones carry a marker
    // in their `done` word, so a repeated call or flood -> more sweeps -> flood never deposits twice
    if (i < n) cand = (c.alive[i] == 0) && !(c.pb[i].x < SM_MINVOL) && c.done[i] != SM_DONE_FLOODED;
    unsigned int m = __ballot_sync(0xFFFFFFFFu, cand);
    if (lane == 0) {
      while (m) {
        const int j = base + __ffs((int)m) - 1;
        m &= m - 1u;
        const float4 pa = c.pa[j];
        const double2 pb = c.pb[j];
        WaterP p;
        p.px = pa.x; p.py = pa.y; p.sx = pa.z; p.sy = pa.w;
        p.volume = pb.x; p.sediment = pb.y; p.contains = c.pc[j].x;
        hydro_flood_particle(a, p, hc);
        c.done[j] = SM_DONE_FLOODED;
      }
    }
    __syncwarp();
  }
  if (lane == 0) { a.flush(); hydro_count_out(out, hc); }
}

// full-grid classification for the seep pass: flag the cells whose visit can change anything
__device__ __forceinline__ void active_set_atomic(const ActiveMap& m, unsigned long long idx) {
  for (int l = 0; l < m.nlevels; l++) {
    const unsigned long long w = idx >> 6, b = 1ull << (idx & 63);
    const unsigned long long old = atomicOr(&m.lvl[l][w], b);
    if (old) return;                 // bit already set, or the word already announced one level up
    idx = w;
  }
}
__global__ void __launch_bounds__(256) k_hydro_classify(DevCtx c, ActiveMap am) {
  const unsigned long long cells = am.ncells;
  for (unsigned long long cell = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; cell < cells;
       cell += (unsigned long long)gridDim.x * blockDim.x) {
    const Sec32 r = c.top[cell];
    if (r.type == SM_EMPTY) continue;
    const int x = (int)(cell / (unsigned long long)c.dimy), y = (int)(cell % (unsigned long long)c.dimy);
    if (r.type == SM_AIR) {
      for (int dx = -1; dx <= 1; dx++) {
        const int xx = x + dx;
        if (xx < 0 || xx >= c.dimx) continue;
        for (int dy = -1; dy <= 1; dy++) {
          const int yy = y + dy;
          if (yy < 0 || yy >= c.dimy) continue;
          active_set_atomic(am, (unsigned long long)xx * c.dimy + yy);
        }
      }
    }
    bool holds = (r.saturation != 0.0);
    for (uint32_t b = r.below; !holds && b != SM_NIL;) {
      const Sec32 s = c.pool[b];
      holds = (s.saturation != 0.0);
      b = s.below;
    }
    if (holds) active_set_atomic(am, cell);
  }
}
// WaterParticle::seep(map, vertexpool), water.h:335-343, over the flagged cells in x-major order
__global__ void __launch_bounds__(32) k_hydro_seep(DevCtx c, ActiveMap am, HydroCount* out) {
  extern __shared__ __align__(32) unsigned char hy_smem[];
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  Sec32* s_rec; uint32_t* s_tag;
  hydro_smem_init(hy_smem, s_rec, s_tag, s_soils, c);
  if (threadIdx.x != 0) return;
  HydroAccess a(c, s_soils, s_rec, s_tag, am, true);
  HydroCount hc{};
  const unsigned long long cells = am.ncells;
  for (unsigned long long cell = active_next(am, 0); cell < cells; cell = active_next(am, cell + 1))
    hydro_seep_visit(a, (int)(cell / (unsigned long long)c.dimy), (int)(cell % (unsigned long long)c.dimy), hc);
  a.flush();
  hydro_count_out(out, hc);
}

// ---- the same two phases executed by one WARP (sm_hydro_coop.cuh): frames evaluated eight neighbours at a time,
// nested particles on the cooperative step.  Records are accessed in place through L2 (a frame's nine records are
// fetched by nine lanes at once, which is what the one-thread executor needs its shared-memory cache for).
struct HydroBack : DevBack<false, false> {
  static constexpr bool kHydroHooks = true;
  ActiveMap act;
  bool marking;
  __device__ __forceinline__ HydroBack(const DevCtx& ctx, const SoilDev* ss, const ActiveMap& am, bool mk)
      : DevBack<false, false>(ctx, ss, 0u), act(am), marking(mk) {}
  // single writer: only the lane that mutates columns calls these
  __device__ __forceinline__ void air_mark(Sec32* r, int x, int y) {
    if (marking && r->type == SM_AIR) active_mark_block(act, x, y, c.dimx, c.dimy);
  }
  __device__ __forceinline__ void wet_mark(int x, int y) {
    if (marking) active_set(act, (unsigned long long)x * c.dimy + y);
  }
};
__global__ void __launch_bounds__(32) k_hydro_flood_w(DevCtx c, int n, HydroCount* out) {
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  __shared__ CoopScratch sc;
  __shared__ HydroScratch hx;
  const int lane = threadIdx.x;
  for (int i = lane; i < c.nsoils; i += 32) s_soils[i] = c.soils[i];
  __syncwarp();
  WarpDev w{lane};
  ActiveMap none{};
  HydroBack back(c, s_soils, none, false);
  CoopWin<HydroBack> a(back, &sc);
  HydroCount hc{};
  for (int base = 0; base < n; base += 32) {
    const int i = base + lane;
    bool cand = false;
    if (i < n) cand = (c.alive[i] == 0) && !(c.pb[i].x < SM_MINVOL) && c.done[i] != SM_DONE_FLOODED;
    unsigned int m = __ballot_sync(0xFFFFFFFFu, cand);
    while (m) {                                   // warp-uniform
      const int j = base + __ffs((int)m) - 1;
      m &= m - 1u;
      const float4 pa = c.pa[j];
      const double2 pb = c.pb[j];
      WaterP p;
      p.px = pa.x; p.py = pa.y; p.sx = pa.z; p.sy = pa.w;
      p.volume = pb.x; p.sediment = pb.y; p.contains = c.pc[j].x;
      hydro_flood_particle_coop(w, a, &hx, p, hc);
      if (lane == 0) c.done[j] = SM_DONE_FLOODED;
      __syncwarp();
    }
  }
  if (lane == 0) hydro_count_out(out, hc);
}
__global__ void __launch_bounds__(32) k_hydro_seep_w(DevCtx c, ActiveMap am, HydroCount* out) {
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  __shared__ CoopScratch sc;
  __shared__ HydroScratch hx;
  const int lane = threadIdx.x;
  for (int i = lane; i < c.nsoils; i += 32) s_soils[i] = c.soils[i];
  __syncwarp();
  WarpDev w{lane};
  HydroBack back(c, s_soils, am, true);
  CoopWin<HydroBack> a(back, &sc);
  HydroCount hc{};
  const unsigned long long cells = am.ncells;
  for (unsigned long long cell = active_next(am, 0); cell < cells; cell = active_next(am, cell + 1)) {
    hydro_seep_visit_coop(w, a, &hx, (int)(cell / (unsigned long long)c.dimy), (int)(cell % (unsigned long long)c.dimy), hc);
    __syncwarp();
  }
  if (lane == 0) hydro_count_out(out, hc);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
struct sm_context {
  sm_config cfg;
  DevCtx d;
  std::string err;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, evt0 = nullptr, evt1 = nullptr;
  size_t cells = 0;        // cells of the whole map (frequency arrays, bins)
  size_t lcells = 0;       // cells of this rank's x-strip (top records); == cells when not sharded
  int nranks = 1, rank = 0, x0 = 0, x1 = 0, share = 1;
  bool peers_attached = false;
  void* ipc_opened[SM_MAX_RANKS][SM_PEER_SLOTS] = {};
  int max_particles = 0;
  int nsoils = 0;
  SoilDev* d_soils = nullptr;
  float* d_spawn = nullptr;
  double* d_scratch = nullptr;    // height download / partial sums
  int32_t* d_iscratch = nullptr;
  CellRes* d_cellres = nullptr;
  float* d_verts = nullptr;       // 11 floats per cell, allocated on first sm_mesh_update
  float4* d_colors = nullptr;
  bool mesh_valid = false;
  unsigned long long* d_act = nullptr;   // active-cell index of the seep pass (allocated on first use)
  unsigned long long act_words = 0;
  HydroCount* d_hydro = nullptr;
  LbmDev lbm = {};                // wind field (sm_lbm_create)
  int lbm_cur = 0;                // buffer holding the current populations
  RunCtl* h_ctl = nullptr;        // pinned
  int64_t launches = 0;
  int cur_kind = -1, cur_n = 0;
  bool timing_pending = false;
  int num_sms = 0;
};

static std::string g_create_err;

#define CK(call)                                                                          \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                      \
      return SM_ERR_CUDA;                                                                 \
    }                                                                                     \
  } while (0)

static int fail(sm_context* ctx, int code, const char* msg) {
  ctx->err = msg;
  return code;
}

static void host_soil_to_dev(const sm_soil& s, SoilDev& d) {
  d.friction = s.friction; d.solubility = s.solubility; d.equrate = s.equrate;
  d.erosionrate = s.erosionrate; d.maxdiff = s.maxdiff; d.settling = s.settling;
  d.suspension = s.suspension; d.porosity = s.porosity;
  d.transports = (uint32_t)s.transports; d.erodes = (uint32_t)s.erodes;
  d.cascades = (uint32_t)s.cascades; d.abrades = (uint32_t)s.abrades;
}

extern "C" {

const char* sm_last_error(const sm_context* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

void sm_destroy(sm_context* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->cfg.device);
  cudaDeviceSynchronize();
  for (int q = 0; q < SM_MAX_RANKS; q++) for (int i = 0; i < SM_PEER_SLOTS; i++) if (ctx->ipc_opened[q][i]) cudaIpcCloseMemHandle(ctx->ipc_opened[q][i]);
  DevCtx& d = ctx->d;
  cudaFree(d.top); cudaFree(d.pool); cudaFree(d.ringbuf[0]); cudaFree(d.ringbuf[1]); cudaFree(d.ringbuf[2]);
  cudaFree(d.wfreq); cudaFree(d.wtrack); cudaFree(d.windfreq); cudaFree(ctx->d_soils);
  cudaFree(d.ctl); cudaFree(d.pa); cudaFree(d.pb); cudaFree(d.pc); cudaFree(d.alive); cudaFree(d.done); cudaFree(d.fin); cudaFree(d.mv); cudaFree(d.bud);
  for (int i = 0; i < 3; i++) cudaFree(d.lmask[i]);
  for (int i = 0; i < 2; i++) { cudaFree(d.head[i]); cudaFree(d.node[i]); }
  cudaFree(ctx->d_verts); cudaFree(ctx->d_colors); cudaFree(d.dbg);
  cudaFree(ctx->d_act); cudaFree(ctx->d_hydro);
  cudaFree(ctx->lbm.F[0]); cudaFree(ctx->lbm.F[1]); cudaFree(ctx->lbm.B); cudaFree(ctx->lbm.RHO); cudaFree(ctx->lbm.V);
  cudaFree(ctx->d_spawn); cudaFree(ctx->d_scratch); cudaFree(ctx->d_iscratch); cudaFree(ctx->d_cellres);
  if (ctx->h_ctl) cudaFreeHost(ctx->h_ctl);
  if (ctx->ev0) cudaEventDestroy(ctx->ev0);
  if (ctx->ev1) cudaEventDestroy(ctx->ev1);
  if (ctx->evt0) cudaEventDestroy(ctx->evt0);
  if (ctx->evt1) cudaEventDestroy(ctx->evt1);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

static int alloc_pool(sm_context* ctx, unsigned long long cap) {
  DevCtx& d = ctx->d;
  if (d.pool && d.pool_cap >= cap) return SM_OK;
  if (d.pool && ctx->nranks > 1) return fail(ctx, SM_ERR_POOL, "sharded context: pool_capacity is fixed at creation and too small");
  cudaFree(d.pool); cudaFree(d.ringbuf[0]); cudaFree(d.ringbuf[1]); cudaFree(d.ringbuf[2]);
  d.pool = nullptr; d.ringbuf[0] = d.ringbuf[1] = d.ringbuf[2] = nullptr;
  CK(cudaMalloc(&d.pool, cap * sizeof(Sec32)));
  CK(cudaMalloc(&d.ringbuf[0], cap * sizeof(uint32_t)));
  CK(cudaMalloc(&d.ringbuf[1], cap * sizeof(uint32_t)));
  CK(cudaMalloc(&d.ringbuf[2], cap * sizeof(uint32_t)));
  d.pool_cap = cap;
  return SM_OK;
}

static int create_impl(const sm_config* cfg, int nranks, int rank, int share, sm_context** out) {
  if (!cfg || !out || cfg->dimx < 2 || cfg->dimy < 2 || cfg->dimx > 16384 || cfg->dimy > 16384 ||
      nranks < 1 || nranks > SM_MAX_RANKS || rank < 0 || rank >= nranks || share < 1) {
    g_create_err = "sm_create: invalid configuration";
    return SM_ERR_INVALID;
  }
  // x-strips of equal width (a multiple of the largest bin edge, 16 cells)
  const int strip_w = (nranks == 1) ? cfg->dimx : ((((cfg->dimx + nranks - 1) / nranks) + 15) / 16) * 16;
  const int sx0 = rank * strip_w, sx1 = std::min(cfg->dimx, sx0 + strip_w);
  if (sx1 <= sx0) {
    g_create_err = "sm_create_sharded: the map is too narrow for this many ranks (needs >= 16 columns per rank)";
    return SM_ERR_INVALID;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    g_create_err = "sm_create: no CUDA device (this library has no CPU fallback)";
    return SM_ERR_NOGPU;
  }
  sm_context* ctx = new sm_context();
  ctx->cfg = *cfg;
  memset(&ctx->d, 0, sizeof(DevCtx));
  int rc = [&]() -> int {
    CK(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, cfg->device));
    ctx->num_sms = prop.multiProcessorCount;
    CK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    CK(cudaEventCreate(&ctx->ev0));
    CK(cudaEventCreate(&ctx->ev1));
    CK(cudaEventCreate(&ctx->evt0));
    CK(cudaEventCreate(&ctx->evt1));
    DevCtx& d = ctx->d;
    d.dimx = cfg->dimx; d.dimy = cfg->dimy; d.scale = cfg->scale;
    d.volume_factor = SM_VOLUME_FACTOR;
    ctx->cells = (size_t)cfg->dimx * cfg->dimy;
    ctx->nranks = nranks; ctx->rank = rank; ctx->share = share; ctx->x0 = sx0; ctx->x1 = sx1;
    ctx->lcells = (size_t)(sx1 - sx0) * cfg->dimy;
    d.nranks = nranks; d.rank = rank; d.strip_w = strip_w;
    ctx->max_particles = cfg->max_particles > 0 ? cfg->max_particles : 262144;
    const size_t C = ctx->cells, N = (size_t)ctx->max_particles;
    const size_t LC = ctx->lcells;
    CK(cudaMalloc(&d.top, LC * sizeof(Sec32)));
    CK(cudaMalloc(&d.wfreq, C * 4)); CK(cudaMalloc(&d.wtrack, C * 4)); CK(cudaMalloc(&d.windfreq, C * 4));
    CK(cudaMemsetAsync(d.wfreq, 0, C * 4, ctx->stream));
    CK(cudaMemsetAsync(d.wtrack, 0, C * 4, ctx->stream));
    CK(cudaMemsetAsync(d.windfreq, 0, C * 4, ctx->stream));
    CK(cudaMalloc(&ctx->d_soils, SM_MAX_SOILS * sizeof(SoilDev)));
    d.soils = ctx->d_soils;
    CK(cudaMalloc(&d.ctl, sizeof(RunCtl)));
    CK(cudaMemsetAsync(d.ctl, 0, sizeof(RunCtl), ctx->stream));
    CK(cudaMalloc(&d.pa, N * sizeof(float4))); CK(cudaMalloc(&d.pb, N * sizeof(double2)));
    CK(cudaMalloc(&d.pc, N * sizeof(uint2))); CK(cudaMalloc(&d.alive, N)); CK(cudaMalloc(&d.done, N * 4));
    CK(cudaMalloc(&d.fin, N * 4)); CK(cudaMalloc(&d.mv, N * 8));
    for (int i = 0; i < 3; i++) {
      CK(cudaMalloc(&d.lmask[i], (N / 32 + 2) * sizeof(unsigned int)));
      CK(cudaMemsetAsync(d.lmask[i], 0, (N / 32 + 2) * sizeof(unsigned int), ctx->stream));
    }
    if (cfg->flags & SM_FLAG_BUDGET) {
      CK(cudaMalloc(&d.bud, N * SM_BUDGET_SLOTS * sizeof(double)));
      CK(cudaMemsetAsync(d.bud, 0, N * SM_BUDGET_SLOTS * sizeof(double), ctx->stream));
    }
    CK(cudaMemsetAsync(d.fin, 0, N * 4, ctx->stream)); CK(cudaMemsetAsync(d.mv, 0, N * 8, ctx->stream));
    d.nbx = (cfg->dimx + SM_MIN_BIN - 1) / SM_MIN_BIN; d.nby = (cfg->dimy + SM_MIN_BIN - 1) / SM_MIN_BIN;
    for (int i = 0; i < 2; i++) {
      CK(cudaMalloc(&d.head[i], (size_t)d.nbx * d.nby * 8));
      CK(cudaMemsetAsync(d.head[i], 0, (size_t)d.nbx * d.nby * 8, ctx->stream));
      CK(cudaMalloc(&d.node[i], N * sizeof(uint2)));
    }
    CK(cudaMalloc(&ctx->d_spawn, N * 8));
    CK(cudaMalloc(&ctx->d_scratch, std::max(C, (size_t)SUM_BLOCKS + 8) * 8));
    CK(cudaMalloc(&ctx->d_iscratch, C * 4));
    CK(cudaMalloc(&ctx->d_cellres, sizeof(CellRes)));
    CK(cudaMalloc(&d.dbg, 8 * 16384 * sizeof(unsigned long long)));
    CK(cudaMemsetAsync(d.dbg, 0, 8 * 16384 * sizeof(unsigned long long), ctx->stream));
    CK(cudaMallocHost(&ctx->h_ctl, sizeof(RunCtl)));
    // tags start at 1 so that zero-initialised bin heads never match
    RunCtl init; memset(&init, 0, sizeof(init)); init.tag_base = 2;
    CK(cudaMemcpyAsync(d.ctl, &init, sizeof(RunCtl), cudaMemcpyHostToDevice, ctx->stream));
    // empty terrain
    {
      std::vector<Sec32> empty(LC);
      for (auto& r : empty) rec_set_empty(r);
      CK(cudaMemcpyAsync(d.top, empty.data(), LC * sizeof(Sec32), cudaMemcpyHostToDevice, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
    }
    // sharded contexts export their pool to the peers, so it is sized once and never re-allocated
    int rcp = alloc_pool(ctx, cfg->pool_capacity > 0 ? (unsigned long long)cfg->pool_capacity
                                                     : (unsigned long long)LC * (nranks > 1 ? 2 : 1) + (4ull << 20));
    if (rcp != SM_OK) return rcp;
    CK(cudaFuncSetAttribute(k_run<KIND_WATER, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_BLOCK * SM_WIN_BYTES));
    CK(cudaFuncSetAttribute(k_run<KIND_WIND, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_BLOCK * SM_WIN_BYTES));
    CK(cudaFuncSetAttribute(k_run<KIND_WATER, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_BLOCK * SM_WIN_BYTES));
    CK(cudaFuncSetAttribute(k_run_exact<KIND_WATER>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_BLOCK * (SM_WIN_BYTES + SM_KX * 4)));
    CK(cudaFuncSetAttribute(k_run_exact<KIND_WIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_BLOCK * (SM_WIN_BYTES + SM_KX * 4)));
    CK(cudaFuncSetAttribute(k_run<KIND_WIND, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_BLOCK * SM_WIN_BYTES));
    CK(cudaStreamSynchronize(ctx->stream));
    return SM_OK;
  }();
  if (rc != SM_OK) {
    g_create_err = ctx->err;
    sm_destroy(ctx);
    return rc;
  }
  *out = ctx;
  return SM_OK;
}

int sm_create(const sm_config* cfg, sm_context** out) { return create_impl(cfg, 1, 0, 1, out); }
int sm_create_sharded(const sm_config* cfg, int32_t nranks, int32_t rank, int32_t share, sm_context** out) {
  return create_impl(cfg, nranks, rank, share, out);
}
int sm_shard_range(sm_context* ctx, int32_t* x0, int32_t* x1) {
  if (x0) *x0 = ctx->x0;
  if (x1) *x1 = ctx->x1;
  return SM_OK;
}

// ---- peers of a sharded map ----------------------------------------------------------------------------
static void own_ptrs(sm_context* ctx, void** p) {
  DevCtx& d = ctx->d;
  p[0] = d.top; p[1] = d.pool; p[2] = d.ringbuf[0]; p[3] = d.ringbuf[1]; p[4] = d.ctl; p[5] = d.pa; p[6] = d.pb;
  p[7] = d.pc; p[8] = d.alive; p[9] = d.done; p[10] = d.head[0]; p[11] = d.head[1]; p[12] = d.node[0]; p[13] = d.node[1];
  p[14] = d.ringbuf[2]; p[15] = d.bud; p[16] = d.fin; p[17] = d.lmask[0]; p[18] = d.lmask[1]; p[19] = d.lmask[2];
}
static void fill_peer(PeerPtrs& P, void* const* p, unsigned long long pool_cap) {
  P.top = (Sec32*)p[0]; P.pool = (Sec32*)p[1]; P.ringbuf[0] = (uint32_t*)p[2]; P.ringbuf[1] = (uint32_t*)p[3];
  P.ctl = (RunCtl*)p[4]; P.pa = (float4*)p[5]; P.pb = (double2*)p[6]; P.pc = (uint2*)p[7];
  P.alive = (unsigned char*)p[8]; P.done = (unsigned int*)p[9]; P.head[0] = (unsigned long long*)p[10];
  P.head[1] = (unsigned long long*)p[11]; P.node[0] = (uint2*)p[12]; P.node[1] = (uint2*)p[13];
  P.ringbuf[2] = (uint32_t*)p[14]; P.bud = (double*)p[15]; P.fin = (unsigned int*)p[16];
  P.lmask[0] = (unsigned int*)p[17]; P.lmask[1] = (unsigned int*)p[18]; P.lmask[2] = (unsigned int*)p[19];
  P.pool_cap = pool_cap;
}
int sm_peer_export(sm_context* ctx, sm_peer_blob* out) {
  if (!out) return fail(ctx, SM_ERR_INVALID, "null blob");
  CK(cudaSetDevice(ctx->cfg.device));
  memset(out, 0, sizeof(*out));
  void* p[SM_PEER_SLOTS] = {};
  own_ptrs(ctx, p);
  for (int i = 0; i < SM_PEER_ARRAYS; i++) {
    out->ptr[i] = (uint64_t)(uintptr_t)p[i];
    if (!p[i]) continue;                      // optional array (mass budget) not allocated
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, p[i]));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(out->ipc[i], &h, 64);
  }
  out->pool_cap = ctx->d.pool_cap;
  out->rank = ctx->rank;
  out->device = ctx->cfg.device;
  return SM_OK;
}
int sm_peer_attach(sm_context* ctx, const sm_peer_blob* blobs, int32_t nblobs, int32_t use_ipc) {
  if (!blobs || nblobs != ctx->nranks) return fail(ctx, SM_ERR_INVALID, "sm_peer_attach: one blob per rank");
  CK(cudaSetDevice(ctx->cfg.device));
  for (int q = 0; q < ctx->nranks; q++) {
    const sm_peer_blob& b = blobs[q];
    if (b.rank != q) return fail(ctx, SM_ERR_INVALID, "sm_peer_attach: blobs must be ordered by rank");
    void* p[SM_PEER_SLOTS] = {};
    if (q == ctx->rank) {
      own_ptrs(ctx, p);
    } else if (!use_ipc) {
      for (int i = 0; i < SM_PEER_ARRAYS; i++) p[i] = (void*)(uintptr_t)b.ptr[i];   // same process
    } else {
      if (b.device != ctx->cfg.device) {
        int can = 0;
        CK(cudaDeviceCanAccessPeer(&can, ctx->cfg.device, b.device));
        if (!can) return fail(ctx, SM_ERR_CUDA, "sm_peer_attach: no peer access between the devices");
        cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { ctx->err = cudaGetErrorString(e); return SM_ERR_CUDA; }
        cudaGetLastError();
      }
      for (int i = 0; i < SM_PEER_ARRAYS; i++) {
        if (!b.ptr[i]) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, b.ipc[i], 64);
        CK(cudaIpcOpenMemHandle(&p[i], h, cudaIpcMemLazyEnablePeerAccess));
        ctx->ipc_opened[q][i] = p[i];
      }
    }
    fill_peer(ctx->d.peer[q], p, b.pool_cap);
  }
  ctx->peers_attached = true;
  return SM_OK;
}

int sm_sync(sm_context* ctx) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

int sm_set_soils(sm_context* ctx, const sm_soil* soils, int32_t n) {
  if (!soils || n < 1 || n > SM_MAX_SOILS) return fail(ctx, SM_ERR_INVALID, "sm_set_soils: 1..64 soils");
  for (int i = 0; i < n; i++) {
    const sm_soil& s = soils[i];
    if (s.transports < 0 || s.transports >= n || s.erodes < 0 || s.erodes >= n || s.cascades < 0 ||
        s.cascades >= n || s.abrades < 0 || s.abrades >= n)
      return fail(ctx, SM_ERR_INVALID, "sm_set_soils: soil reference out of range");
  }
  std::vector<SoilDev> dev(n);
  for (int i = 0; i < n; i++) host_soil_to_dev(soils[i], dev[i]);
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaMemcpyAsync(ctx->d_soils, dev.data(), n * sizeof(SoilDev), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->nsoils = n;
  ctx->d.nsoils = n;
  return SM_OK;
}

// ---- columns --------------------------------------------------------------------------------
namespace {
struct HostBuild {  // accessor used to replay add() on the host while building the upload image
  std::vector<Sec32>* pool;
  Sec32 pool_load(uint32_t i) { return (*pool)[i]; }
  void pool_store(uint32_t i, const Sec32& r) { (*pool)[i] = r; }
  uint32_t pool_alloc() { pool->push_back(Sec32{}); return (uint32_t)(pool->size() - 1); }
  void pool_free(uint32_t) {}
};
}  // namespace

static int reset_pool_ctl(sm_context* ctx, unsigned long long used) {
  // bump = used, rings empty
  CK(cudaStreamSynchronize(ctx->stream));
  RunCtl h;
  CK(cudaMemcpy(&h, ctx->d.ctl, sizeof(RunCtl), cudaMemcpyDeviceToHost));
  h.bump = used;
  h.ring[0].head = h.ring[0].tail = 0;
  h.ring[1].head = h.ring[1].tail = 0;
  h.ring[2].head = h.ring[2].tail = 0;
  h.err = 0; h.drops = 0;
  CK(cudaMemcpy(ctx->d.ctl, &h, sizeof(RunCtl), cudaMemcpyHostToDevice));
  return SM_OK;
}

int sm_upload_columns(sm_context* ctx, const int64_t* offsets, const int32_t* type, const double* size,
                      const double* saturation) {
  if (!offsets || !type || !size) return fail(ctx, SM_ERR_INVALID, "sm_upload_columns: null argument");
  CK(cudaSetDevice(ctx->cfg.device));
  const size_t C = ctx->lcells;   // CSR of this rank's strip, cell order (x - x0)*dimy + y
  std::vector<Sec32> top(C), pool;
  pool.reserve((size_t)std::max<int64_t>(0, offsets[C] - (int64_t)C) + 16);
  HostBuild hb{&pool};
  for (size_t c = 0; c < C; c++) {
    rec_set_empty(top[c]);
    for (int64_t k = offsets[c]; k < offsets[c + 1]; k++) {
      if (type[k] < 0 || (ctx->nsoils > 0 && type[k] >= ctx->nsoils))
        return fail(ctx, SM_ERR_INVALID, "sm_upload_columns: section type out of range");
      col_add(hb, top[c], size[k], (uint32_t)type[k], saturation ? saturation[k] : 0.0);
    }
  }
  const unsigned long long need = pool.size();
  if (ctx->cfg.pool_capacity > 0) {
    if (need > ctx->d.pool_cap) return fail(ctx, SM_ERR_POOL, "sm_upload_columns: pool_capacity too small");
  } else {
    int rc = alloc_pool(ctx, ctx->nranks > 1 ? need : need + (unsigned long long)C + (4ull << 20));
    if (rc != SM_OK) return rc;
  }
  CK(cudaMemcpy(ctx->d.top, top.data(), C * sizeof(Sec32), cudaMemcpyHostToDevice));
  if (need) CK(cudaMemcpy(ctx->d.pool, pool.data(), need * sizeof(Sec32), cudaMemcpyHostToDevice));
  return reset_pool_ctl(ctx, need);
}

static int fetch_image(sm_context* ctx, std::vector<Sec32>& top, std::vector<Sec32>& pool) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  RunCtl h;
  CK(cudaMemcpy(&h, ctx->d.ctl, sizeof(RunCtl), cudaMemcpyDeviceToHost));
  const size_t used = (size_t)std::min<unsigned long long>(h.bump, ctx->d.pool_cap);
  top.resize(ctx->lcells);
  pool.resize(used);
  CK(cudaMemcpy(top.data(), ctx->d.top, ctx->lcells * sizeof(Sec32), cudaMemcpyDeviceToHost));
  if (used) CK(cudaMemcpy(pool.data(), ctx->d.pool, used * sizeof(Sec32), cudaMemcpyDeviceToHost));
  return SM_OK;
}

int sm_section_count(sm_context* ctx, int64_t* n) {
  std::vector<Sec32> top, pool;
  int rc = fetch_image(ctx, top, pool);
  if (rc != SM_OK) return rc;
  int64_t cnt = 0;
  for (const Sec32& r : top) {
    if (r.type == SM_EMPTY) continue;
    cnt++;
    for (uint32_t b = r.below; b != SM_NIL; b = pool[b].below) cnt++;
  }
  *n = cnt;
  return SM_OK;
}

int sm_download_columns(sm_context* ctx, int64_t capacity, int64_t* offsets, int32_t* type, double* size,
                        double* floor_, double* saturation) {
  std::vector<Sec32> top, pool;
  int rc = fetch_image(ctx, top, pool);
  if (rc != SM_OK) return rc;
  int64_t n = 0;
  std::vector<const Sec32*> st;
  for (size_t c = 0; c < top.size(); c++) {
    offsets[c] = n;
    st.clear();
    const Sec32& r = top[c];
    if (r.type != SM_EMPTY) {
      st.push_back(&r);
      for (uint32_t b = r.below; b != SM_NIL; b = pool[b].below) {
        if (b >= pool.size()) return fail(ctx, SM_ERR_INVALID, "sm_download_columns: corrupt chain");
        st.push_back(&pool[b]);
      }
    }
    if (n + (int64_t)st.size() > capacity) return fail(ctx, SM_ERR_INVALID, "sm_download_columns: capacity");
    for (size_t i = st.size(); i-- > 0;) {
      if (type) type[n] = (int32_t)st[i]->type;
      if (size) size[n] = st[i]->size;
      if (floor_) floor_[n] = st[i]->floor;
      if (saturation) saturation[n] = st[i]->saturation;
      n++;
    }
  }
  offsets[top.size()] = n;
  return SM_OK;
}

int sm_download_height(sm_context* ctx, double* height) {
  CK(cudaSetDevice(ctx->cfg.device));
  k_heights<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d.top, ctx->d_scratch, nullptr, ctx->lcells);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(height, ctx->d_scratch, ctx->lcells * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

int sm_download_surface(sm_context* ctx, int32_t* surface) {
  CK(cudaSetDevice(ctx->cfg.device));
  k_heights<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d.top, nullptr, ctx->d_iscratch, ctx->lcells);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(surface, ctx->d_iscratch, ctx->lcells * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

int sm_height_sum(sm_context* ctx, double* sum) {
  CK(cudaSetDevice(ctx->cfg.device));
  k_height_sum1<<<SUM_BLOCKS, 256, 0, ctx->stream>>>(ctx->d.top, ctx->lcells, ctx->d_scratch);
  k_height_sum2<<<1, 256, 0, ctx->stream>>>(ctx->d_scratch, ctx->d_scratch + SUM_BLOCKS);
  ctx->launches += 2;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(sum, ctx->d_scratch + SUM_BLOCKS, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

int sm_checksum(sm_context* ctx, uint64_t* out) {
  if (!out) return fail(ctx, SM_ERR_INVALID, "null argument");
  CK(cudaSetDevice(ctx->cfg.device));
  unsigned long long* d_out = (unsigned long long*)(ctx->d_scratch + SUM_BLOCKS + 1);
  CK(cudaMemsetAsync(d_out, 0, 8, ctx->stream));
  k_checksum<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, d_out);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, d_out, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

int sm_get_frequency(sm_context* ctx, float* wf, float* wt, float* windf) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  if (wf) CK(cudaMemcpy(wf, ctx->d.wfreq, ctx->cells * 4, cudaMemcpyDeviceToHost));
  if (wt) CK(cudaMemcpy(wt, ctx->d.wtrack, ctx->cells * 4, cudaMemcpyDeviceToHost));
  if (windf) CK(cudaMemcpy(windf, ctx->d.windfreq, ctx->cells * 4, cudaMemcpyDeviceToHost));
  return SM_OK;
}
int sm_set_frequency(sm_context* ctx, const float* wf, const float* wt, const float* windf) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  if (wf) CK(cudaMemcpy(ctx->d.wfreq, wf, ctx->cells * 4, cudaMemcpyHostToDevice));
  if (wt) CK(cudaMemcpy(ctx->d.wtrack, wt, ctx->cells * 4, cudaMemcpyHostToDevice));
  if (windf) CK(cudaMemcpy(ctx->d.windfreq, windf, ctx->cells * 4, cudaMemcpyHostToDevice));
  return SM_OK;
}
int sm_frequency_update(sm_context* ctx) {
  CK(cudaSetDevice(ctx->cfg.device));
  k_frequency_update<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d.wfreq, ctx->d.wtrack, ctx->cells);
  ctx->launches++;
  CK(cudaGetLastError());
  return SM_OK;
}

// ---- single-cell operations -----------------------------------------------------------------------
static int cell_op(sm_context* ctx, const CellOp& o, CellRes* out) {
  if (ctx->nsoils < 1) return fail(ctx, SM_ERR_INVALID, "soil table not set");
  if (ctx->nranks > 1) return fail(ctx, SM_ERR_INVALID, "single-cell operations are not available on a sharded context");
  CK(cudaSetDevice(ctx->cfg.device));
  k_cell_op<<<1, 1, 0, ctx->stream>>>(ctx->d, o, ctx->d_cellres);
  ctx->launches++;
  CK(cudaGetLastError());
  CellRes r;
  CK(cudaMemcpyAsync(&r, ctx->d_cellres, sizeof(CellRes), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (out) *out = r;
  return SM_OK;
}
static bool inb(sm_context* ctx, int x, int y) { return x >= 0 && y >= 0 && x < ctx->d.dimx && y < ctx->d.dimy; }

int sm_cell_add(sm_context* ctx, int32_t x, int32_t y, double size, int32_t type) {
  if (!inb(ctx, x, y) || type < 0 || type >= ctx->nsoils) return fail(ctx, SM_ERR_INVALID, "sm_cell_add: range");
  return cell_op(ctx, CellOp{0, x, y, 0.f, 0.f, size, type}, nullptr);
}
int sm_cell_remove(sm_context* ctx, int32_t x, int32_t y, double h, double* leftover) {
  if (!inb(ctx, x, y)) return fail(ctx, SM_ERR_INVALID, "sm_cell_remove: range");
  CellRes r;
  int rc = cell_op(ctx, CellOp{1, x, y, 0.f, 0.f, h, 0}, &r);
  if (rc == SM_OK && leftover) *leftover = r.d;
  return rc;
}
int sm_cell_cascade(sm_context* ctx, float x, float y, int32_t transferloop) {
  if (!inb(ctx, (int)roundf(x), (int)roundf(y)) || transferloop < 0 || transferloop > 3)
    return fail(ctx, SM_ERR_INVALID, "sm_cell_cascade: range (transferloop 0..3)");
  return cell_op(ctx, CellOp{2, 0, 0, x, y, 0.0, transferloop}, nullptr);
}
int sm_cell_query(sm_context* ctx, int32_t x, int32_t y, double* height, int32_t* surface, float* normal3) {
  if (!inb(ctx, x, y)) return fail(ctx, SM_ERR_INVALID, "sm_cell_query: range");
  CellRes r;
  int rc = cell_op(ctx, CellOp{3, x, y, 0.f, 0.f, 0.0, 0}, &r);
  if (rc != SM_OK) return rc;
  if (height) *height = r.d;
  if (surface) *surface = r.surface;
  if (normal3) { normal3[0] = r.n[0]; normal3[1] = r.n[1]; normal3[2] = r.n[2]; }
  return SM_OK;
}
int sm_cell_seep(sm_context* ctx, int32_t x, int32_t y) {
  if (!inb(ctx, x, y)) return fail(ctx, SM_ERR_INVALID, "sm_cell_seep: range");
  ctx->mesh_valid = false;
  return cell_op(ctx, CellOp{5, x, y, 0.f, 0.f, 0.0, 0}, nullptr);
}
int sm_cell_water_cascade(sm_context* ctx, int32_t x, int32_t y, int32_t spill) {
  if (!inb(ctx, x, y) || spill < 0 || spill > 3) return fail(ctx, SM_ERR_INVALID, "sm_cell_water_cascade: range (spill 0..3)");
  ctx->mesh_valid = false;
  return cell_op(ctx, CellOp{6, x, y, 0.f, 0.f, 0.0, spill}, nullptr);
}
int sm_cell_column(sm_context* ctx, int32_t x, int32_t y, int32_t capacity, int32_t* n, int32_t* type, double* size,
                   double* floor_, double* saturation) {
  if (!inb(ctx, x, y) || !n || capacity < 0) return fail(ctx, SM_ERR_INVALID, "sm_cell_column: range");
  if (ctx->nranks > 1) return fail(ctx, SM_ERR_INVALID, "single-cell operations are not available on a sharded context");
  CK(cudaSetDevice(ctx->cfg.device));
  const int cap = std::min(capacity, 1024);
  Sec32* d_out = nullptr; int* d_n = nullptr;
  CK(cudaMalloc(&d_out, (size_t)std::max(cap, 1) * sizeof(Sec32)));
  if (cudaMalloc(&d_n, sizeof(int)) != cudaSuccess) { cudaFree(d_out); return fail(ctx, SM_ERR_CUDA, "cudaMalloc"); }
  k_cell_column<<<1, 1, 0, ctx->stream>>>(ctx->d, x, y, cap, d_n, d_out);
  ctx->launches++;
  std::vector<Sec32> tmp((size_t)std::max(cap, 1));
  int cnt = 0;
  cudaError_t e = cudaMemcpyAsync(&cnt, d_n, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(tmp.data(), d_out, tmp.size() * sizeof(Sec32), cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  cudaFree(d_out); cudaFree(d_n);
  if (e != cudaSuccess) { ctx->err = cudaGetErrorString(e); return SM_ERR_CUDA; }
  *n = cnt;
  const int m = std::min(cnt, cap);
  for (int i = 0; i < m; i++) {       // bottom -> top
    const Sec32& r = tmp[(size_t)(m - 1 - i)];
    if (type) type[i] = (int32_t)r.type;
    if (size) size[i] = r.size;
    if (floor_) floor_[i] = r.floor;
    if (saturation) saturation[i] = r.saturation;
  }
  return SM_OK;
}
int sm_set_volume_factor(sm_context* ctx, double v) {
  if (!(v > 0.0)) return fail(ctx, SM_ERR_INVALID, "sm_set_volume_factor: must be positive");
  ctx->d.volume_factor = v;
  return SM_OK;
}
int sm_height_bilinear(sm_context* ctx, float x, float y, double* height) {
  if (!(x >= 0.f && y >= 0.f && x < (float)(ctx->d.dimx - 1) && y < (float)(ctx->d.dimy - 1)))
    return fail(ctx, SM_ERR_INVALID, "sm_height_bilinear: range");
  CellRes r;
  int rc = cell_op(ctx, CellOp{4, 0, 0, x, y, 0.0, 0}, &r);
  if (rc == SM_OK && height) *height = r.d;
  return rc;
}

// ---- the hot path -----------------------------------------------------------------------------------
static int launch_run(sm_context* ctx, int kind, int n, const float* d_spawn, int max_sweeps) {
  if (ctx->nsoils < 1) return fail(ctx, SM_ERR_INVALID, "soil table not set");
  if (n < 0 || n > ctx->max_particles) return fail(ctx, SM_ERR_INVALID, "batch larger than max_particles");
  const bool multi = ctx->nranks > 1;
  if (multi && !ctx->peers_attached) return fail(ctx, SM_ERR_INVALID, "sharded context: call sm_peer_attach first");
  if (multi && n >= (1 << 28)) return fail(ctx, SM_ERR_INVALID, "sharded context: at most 2^28 particles");
  CK(cudaSetDevice(ctx->cfg.device));
  const int threads = SM_BLOCK;
  // lanes per particle (a power of two): only the first lane of each group carries a particle, which
  // keeps divergent particle-steps out of each other's warps and shrinks the window footprint
  int lshift = 0, blocks = 1;
  size_t smem = 0;
  {
    const char* e = getenv("SM_LANES");
    int want = e ? atoi(e) : 8;
    int ls = 0;
    while ((1 << (ls + 1)) <= want && ls < 5) ls++;
    for (;; ls--) {
      smem = (size_t)(threads >> ls) * SM_WIN_BYTES;
      int occ = 0;
      if (kind == KIND_WATER) {
        if (multi) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_run<KIND_WATER, true>, threads, smem));
        else CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_run<KIND_WATER, false>, threads, smem));
      } else {
        if (multi) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_run<KIND_WIND, true>, threads, smem));
        else CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_run<KIND_WIND, false>, threads, smem));
      }
      if (occ < 1) return fail(ctx, SM_ERR_CUDA, "sweep kernel does not fit an SM");
      // contexts that share the device must all be resident at once (they meet in the cross-rank barrier)
      const long long maxblocks = std::max<long long>(1, (long long)ctx->num_sms * occ / ctx->share);
      const long long need_threads = (long long)std::max(n, 1) << ls;
      lshift = ls;
      blocks = (int)std::min<long long>(maxblocks, (need_threads + threads - 1) / threads);
      if (need_threads <= maxblocks * threads || ls == 0) break;   // every particle has its own thread
    }
    if (blocks < 1) blocks = 1;
  }
  // single rank: exact-footprint kernel.  SM_EXACT = bit mask of kinds (1 water, 2 wind); default 1:
  // measured -16 % on the water batch of config 3
  bool use_exact = false;
  if (!multi) {
    const char* e = getenv("SM_EXACT");
    const int mask = e ? atoi(e) : 1;
    if (mask & (1 << kind)) {
      for (int ls = lshift;; ls--) {
        const size_t sm2 = (size_t)(threads >> ls) * (SM_WIN_BYTES + SM_KX * 4);
        int occ = 0;
        if (kind == KIND_WATER) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_run_exact<KIND_WATER>, threads, sm2));
        else CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_run_exact<KIND_WIND>, threads, sm2));
        const long long need_threads = (long long)std::max(n, 1) << ls;
        const long long maxblocks = (long long)ctx->num_sms * occ;
        if (occ >= 1 && (need_threads <= maxblocks * threads || ls == 0)) {
          use_exact = true; lshift = ls; smem = sm2;
          blocks = (int)std::max<long long>(1, std::min<long long>(maxblocks, (need_threads + threads - 1) / threads));
          break;
        }
        if (ls == 0) break;
      }
    }
  }
  // default: the warp-per-particle kernel (sm_sweep.cuh).  SM_KERNEL=thread selects the thread-per-particle
  // kernels above (kept for comparison measurements).
  // the mass budget and the wind-field coupling live in the warp kernel
  bool use_coop = SM_DEFAULT_COOP || ctx->d.bud != nullptr || ctx->d.wind_v4 != nullptr;
  {
    const char* e = getenv("SM_KERNEL");
    if (e && strcmp(e, "thread") == 0) use_coop = false;
    if (e && strcmp(e, "warp") == 0) use_coop = true;
  }
  if (use_coop) {
    const int cthreads = SM_SW_WARPS * 32;
    int occ = 0;
    const bool budget = ctx->d.bud != nullptr;
    // SM_EXACT: bit mask of the kinds that use exact footprints (sweep_exact): 1 = water, 2 = wind
    bool exact = false;
    {
      const char* e = getenv("SM_EXACT");
      exact = (((e ? atoi(e) : SM_DEFAULT_EXACT) >> kind) & 1) != 0;
    }
    void* const fns[16] = {(void*)k_sweep<KIND_WATER, false, false, false>, (void*)k_sweep<KIND_WIND, false, false, false>,
                           (void*)k_sweep<KIND_WATER, true, false, false>,  (void*)k_sweep<KIND_WIND, true, false, false>,
                           (void*)k_sweep<KIND_WATER, false, true, false>,  (void*)k_sweep<KIND_WIND, false, true, false>,
                           (void*)k_sweep<KIND_WATER, true, true, false>,   (void*)k_sweep<KIND_WIND, true, true, false>,
                           (void*)k_sweep<KIND_WATER, false, false, true>,  (void*)k_sweep<KIND_WIND, false, false, true>,
                           (void*)k_sweep<KIND_WATER, true, false, true>,   (void*)k_sweep<KIND_WIND, true, false, true>,
                           (void*)k_sweep<KIND_WATER, false, true, true>,   (void*)k_sweep<KIND_WIND, false, true, true>,
                           (void*)k_sweep<KIND_WATER, true, true, true>,    (void*)k_sweep<KIND_WIND, true, true, true>};
    void* fn = fns[(exact ? 8 : 0) + (budget ? 4 : 0) + (multi ? 2 : 0) + (kind == KIND_WATER ? 0 : 1)];
    // dynamic shared memory: the live mask of the batch and its popcount prefix (2 x n/32 words per block)
    const size_t csmem = (size_t)2 * (((size_t)std::max(n, 1) + 31) / 32) * sizeof(unsigned int);
    if (csmem > 40 * 1024) CK(cudaFuncSetAttribute((const void*)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)csmem));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void*)fn, cthreads, csmem));
    if (occ < 1) return fail(ctx, SM_ERR_CUDA, "sweep kernel does not fit an SM");
    // contexts that share the device must all be resident at once (they meet in the cross-rank barrier)
    const long long maxblocks = std::max<long long>(1, (long long)ctx->num_sms * occ / ctx->share);
    const long long want = ((long long)std::max(n, 1) + SM_SW_WARPS - 1) / SM_SW_WARPS;
    const int cblocks = (int)std::max<long long>(1, std::min(maxblocks, want));
    DevCtx dd = ctx->d;
    int ms = max_sweeps;
    if (ms <= 0) ms = -1;
    if (max_sweeps == SM_SWEEPS_NONE) ms = 0;
    void* cargs[] = {&dd, &n, (void*)&d_spawn, &ms};
    CK(cudaMemsetAsync(ctx->d.ctl, 0, 4 * sizeof(unsigned int), ctx->stream));  // barrier + alive_slot[3]
    CK(cudaMemsetAsync(&ctx->d.ctl->ticket[0], 0, 3 * sizeof(unsigned int), ctx->stream));
    for (int i = 0; i < 3; i++)      // the kernel's prologue sets the bits of the live particles
      CK(cudaMemsetAsync(ctx->d.lmask[i], 0, ((size_t)ctx->max_particles / 32 + 2) * sizeof(unsigned int), ctx->stream));
    CK(cudaEventRecord(ctx->ev0, ctx->stream));
    CK(cudaLaunchCooperativeKernel(fn, dim3(cblocks), dim3(cthreads), cargs, csmem, ctx->stream));
    CK(cudaEventRecord(ctx->ev1, ctx->stream));
    ctx->launches++;
    ctx->timing_pending = true;
    return SM_OK;
  }
  DevCtx d = ctx->d;
  if (max_sweeps <= 0) max_sweeps = -1;            // run until every particle is dead
  if (max_sweeps == SM_SWEEPS_NONE) max_sweeps = 0;  // prologue only (the *_begin calls)
  void* args[] = {&d, &n, (void*)&d_spawn, &max_sweeps, &lshift};
  CK(cudaMemsetAsync(ctx->d.ctl, 0, 4 * sizeof(unsigned int), ctx->stream));  // barrier + alive_slot[3]
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  if (multi && kind == KIND_WATER)
    CK(cudaLaunchCooperativeKernel((void*)k_run<KIND_WATER, true>, dim3(blocks), dim3(threads), args, smem, ctx->stream));
  else if (multi)
    CK(cudaLaunchCooperativeKernel((void*)k_run<KIND_WIND, true>, dim3(blocks), dim3(threads), args, smem, ctx->stream));
  else if (use_exact && kind == KIND_WATER)
    CK(cudaLaunchCooperativeKernel((void*)k_run_exact<KIND_WATER>, dim3(blocks), dim3(threads), args, smem, ctx->stream));
  else if (use_exact)
    CK(cudaLaunchCooperativeKernel((void*)k_run_exact<KIND_WIND>, dim3(blocks), dim3(threads), args, smem, ctx->stream));
  else if (kind == KIND_WATER)
    CK(cudaLaunchCooperativeKernel((void*)k_run<KIND_WATER, false>, dim3(blocks), dim3(threads), args, smem, ctx->stream));
  else
    CK(cudaLaunchCooperativeKernel((void*)k_run<KIND_WIND, false>, dim3(blocks), dim3(threads), args, smem, ctx->stream));
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  ctx->launches++;
  ctx->timing_pending = true;
  return SM_OK;
}

static int zero_counters(sm_context* ctx) {
  // steps..alive are contiguous in RunCtl.  The error bits are per call as well: a pool exhaustion or a reach
  // violation is reported by the call it happened in (stats.pool_drops says how many sections were dropped)
  // and does not poison later calls - upstream prints and keeps running (layermap.h:92-95).
  CK(cudaMemsetAsync(&ctx->d.ctl->steps, 0, 7 * sizeof(unsigned long long), ctx->stream));
  CK(cudaMemsetAsync(&ctx->d.ctl->err, 0, sizeof(unsigned int), ctx->stream));
  return SM_OK;
}

int sm_last_stats(sm_context* ctx, sm_stats* st) {
  CK(cudaSetDevice(ctx->cfg.device));
  // only the counters travel: barrier .. bump (SM_STATS_READBACK_BYTES, what bench.py counts as d2h per batch)
  static_assert(offsetof(RunCtl, ring) == 88, "bench.py counts 88 bytes read back per batch");
  CK(cudaMemcpyAsync(ctx->h_ctl, ctx->d.ctl, offsetof(RunCtl, ring), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  const RunCtl& h = *ctx->h_ctl;
  float ms = 0.f;
  if (ctx->timing_pending) CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
  if (st) {
    st->steps = (int64_t)h.steps; st->sweeps = (int64_t)h.sweeps; st->exit_oob = (int64_t)h.exit_oob;
    st->exit_evap = (int64_t)h.exit_evap; st->exit_stall = (int64_t)h.exit_stall;
    st->pool_drops = (int64_t)h.drops; st->alive = (int64_t)h.alive; st->device_ms = ms;
  }
  if (h.err & (1u << 4)) return fail(ctx, SM_ERR_REACH, "a particle step left its conflict box");
  if (h.err & (1u << 3)) return fail(ctx, SM_ERR_POOL, "section pool exhausted (sections were dropped)");
  return SM_OK;
}

static int run_host(sm_context* ctx, int kind, int n, const float* spawn_xy, int max_sweeps, sm_stats* st) {
  if (n > 0 && !spawn_xy) return fail(ctx, SM_ERR_INVALID, "null spawn list");
  if (ctx->nranks > 1 && ctx->share > 1)
    return fail(ctx, SM_ERR_INVALID, "contexts sharing a device must use sm_*_run_device on every rank, then sm_last_stats");
  if (n < 0 || n > ctx->max_particles) return fail(ctx, SM_ERR_INVALID, "batch larger than max_particles");
  CK(cudaSetDevice(ctx->cfg.device));
  if (n) CK(cudaMemcpyAsync(ctx->d_spawn, spawn_xy, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  int rc = zero_counters(ctx);
  if (rc != SM_OK) return rc;
  ctx->cur_kind = kind; ctx->cur_n = n;
  rc = launch_run(ctx, kind, n, ctx->d_spawn, max_sweeps);
  if (rc != SM_OK) return rc;
  return sm_last_stats(ctx, st);
}

// ---- mass budget (SURVEY.md A.7) --------------------------------------------------------------------------
int sm_budget_particles(sm_context* ctx, int32_t n, double* out) {
  if (!ctx->d.bud) return fail(ctx, SM_ERR_INVALID, "context was created without SM_FLAG_BUDGET");
  if (n < 0 || n > ctx->max_particles || (n && !out)) return fail(ctx, SM_ERR_INVALID, "sm_budget_particles: range");
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  if (n) CK(cudaMemcpy(out, ctx->d.bud, (size_t)n * SM_BUDGET_SLOTS * sizeof(double), cudaMemcpyDeviceToHost));
  return SM_OK;
}
int sm_last_budget(sm_context* ctx, sm_budget* out) {
  if (!out) return fail(ctx, SM_ERR_INVALID, "null argument");
  if (ctx->cur_n < 0) return fail(ctx, SM_ERR_INVALID, "no batch yet");
  std::vector<double> per((size_t)std::max(ctx->cur_n, 0) * SM_BUDGET_SLOTS);
  int rc = sm_budget_particles(ctx, std::max(ctx->cur_n, 0), per.data());
  if (rc != SM_OK) return rc;
  double s6[SM_BUDGET_SLOTS] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < ctx->cur_n; i++)             // particle order: the same sums on any number of SMs or ranks
    for (int k = 0; k < SM_BUDGET_SLOTS; k++) s6[k] += per[(size_t)i * SM_BUDGET_SLOTS + k];
  out->eroded = s6[0]; out->deposited = s6[1]; out->cascade_net = s6[2]; out->discarded = s6[3];
  out->clamped = s6[4]; out->wind_negative = s6[5]; out->particles = ctx->cur_n;
  return SM_OK;
}

int sm_water_run(sm_context* ctx, int32_t n, const float* xy, int32_t max_sweeps, sm_stats* st) {
  return run_host(ctx, KIND_WATER, n, xy, max_sweeps, st);
}
int sm_wind_run(sm_context* ctx, int32_t n, const float* xy, int32_t max_sweeps, sm_stats* st) {
  return run_host(ctx, KIND_WIND, n, xy, max_sweeps, st);
}
int sm_water_run_device(sm_context* ctx, int32_t n, const float* d_xy, int32_t max_sweeps) {
  int rc = zero_counters(ctx);
  if (rc != SM_OK) return rc;
  ctx->cur_kind = KIND_WATER; ctx->cur_n = n;
  return launch_run(ctx, KIND_WATER, n, d_xy, max_sweeps);
}
int sm_wind_run_device(sm_context* ctx, int32_t n, const float* d_xy, int32_t max_sweeps) {
  int rc = zero_counters(ctx);
  if (rc != SM_OK) return rc;
  ctx->cur_kind = KIND_WIND; ctx->cur_n = n;
  return launch_run(ctx, KIND_WIND, n, d_xy, max_sweeps);
}

// ---- pooling hydrology ----------------------------------------------------------------------------
// SM_HYDRO=warp | thread selects the executor of the flood phase and the seep pass
static bool hydro_warp() {
  const char* e = getenv("SM_HYDRO");
  if (e && strcmp(e, "warp") == 0) return true;
  if (e && strcmp(e, "thread") == 0) return false;
  return false;     // without a record cache the warp executor's seep pass does not keep up with the one-thread
                    // executor and its shared-memory cache
}
static int hydro_ready(sm_context* ctx) {
  if (ctx->nsoils < 1) return fail(ctx, SM_ERR_INVALID, "soil table not set");
  if (ctx->nranks > 1) return fail(ctx, SM_ERR_INVALID, "pooling hydrology is not available on a sharded context");
  CK(cudaSetDevice(ctx->cfg.device));
  if (!ctx->d_hydro) {
    CK(cudaMalloc(&ctx->d_hydro, sizeof(HydroCount)));
    CK(cudaFuncSetAttribute(k_hydro_flood, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_HC_BYTES));
    CK(cudaFuncSetAttribute(k_hydro_seep, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_HC_BYTES));
  }
  // status and drop counter are per call (see zero_counters)
  CK(cudaMemsetAsync(&ctx->d.ctl->err, 0, sizeof(unsigned int), ctx->stream));
  CK(cudaMemsetAsync(&ctx->d.ctl->drops, 0, sizeof(unsigned long long), ctx->stream));
  return SM_OK;
}
static int hydro_finish(sm_context* ctx, sm_hydro_stats* st) {
  HydroCount hc;
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(cudaMemcpyAsync(&hc, ctx->d_hydro, sizeof(hc), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
  ctx->timing_pending = false;
  ctx->mesh_valid = false;
  if (st) {
    st->floods = (int64_t)hc.floods; st->nested = (int64_t)hc.nested; st->nested_steps = (int64_t)hc.nested_steps;
    st->transfers = (int64_t)hc.transfers; st->cells = (int64_t)hc.cells; st->device_ms = ms; st->classify_ms = 0.0;
  }
  if (hc.overflow) return fail(ctx, SM_ERR_REACH, "water cascade nesting exceeded its bound");
  unsigned int err = 0;
  CK(cudaMemcpy(&err, &ctx->d.ctl->err, sizeof(err), cudaMemcpyDeviceToHost));
  if (err & (1u << 3)) return fail(ctx, SM_ERR_POOL, "section pool exhausted (sections were dropped)");
  return SM_OK;
}
int sm_water_flood(sm_context* ctx, sm_hydro_stats* st) {
  int rc = hydro_ready(ctx);
  if (rc != SM_OK) return rc;
  if (ctx->cur_kind != KIND_WATER) return fail(ctx, SM_ERR_INVALID, "sm_water_flood: the last batch was not a water batch");
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  if (hydro_warp()) k_hydro_flood_w<<<1, 32, 0, ctx->stream>>>(ctx->d, ctx->cur_n, ctx->d_hydro);
  else k_hydro_flood<<<1, 32, SM_HC_BYTES, ctx->stream>>>(ctx->d, ctx->cur_n, ctx->d_hydro);
  ctx->launches++;
  CK(cudaGetLastError());
  return hydro_finish(ctx, st);
}
int sm_seep(sm_context* ctx, sm_hydro_stats* st) {
  int rc = hydro_ready(ctx);
  if (rc != SM_OK) return rc;
  ActiveMap am{};
  am.ncells = ctx->cells;
  const unsigned long long total = active_layout(ctx->cells, am.nwords, &am.nlevels);
  if (!ctx->d_act || ctx->act_words < total) {
    cudaFree(ctx->d_act); ctx->d_act = nullptr;
    CK(cudaMalloc(&ctx->d_act, total * sizeof(unsigned long long)));
    ctx->act_words = total;
  }
  unsigned long long off = 0;
  for (int l = 0; l < am.nlevels; l++) { am.lvl[l] = ctx->d_act + off; off += am.nwords[l]; }
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  CK(cudaMemsetAsync(ctx->d_act, 0, total * sizeof(unsigned long long), ctx->stream));
  CK(cudaEventRecord(ctx->evt0, ctx->stream));
  k_hydro_classify<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, am);
  CK(cudaEventRecord(ctx->evt1, ctx->stream));
  if (hydro_warp()) k_hydro_seep_w<<<1, 32, 0, ctx->stream>>>(ctx->d, am, ctx->d_hydro);
  else k_hydro_seep<<<1, 32, SM_HC_BYTES, ctx->stream>>>(ctx->d, am, ctx->d_hydro);
  ctx->launches += 2;
  CK(cudaGetLastError());
  int rc2 = hydro_finish(ctx, st);
  if (st) {     // the full-grid classification alone (the HBM-bound part of the pass)
    float cms = 0.f;
    if (cudaEventElapsedTime(&cms, ctx->evt0, ctx->evt1) == cudaSuccess) st->classify_ms = cms;
  }
  return rc2;
}

// stepping interface: *_begin runs the prologue only (spawn + bins), *_sweeps(k) resumes the batch
int sm_water_begin(sm_context* ctx, int32_t n, const float* xy) {
  return run_host(ctx, KIND_WATER, n, xy, SM_SWEEPS_NONE, nullptr);
}
int sm_wind_begin(sm_context* ctx, int32_t n, const float* xy) {
  return run_host(ctx, KIND_WIND, n, xy, SM_SWEEPS_NONE, nullptr);
}
static int sweeps_k(sm_context* ctx, int kind, int k, sm_stats* st) {
  if (ctx->cur_kind != kind) return fail(ctx, SM_ERR_INVALID, "no batch of this kind in flight");
  if (k <= 0) return fail(ctx, SM_ERR_INVALID, "k must be positive");
  int rc = zero_counters(ctx);
  if (rc != SM_OK) return rc;
  rc = launch_run(ctx, kind, ctx->cur_n, nullptr, k);
  if (rc != SM_OK) return rc;
  return sm_last_stats(ctx, st);
}
int sm_water_sweeps(sm_context* ctx, int32_t k, sm_stats* st) { return sweeps_k(ctx, KIND_WATER, k, st); }
int sm_wind_sweeps(sm_context* ctx, int32_t k, sm_stats* st) { return sweeps_k(ctx, KIND_WIND, k, st); }

static int fetch_state(sm_context* ctx, int kind, std::vector<float4>& a, std::vector<double2>& b,
                       std::vector<uint2>& c, std::vector<unsigned char>& al) {
  if (ctx->cur_kind != kind) return fail(ctx, SM_ERR_INVALID, "no batch of this kind in flight");
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  const size_t n = (size_t)ctx->cur_n;
  a.resize(n); b.resize(n); c.resize(n); al.resize(n);
  if (!n) return SM_OK;
  CK(cudaMemcpy(a.data(), ctx->d.pa, n * sizeof(float4), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(b.data(), ctx->d.pb, n * sizeof(double2), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(c.data(), ctx->d.pc, n * sizeof(uint2), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(al.data(), ctx->d.alive, n, cudaMemcpyDeviceToHost));
  return SM_OK;
}
int sm_water_state(sm_context* ctx, float* pos2, float* speed2, double* volume, double* sediment,
                   int32_t* contains, int32_t* alive) {
  std::vector<float4> a; std::vector<double2> b; std::vector<uint2> c; std::vector<unsigned char> al;
  int rc = fetch_state(ctx, KIND_WATER, a, b, c, al);
  if (rc != SM_OK) return rc;
  for (size_t i = 0; i < a.size(); i++) {
    if (pos2) { pos2[2 * i] = a[i].x; pos2[2 * i + 1] = a[i].y; }
    if (speed2) { speed2[2 * i] = a[i].z; speed2[2 * i + 1] = a[i].w; }
    if (volume) volume[i] = b[i].x;
    if (sediment) sediment[i] = b[i].y;
    if (contains) contains[i] = (int32_t)c[i].x;
    if (alive) alive[i] = al[i];
  }
  return SM_OK;
}
int sm_wind_state(sm_context* ctx, float* pos2, float* speed3, double* height, double* sediment,
                  int32_t* contains, int32_t* alive) {
  std::vector<float4> a; std::vector<double2> b; std::vector<uint2> c; std::vector<unsigned char> al;
  int rc = fetch_state(ctx, KIND_WIND, a, b, c, al);
  if (rc != SM_OK) return rc;
  for (size_t i = 0; i < a.size(); i++) {
    if (pos2) { pos2[2 * i] = a[i].x; pos2[2 * i + 1] = a[i].y; }
    if (speed3) {
      speed3[3 * i] = a[i].z; speed3[3 * i + 1] = a[i].w;
      float sz; memcpy(&sz, &c[i].y, 4); speed3[3 * i + 2] = sz;
    }
    if (sediment) sediment[i] = b[i].x;
    if (height) height[i] = b[i].y;
    if (contains) contains[i] = (int32_t)c[i].x;
    if (alive) alive[i] = al[i];
  }
  return SM_OK;
}

int sm_set_soil_colors(sm_context* ctx, const float* rgba, int32_t n) {
  if (!rgba || n < 1 || n > SM_MAX_SOILS) return fail(ctx, SM_ERR_INVALID, "sm_set_soil_colors: 1..64 soils");
  CK(cudaSetDevice(ctx->cfg.device));
  if (!ctx->d_colors) CK(cudaMalloc(&ctx->d_colors, SM_MAX_SOILS * sizeof(float4)));
  CK(cudaMemcpy(ctx->d_colors, rgba, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice));
  return SM_OK;
}
int sm_mesh_update(sm_context* ctx, int32_t slice, float* host_vertices) {
  if (!ctx->d_colors) return fail(ctx, SM_ERR_INVALID, "sm_mesh_update: soil colours not set");
  if (ctx->nranks > 1) return fail(ctx, SM_ERR_INVALID, "sm_mesh_update is not available on a sharded context");
  CK(cudaSetDevice(ctx->cfg.device));
  if (!ctx->d_verts) CK(cudaMalloc(&ctx->d_verts, ctx->cells * 11 * sizeof(float)));
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  k_mesh<<<ctx->num_sms * 16, MESH_BLOCK, 0, ctx->stream>>>(ctx->d, slice, ctx->d_colors, ctx->d_verts);
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  ctx->launches++;
  ctx->timing_pending = true;
  ctx->mesh_valid = true;
  CK(cudaGetLastError());
  if (host_vertices) {
    CK(cudaMemcpyAsync(host_vertices, ctx->d_verts, ctx->cells * 11 * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  return SM_OK;
}
int sm_mesh_device_ptr(sm_context* ctx, void** dptr) {
  if (!ctx->mesh_valid) return fail(ctx, SM_ERR_INVALID, "no mesh yet: call sm_mesh_update");
  *dptr = ctx->d_verts;
  return SM_OK;
}
static int export_maps(sm_context* ctx, float* height, float* bgra) {
  if (!ctx->mesh_valid) return fail(ctx, SM_ERR_INVALID, "no mesh yet: call sm_mesh_update");
  CK(cudaSetDevice(ctx->cfg.device));
  float* d_out = nullptr;
  const size_t n = ctx->cells * (height ? 1 : 4);
  CK(cudaMalloc(&d_out, n * sizeof(float)));
  k_export<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d_verts, ctx->cells, ctx->d.scale, height ? d_out : nullptr,
                                                     height ? nullptr : d_out);
  ctx->launches++;
  cudaError_t e = cudaMemcpyAsync(height ? height : bgra, d_out, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  cudaFree(d_out);
  if (e != cudaSuccess) { ctx->err = cudaGetErrorString(e); return SM_ERR_CUDA; }
  return SM_OK;
}
int sm_export_height(sm_context* ctx, float* height) {
  if (!height) return fail(ctx, SM_ERR_INVALID, "null buffer");
  return export_maps(ctx, height, nullptr);
}
int sm_export_color(sm_context* ctx, float* bgra) {
  if (!bgra) return fail(ctx, SM_ERR_INVALID, "null buffer");
  return export_maps(ctx, nullptr, bgra);
}
int sm_parse_soil_file(const char* path, sm_soil* soils, char* names, float* colors, int32_t max_soils,
                       int32_t* nsoils, sm_layer* layers, int32_t max_layers, int32_t* nlayers, int32_t* world5) {
  if (!path || !nsoils || !nlayers) { g_create_err = "sm_parse_soil_file: null argument"; return SM_ERR_INVALID; }
  soilmachine::SoilFile f;
  try {
    soilmachine::parse_soil_file(path, f);
  } catch (const std::exception& e) {
    g_create_err = e.what();
    return SM_ERR_INVALID;
  }
  if ((int)f.soils.size() > max_soils || (int)f.layers.size() > max_layers) {
    g_create_err = "sm_parse_soil_file: output buffers too small";
    return SM_ERR_INVALID;
  }
  *nsoils = (int32_t)f.soils.size();
  *nlayers = (int32_t)f.layers.size();
  for (size_t i = 0; i < f.soils.size(); i++) {
    const soilmachine::SoilEntry& e = f.soils[i];
    if (soils) soils[i] = sm_soil{e.transports, e.erodes, e.cascades, e.abrades, e.density, e.porosity, e.solubility,
                                  e.equrate, e.friction, e.erosionrate, e.maxdiff, e.settling, e.suspension, e.abrasion};
    if (names) { memset(names + 32 * i, 0, 32); strncpy(names + 32 * i, e.name.c_str(), 31); }
    if (colors) for (int k = 0; k < 4; k++) colors[4 * i + k] = e.color[k];
  }
  for (size_t i = 0; i < f.layers.size(); i++) {
    const soilmachine::LayerEntry& l = f.layers[i];
    if (layers) layers[i] = sm_layer{l.type, l.min, l.bias, l.scale, l.octaves, l.lacunarity, l.gain, l.frequency};
  }
  if (world5) { world5[0] = f.world.sizex; world5[1] = f.world.sizey; world5[2] = f.world.scale; world5[3] = f.world.nwater; world5[4] = f.world.nwind; }
  return SM_OK;
}
// ---- wind field: D3Q19 lattice Boltzmann (sm_lbm.cuh) ----------------------------------------------------------
// boundary from the terrain, SoilMachine.cpp:234-239 with lbmwind.h:119 scale = (SIZEX, SCALE, SIZEY)/(NX, 32, NZ)
__global__ void k_lbm_boundary_from_map(DevCtx c, LbmDev L) {
  const size_t n = (size_t)L.nx * L.ny * L.nz;
  const float sx = (float)c.dimx / (float)L.nx, sy = (float)c.scale / 32.0f, sz = (float)c.dimy / (float)L.nz;
  for (size_t ind = (size_t)blockIdx.x * blockDim.x + threadIdx.x; ind < n; ind += (size_t)gridDim.x * blockDim.x) {
    const int z = (int)(ind % L.nz), y = (int)((ind / L.nz) % L.ny), x = (int)(ind / ((size_t)L.nz * L.ny));
    const int mx = (int)(sx * (float)x), mz = (int)(sz * (float)z);
    const double h = rec_height(c.top[(size_t)mx * c.dimy + mz]);
    L.B[ind] = (h > (double)((sy * (float)y) / (float)c.scale)) ? 1.0f : 0.0f;
  }
}
static int lbm_ready(sm_context* ctx) {
  if (!ctx->lbm.F[0]) return fail(ctx, SM_ERR_INVALID, "no wind field: call sm_lbm_create");
  CK(cudaSetDevice(ctx->cfg.device));
  return SM_OK;
}
int sm_lbm_init(sm_context* ctx) {
  int rc = lbm_ready(ctx);
  if (rc != SM_OK) return rc;
  ctx->lbm_cur = 0;
  k_lbm_init<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->lbm, 0);
  ctx->launches++;
  CK(cudaGetLastError());
  return SM_OK;
}
int sm_lbm_create(sm_context* ctx, int32_t nx, int32_t ny, int32_t nz) {
  if (nx < 3 || ny < 3 || nz < 3 || (int64_t)nx * ny * nz * LBM_Q >= (1ll << 31))
    return fail(ctx, SM_ERR_INVALID, "sm_lbm_create: 3 <= nx, ny, nz and nx*ny*nz*19 < 2^31");
  CK(cudaSetDevice(ctx->cfg.device));
  LbmDev& L = ctx->lbm;
  cudaFree(L.F[0]); cudaFree(L.F[1]); cudaFree(L.B); cudaFree(L.RHO); cudaFree(L.V);
  L = LbmDev{};
  ctx->d.wind_v4 = nullptr;
  L.nx = nx; L.ny = ny; L.nz = nz;
  const size_t n = (size_t)nx * ny * nz;
  CK(cudaMalloc(&L.F[0], n * LBM_Q * 4)); CK(cudaMalloc(&L.F[1], n * LBM_Q * 4));
  CK(cudaMalloc(&L.B, n * 4)); CK(cudaMalloc(&L.RHO, n * 4)); CK(cudaMalloc(&L.V, n * 16));
  CK(cudaMemsetAsync(L.B, 0, n * 4, ctx->stream));
  CK(cudaMemsetAsync(L.F[1], 0, n * LBM_Q * 4, ctx->stream));
  // constants, evaluated as oracle/lbm_oracle.c does (fp32, left to right)
  LbmConst K;
  K.w[0] = 1.0f / 3.0f; K.w[1] = 1.0f / 18.0f; K.w[2] = 1.0f / 36.0f;
  K.force[0] = 0.05f * -2.0f; K.force[1] = 0.05f * 0.0f; K.force[2] = 0.05f * 1.0f;
  const float cs = 1.0f / sqrtf(3.0f);
  K.cs2 = 1.0f / cs / cs;
  K.cs4 = 1.0f / cs / cs / cs / cs;
  const float zero[3] = {0.0f, 0.0f, 0.0f};
  LbmEqAll<LBM_Q - 1>::run(K, 1.0f, K.force, K.eq_force);
  LbmEqAll<LBM_Q - 1>::run(K, 1.0f, zero, K.eq_rest);
  CK(cudaMemcpyToSymbolAsync(c_lbm, &K, sizeof(K), 0, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return sm_lbm_init(ctx);       // lbmwind.h:101-107: init.cs runs while the boundary is still all zero
}
int sm_lbm_set_boundary(sm_context* ctx, const float* boundary) {
  int rc = lbm_ready(ctx);
  if (rc != SM_OK) return rc;
  const size_t n = (size_t)ctx->lbm.nx * ctx->lbm.ny * ctx->lbm.nz;
  if (boundary) {
    CK(cudaMemcpyAsync(ctx->lbm.B, boundary, n * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  } else {                       // from the terrain of this context
    if (ctx->nranks > 1) return fail(ctx, SM_ERR_INVALID, "sm_lbm_set_boundary: not on a sharded context");
    k_lbm_boundary_from_map<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, ctx->lbm);
    ctx->launches++;
    CK(cudaGetLastError());
  }
  return SM_OK;
}
int sm_lbm_step(sm_context* ctx, int32_t nsteps, double* device_ms) {
  int rc = lbm_ready(ctx);
  if (rc != SM_OK) return rc;
  if (nsteps < 0) return fail(ctx, SM_ERR_INVALID, "sm_lbm_step: nsteps");
  const size_t n = (size_t)ctx->lbm.nx * ctx->lbm.ny * ctx->lbm.nz;
  const int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)ctx->num_sms * 16);
  CK(cudaEventRecord(ctx->evt0, ctx->stream));
  for (int i = 0; i < nsteps; i++) {
    k_lbm_step<<<blocks, 256, 0, ctx->stream>>>(ctx->lbm, ctx->lbm_cur);
    ctx->lbm_cur ^= 1;
  }
  CK(cudaEventRecord(ctx->evt1, ctx->stream));
  ctx->launches += nsteps;
  CK(cudaGetLastError());
  CK(cudaEventSynchronize(ctx->evt1));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, ctx->evt0, ctx->evt1));
  if (device_ms) *device_ms = ms;
  return SM_OK;
}
int sm_lbm_get(sm_context* ctx, float* f, float* rho, float* v4) {
  int rc = lbm_ready(ctx);
  if (rc != SM_OK) return rc;
  CK(cudaStreamSynchronize(ctx->stream));
  const size_t n = (size_t)ctx->lbm.nx * ctx->lbm.ny * ctx->lbm.nz;
  if (f) {                       // device: F[q][cell]; caller (as upstream): F[cell*19 + q]
    std::vector<float> soa(n * LBM_Q);
    CK(cudaMemcpy(soa.data(), ctx->lbm.F[ctx->lbm_cur], n * LBM_Q * 4, cudaMemcpyDeviceToHost));
    for (size_t ind = 0; ind < n; ind++) for (int q = 0; q < LBM_Q; q++) f[ind * LBM_Q + q] = soa[(size_t)q * n + ind];
  }
  if (rho) CK(cudaMemcpy(rho, ctx->lbm.RHO, n * 4, cudaMemcpyDeviceToHost));
  if (v4) CK(cudaMemcpy(v4, ctx->lbm.V, n * 16, cudaMemcpyDeviceToHost));
  return SM_OK;
}
int sm_wind_use_lbm(sm_context* ctx, int32_t on) {
  if (!on) { ctx->d.wind_v4 = nullptr; return SM_OK; }
  int rc = lbm_ready(ctx);
  if (rc != SM_OK) return rc;
  ctx->d.wind_v4 = (const float*)ctx->lbm.V;
  ctx->d.wind_nx = ctx->lbm.nx; ctx->d.wind_ny = ctx->lbm.ny; ctx->d.wind_nz = ctx->lbm.nz;
  return SM_OK;
}
int sm_lbm_advect(sm_context* ctx, int32_t n, float* pos4) {
  int rc = lbm_ready(ctx);
  if (rc != SM_OK) return rc;
  if (n < 0 || (n && !pos4)) return fail(ctx, SM_ERR_INVALID, "sm_lbm_advect: arguments");
  if (!n) return SM_OK;
  float4* d_pos = nullptr;
  CK(cudaMalloc(&d_pos, (size_t)n * 16));
  cudaError_t e = cudaMemcpyAsync(d_pos, pos4, (size_t)n * 16, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) {
    k_lbm_advect<<<(n + 255) / 256, 256, 0, ctx->stream>>>(ctx->lbm, n, d_pos);
    ctx->launches++;
    e = cudaMemcpyAsync(pos4, d_pos, (size_t)n * 16, cudaMemcpyDeviceToHost, ctx->stream);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  cudaFree(d_pos);
  if (e != cudaSuccess) { ctx->err = cudaGetErrorString(e); return SM_ERR_CUDA; }
  return SM_OK;
}

int sm_timer_start(sm_context* ctx) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaEventRecord(ctx->evt0, ctx->stream));
  return SM_OK;
}
int sm_timer_stop(sm_context* ctx, double* elapsed_ms) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaEventRecord(ctx->evt1, ctx->stream));
  CK(cudaEventSynchronize(ctx->evt1));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, ctx->evt0, ctx->evt1));
  if (elapsed_ms) *elapsed_ms = ms;
  return SM_OK;
}
int sm_launch_count(sm_context* ctx, int64_t* n) { *n = ctx->launches; return SM_OK; }
// debug (only meaningful in a -DSM_PROFILE build): clock64() totals per phase, summed over particles
// -DSM_PROFILE builds of k_sweep: 8 words per sweep - live particles, max step cycles, max wait cycles, max cycles a
// warp spent on its particles, sum of step cycles, steps, globaltimer at the first warp's start, at the last warp's end
int sm_debug_sweeps8(sm_context* ctx, uint64_t* out, int nsweeps) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaMemcpy(out, ctx->d.dbg, (size_t)std::min(nsweeps, 16384) * 64, cudaMemcpyDeviceToHost));
  CK(cudaMemset(ctx->d.dbg, 0, 8 * 16384 * sizeof(unsigned long long)));
  return SM_OK;
}
int sm_debug_sweeps(sm_context* ctx, uint64_t* out, int nsweeps) {   // -DSM_PROFILE builds: (clock64, alive) per sweep
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaMemcpy(out, ctx->d.dbg, (size_t)std::min(nsweeps, 16384) * 16, cudaMemcpyDeviceToHost));
  return SM_OK;
}
int sm_debug_profile(sm_context* ctx, uint64_t* out16, int reset) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  RunCtl h;
  CK(cudaMemcpy(&h, ctx->d.ctl, sizeof(RunCtl), cudaMemcpyDeviceToHost));
  for (int i = 0; i < 16; i++) out16[i] = h.prof[i];
  for (int i = 1; i < 4; i++) out16[12 + i] = h.marks[i] + (i == 3 ? h.marks[4] + h.marks[5] + h.marks[6] : 0);
  out16[13] = h.marks[1]; out16[14] = h.marks[2]; out16[15] = h.marks[3] + h.marks[4] + h.marks[5] + h.marks[6];
  if (reset == 2) { out16[13] = h.marks[0]; out16[14] = h.marks[7]; out16[15] = h.prof[15]; out16[10] = h.prof[12]; out16[11] = h.prof[13]; out16[12] = h.prof[14]; }
  if (reset == 3) { out16[0] = h.ring[0].tail; out16[1] = h.ring[1].tail; out16[2] = h.ring[0].head; out16[3] = h.ring[1].head; out16[4] = h.bump; return SM_OK; }
  if (reset) { CK(cudaMemset(&ctx->d.ctl->prof[0], 0, sizeof(h.prof))); CK(cudaMemset(&ctx->d.ctl->marks[0], 0, sizeof(h.marks))); }
  return SM_OK;
}
int sm_device_alloc(sm_context* ctx, int64_t bytes, void** dptr) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaMalloc(dptr, (size_t)bytes));
  return SM_OK;
}
int sm_device_free(sm_context* ctx, void* dptr) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaFree(dptr));
  return SM_OK;
}
int sm_device_upload(sm_context* ctx, void* dptr, const void* host, int64_t bytes) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaMemcpyAsync(dptr, host, (size_t)bytes, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

int sm_initialize(sm_context* ctx, int32_t seed, const sm_layer* layers, int32_t nlayers) {
  if (!layers || nlayers < 1 || nlayers > SM_MAX_LAYERS)
    return fail(ctx, SM_ERR_INVALID, "sm_initialize: 1..16 layers");
  CK(cudaSetDevice(ctx->cfg.device));
  LayerSet ls;
  ls.n = nlayers;
  for (int l = 0; l < nlayers; l++) {
    if (layers[l].type < 0 || (ctx->nsoils > 0 && layers[l].type >= ctx->nsoils))
      return fail(ctx, SM_ERR_INVALID, "sm_initialize: layer type out of range");
    LayerDev& L = ls.L[l];
    L.type = (uint32_t)layers[l].type; L.min = layers[l].min; L.bias = layers[l].bias;
    L.scale = layers[l].scale; L.octaves = (int)layers[l].octaves; L.lacunarity = layers[l].lacunarity;
    L.gain = layers[l].gain; L.frequency = layers[l].frequency;
    L.bounding = fnl_fractal_bounding(L.octaves, L.gain);
    ls.zslice[l] = layer_zslice(seed, l, nlayers);
  }
  const unsigned long long need = (unsigned long long)ctx->lcells * (unsigned long long)(nlayers - 1);
  if (ctx->cfg.pool_capacity > 0) {
    if (need > ctx->d.pool_cap) return fail(ctx, SM_ERR_POOL, "sm_initialize: pool_capacity too small");
  } else {
    int rc = alloc_pool(ctx, ctx->nranks > 1 ? need : need + (unsigned long long)ctx->cells + (4ull << 20));
    if (rc != SM_OK) return rc;
  }
  int rc = reset_pool_ctl(ctx, 0);
  if (rc != SM_OK) return rc;
  k_initialize<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, ls);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

}  // extern "C"
