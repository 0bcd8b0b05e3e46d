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
#include "sm_snap.cuh"
#include "sm_layer.cuh"
#include "sm_relax.cuh"
#include "sm_strata.cuh"
#include "sm_drain.cuh"
#include <cub/device/device_scan.cuh>
#include <type_traits>

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
// MULTI: the n cells of the whole sharded map in global cell order, each read from its column's owner, so that the
// tree - and with it every bit of the sum - is the one context's
template <bool MULTI> __global__ void k_height_sum1(DevCtx c, size_t n, double* __restrict__ partial) {
  const Sec32* __restrict__ const top = c.top;
  __shared__ double sh[256];
  const size_t chunk = (n + SUM_BLOCKS - 1) / SUM_BLOCKS;
  const size_t lo = (size_t)blockIdx.x * chunk, hi = (lo + chunk < n) ? lo + chunk : n;
  double acc = 0.0;
  for (size_t i = lo + threadIdx.x; i < hi; i += 256)
    acc += rec_height(MULTI ? *cell_ptr<MULTI>(c, (int)(i / (size_t)c.dimy), (int)(i % (size_t)c.dimy)) : top[i]);
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

// ---- snapshots (sm_snap.cuh): one thread per cell of this context's strip -------------------------------------------
// save: off[c] = length of column c (its own pool), off[cells] = 0; CUB's in-place exclusive scan turns this into the
// offsets
__global__ void __launch_bounds__(256) k_snap_count(DevCtx c, size_t cells, unsigned long long* __restrict__ off) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (size_t)gridDim.x * blockDim.x)
    off[i] = snap_count_cell(c.top[i], c.pool);
  if (blockIdx.x == 0 && threadIdx.x == 0) off[cells] = 0;
}
// save: the records of cells [lo, hi), bottom -> top, at out[off[c] - off[lo]]
__global__ void __launch_bounds__(256) k_snap_pack(DevCtx c, const unsigned long long* __restrict__ off, size_t lo,
                                                   size_t hi, SnapRec* __restrict__ out) {
  const unsigned long long base = off[lo];
  for (size_t i = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (size_t)gridDim.x * blockDim.x)
    snap_pack_cell(c.top[i], c.pool, off[i + 1] - off[i], out + (off[i] - base));
}
// save: out[i] = off[i] + add for i <= n (a rank's offsets placed in a whole-map snapshot)
__global__ void __launch_bounds__(256) k_snap_offsets(const unsigned long long* __restrict__ off, size_t n,
                                                      unsigned long long add, unsigned long long* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = off[i] + add;
}
// restore, before any map write: reads the snapshot's slice only.  err[0] |= 1 on a bad cell; buried[c] = the pool slots
// column c needs, buried[cells] = 0, for the in-place exclusive scan that gives each column its pool base
__global__ void __launch_bounds__(256) k_snap_validate(const unsigned long long* __restrict__ off,
                                                       const SnapRec* __restrict__ rec, size_t cells, int nsoils,
                                                       unsigned long long* __restrict__ buried, unsigned int* err) {
  bool bad = false;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (size_t)gridDim.x * blockDim.x) {
    const bool ok = snap_valid_cell((const uint64_t*)off, rec, cells, i, nsoils);
    buried[i] = ok ? snap_buried((const uint64_t*)off, i) : 0;
    bad |= !ok;
  }
  if (bad) atomicOr(err, 1u);
  if (blockIdx.x == 0 && threadIdx.x == 0) buried[cells] = 0;
}
// restore: every column of the strip from its records; base = the scanned buried counts
__global__ void __launch_bounds__(256) k_snap_unpack(DevCtx c, const unsigned long long* __restrict__ off,
                                                     const SnapRec* __restrict__ rec, size_t cells,
                                                     const unsigned long long* __restrict__ base) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (size_t)gridDim.x * blockDim.x)
    snap_unpack_cell((const uint64_t*)off, rec, i, (uint32_t)base[i], c.top[i], c.pool);
}

// ---- layer rasters (sm_layer.cuh): one thread per cell of this context's strip, pool phase 0 as k_cell_op ------------
// the block's sum of v into *out
__device__ __forceinline__ void block_add_u64(unsigned long long v, unsigned long long* out) {
  __shared__ unsigned long long sh[8];
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long s = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += sh[w];
    if (s) atomicAdd(out, s);
  }
}
// before any write: out[0] += pool slots the raster will allocate, out[1] += cells it touches, out[2] |= 1 when an
// entry is not finite or the type is out of range.  Reads the raster and, where delta > 0, the top record (and on an Air
// top the record underneath).
__global__ void __launch_bounds__(256) k_layer_check(DevCtx c, const double* __restrict__ delta, size_t cells, int type,
                                                     unsigned long long* __restrict__ out) {
  DevAccess a(c, nullptr, 0u);
  unsigned long long pushed = 0, touched = 0;
  bool bad = false;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (size_t)gridDim.x * blockDim.x) {
    const double d = delta[i];
    if (!layer_input_ok(d, type, c.nsoils)) { bad = true; continue; }
    touched += d != 0.0;
    if (d > 0) pushed += layer_pushes(a, c.top[i], d, (uint32_t)type);
  }
  if (bad) atomicOr(&out[2], 1ull);
  block_add_u64(pushed, &out[0]);
  __syncthreads();
  block_add_u64(touched, &out[1]);
}
// every cell with delta != 0: read the top record, apply, write it back; frees to ring 0, allocations from ring 1 or the
// bump counter.  leftover (nullable) gets every cell's leftover, *emptied += cells whose leftover is > 0.
__global__ void __launch_bounds__(256) k_layer_apply(DevCtx c, const double* __restrict__ delta, size_t cells,
                                                     uint32_t type, double* __restrict__ leftover,
                                                     unsigned long long* __restrict__ emptied) {
  DevAccess a(c, nullptr, 0u);
  unsigned long long n = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (size_t)gridDim.x * blockDim.x) {
    const double d = delta[i];
    double left = 0.0;
    if (d != 0.0) {
      Sec32 r = c.top[i];
      left = layer_apply_cell(a, r, d, type);
      c.top[i] = r;
    }
    if (leftover) leftover[i] = left;
    n += left > 0;
  }
  block_add_u64(n, emptied);
}

// ---- strata views (sm_strata.cuh): one thread per cell, read-only --------------------------------------------------
// the requested types: slot[t] = output slot of soil type t, -1 where t is not requested
struct StrataSel { signed char slot[SM_MAX_SOILS]; };
// cells [c0, c1) of this context's strip; slot i of cell i0 goes to out[i * stride + (i0 - c0)].  *nsec += sections read.
__global__ void __launch_bounds__(256) k_strata_compose(DevCtx c, const __grid_constant__ StrataSel sel, int ntypes, double lo, double hi,
                                                        int flags, size_t c0, size_t c1, double* __restrict__ out,
                                                        size_t stride, unsigned long long* __restrict__ nsec) {
  __shared__ float s_por[SM_MAX_SOILS];
  __shared__ signed char s_slot[SM_MAX_SOILS];
  for (int t = threadIdx.x; t < SM_MAX_SOILS; t += blockDim.x) {
    s_por[t] = t < c.nsoils ? c.soils[t].porosity : 0.f;
    s_slot[t] = sel.slot[t];
  }
  __syncthreads();
  const StrataPool a{c.pool};
  unsigned long long n = 0;
  for (size_t i = c0 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < c1; i += (size_t)gridDim.x * blockDim.x)
    n += strata_compose_cell(a, c.top[i], lo, hi, flags, s_slot, ntypes, s_por, out + (i - c0), stride);
  block_add_u64(n, nsec);
}
// cells [j0, j1) of this context's part of a voxel window: part cell j is column xs + j / wy, row y0 + j % wy (global
// coordinates; cx0 = the strip's first column); sample k of part cell j goes to out[k * stride + (j - j0)].
__global__ void __launch_bounds__(256) k_strata_voxel(DevCtx c, int cx0, int xs, int y0, int wy, double z0, double dz,
                                                      double rdz, uint32_t nz, size_t j0, size_t j1, unsigned char* __restrict__ out,
                                                      size_t stride, unsigned long long* __restrict__ nsec) {
  const StrataPool a{c.pool};
  unsigned long long n = 0;
  for (size_t j = j0 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < j1; j += (size_t)gridDim.x * blockDim.x) {
    const size_t x = (size_t)(xs - cx0) + j / (size_t)wy, y = (size_t)y0 + j % (size_t)wy;
    n += strata_voxel_cell(a, c.top[x * c.dimy + y], z0, dz, rdz, nz, out + (j - j0), stride);
  }
  block_add_u64(n, nsec);
}

// ---- slope relaxation (sm_relax.cuh): one phase of a pass, one thread per phase cell of this context's strip ---------
// Launch j of a call frees into ring[j & 1] and pops ring[(j & 1) ^ 1], which launch j - 1 filled and which nobody
// appends to now.  The counts go to this rank's counter block; a launch that could not serve a section raises the stop
// flag of every rank, and the launches after it return at once.
template <bool MULTI>
__global__ void __launch_bounds__(256) k_relax_phase(DevCtx c, int px, int py, int transferloop, unsigned int parity,
                                                     const __grid_constant__ RelaxMaps m) {
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  __shared__ int stop;
  for (int i = threadIdx.x; i < c.nsoils; i += blockDim.x) s_soils[i] = c.soils[i];
  const int me = MULTI ? c.rank : 0;
  if (threadIdx.x == 0) stop = (int)*((volatile unsigned long long*)&m.cnt[me][4]);
  __syncthreads();
  if (stop) return;
  const int P = relax_period(transferloop);
  const int x0 = MULTI ? c.rank * c.strip_w : 0, x1 = MULTI ? min(x0 + c.strip_w, c.dimx) : c.dimx;
  const int fx = relax_first(x0, px, P);
  const size_t nx = fx < x1 ? (size_t)((x1 - 1 - fx) / P + 1) : 0, ny = py < c.dimy ? (size_t)((c.dimy - 1 - py) / P + 1) : 0;
  typename std::conditional<MULTI, RelaxMulti, RelaxDev>::type a(c, s_soils, parity, m, transferloop);
  unsigned long long visits = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nx * ny; i += (size_t)gridDim.x * blockDim.x)
    visits += relax_visit(a, fx + (int)(i / ny) * P, py + (int)(i % ny) * P, transferloop);
  unsigned long long* const cnt = m.cnt[me];
  block_add_u64(visits, &cnt[0]);
  __syncthreads();
  block_add_u64(a.rs.changes, &cnt[1]);
  __syncthreads();
  block_add_u64(a.rs.transfers, &cnt[2]);
  if (a.rs.drops) {
    atomicAdd(&cnt[3], a.rs.drops);
    for (int q = 0; q < (MULTI ? c.nranks : 1); q++) m.cnt[q][4] = 1;
  }
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
__device__ __forceinline__ Sec32 ldg_rec(const Sec32* p) {
  const double2 a = __ldg((const double2*)p);
  const double2 b = __ldg(((const double2*)p) + 1);
  Sec32 r;
  r.size = a.x; r.floor = a.y; r.saturation = b.x;
  const unsigned long long w = (unsigned long long)__double_as_longlong(b.y);
  r.type = (uint32_t)w; r.below = (uint32_t)(w >> 32);
  return r;
}
// Read-only view of the whole map, in the accessor interface map_normal() and map_height_bilinear() expect.
// rec(x, y) is the top record of the global cell (x, y): on a sharded map it lies in the strip of the column's
// owner and is reached through that rank's peer pointer.  below(x, r) is the section under r, read from the pool of
// the column's owner (a column's buried sections always live there).  Every load takes the read-only __ldg path.
// That is valid only because nothing writes the map while a kernel using this view runs: on one context the
// kernel is ordered after the earlier work of its stream, and on a sharded map the caller has made every rank's
// earlier work complete before the call (sm_sync on every rank, then a host barrier; see the header).
template <bool MULTI> struct MapView {
  const DevCtx& c;
  Sec32 tmp;
  __device__ __forceinline__ int dimx() const { return c.dimx; }
  __device__ __forceinline__ int dimy() const { return c.dimy; }
  __device__ __forceinline__ int scale() const { return c.scale; }
  __device__ __forceinline__ const Sec32* rec(int x, int y) { tmp = ldg_rec(cell_ptr<MULTI>(c, x, y)); return &tmp; }
  __device__ __forceinline__ double height(int x, int y) { return rec_height(*rec(x, y)); }
  __device__ __forceinline__ Sec32 below(int x, const Sec32& r) const {
    const Sec32* pool = MULTI ? c.peer[owner_of_x<MULTI>(c, x)].pool : c.pool;
    return ldg_rec(&pool[r.below]);
  }
};
#define MESH_BLOCK 256
// Meshes this rank's strip [x0, x1) (the whole map on one context): one vertex per cell in strip cell order
// (x - x0)*dimy + y, which is the slice [x0*dimy, x1*dimy) of the unsharded vertex array.  The walk down to the
// slice plane stays in this rank's own columns and pool; only the normals of the columns x0 and x1 - 1 read the
// neighbouring strips, through MapView.
template <bool MULTI>
__global__ void __launch_bounds__(MESH_BLOCK) k_mesh(DevCtx c, int slice, const float4* __restrict__ colors,
                                                     float* __restrict__ verts) {
  __shared__ __align__(16) float s_v[MESH_BLOCK * 11];   // staged so the 44-byte vertices leave as 16-byte rows
  const int x0 = MULTI ? c.rank * c.strip_w : 0;
  const int x1 = MULTI ? min(x0 + c.strip_w, c.dimx) : c.dimx;
  const size_t cells = (size_t)(x1 - x0) * c.dimy;
  const float plane = (float)slice / (float)c.scale;             // (float)SLICE/(float)SCALE
  for (size_t base = (size_t)blockIdx.x * MESH_BLOCK; base < cells; base += (size_t)gridDim.x * MESH_BLOCK) {
    const size_t cell = base + threadIdx.x;
    if (cell < cells) {
      const int x = x0 + (int)(cell / c.dimy), y = (int)(cell % c.dimy);
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
        MapView<MULTI> m{c, Sec32{}};
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
// 3 query (height, surface, normal), 4 bilinear height, 5 seep, 6 water cascade.  The read-only ops 3 and 4 run in
// k_cell_read, which also serves sharded maps; the others change the map and run on one context only.
struct CellOp { int op; int x, y; float fx, fy; double v; int t; };
struct CellRes { double d; int32_t surface; float n[3]; };
template <bool MULTI> __global__ void k_cell_read(DevCtx c, CellOp o, CellRes* res) {
  MapView<MULTI> v{c, Sec32{}};
  CellRes r{0.0, 0, {0.f, 0.f, 0.f}};
  if (o.op == 3) {
    r.d = map_height(v, o.x, o.y);
    r.surface = (int32_t)rec_surface(*v.rec(o.x, o.y));
    sm_f3 n = map_normal(v, o.x, o.y);
    r.n[0] = n.x; r.n[1] = n.y; r.n[2] = n.z;
  } else if (o.op == 4) r.d = map_height_bilinear(v, o.fx, o.fy);
  *res = r;
}
__global__ void k_cell_op(DevCtx c, CellOp o, CellRes* res) {
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  for (int i = 0; i < c.nsoils; i++) s_soils[i] = c.soils[i];
  DevAccess a(c, s_soils, 0u);
  CellRes r{0.0, 0, {0.f, 0.f, 0.f}};
  if (o.op == 0) col_add(a, *a.rec(o.x, o.y), o.v, (uint32_t)o.t);
  else if (o.op == 1) r.d = col_remove(a, *a.rec(o.x, o.y), o.v);
  else if (o.op == 2) Cascade<3, DevAccess>::run(a, (int)roundf(o.fx), (int)roundf(o.fy), o.t);
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
template <bool MULTI> __global__ void k_cell_column(DevCtx c, int x, int y, int cap, int* n_out, Sec32* out) {
  MapView<MULTI> v{c, Sec32{}};
  Sec32 r = *v.rec(x, y);
  int n = 0;
  if (r.type != SM_EMPTY) {
    for (;;) {
      if (n < cap) out[n] = r;
      n++;
      if (r.below == SM_NIL) break;
      r = v.below(x, r);
    }
  }
  *n_out = n;       // top first; the host reverses
}

// wind-field boundary from the terrain, SoilMachine.cpp:234-239 with lbmwind.h:119 scale = (SIZEX, SCALE, SIZEY)/(NX,
// 32, NZ).  Always the whole lattice; on a sharded map each sampled column is read from its owner.
template <bool MULTI> __global__ void k_lbm_boundary_from_map(DevCtx c, LbmDev L) {
  const size_t n = (size_t)L.nx * L.ny * L.nz;
  const float sx = (float)c.dimx / (float)L.nx, sy = (float)c.scale / 32.0f, sz = (float)c.dimy / (float)L.nz;
  MapView<MULTI> v{c, Sec32{}};
  for (size_t ind = (size_t)blockIdx.x * blockDim.x + threadIdx.x; ind < n; ind += (size_t)gridDim.x * blockDim.x) {
    const int z = (int)(ind % L.nz), y = (int)((ind / L.nz) % L.ny), x = (int)(ind / ((size_t)L.nz * L.ny));
    const int mx = (int)(sx * (float)x), mz = (int)(sz * (float)z);
    const double h = v.height(mx, mz);
    L.B[ind] = (h > (double)((sy * (float)y) / (float)c.scale)) ? 1.0f : 0.0f;
  }
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
// MULTI: the whole map of a sharded context, each column and its buried sections read from the column's owner, into
// the issuing rank's whole-map bitmap
template <bool MULTI>
__global__ void __launch_bounds__(256) k_hydro_classify(DevCtx c, ActiveMap am) {
  const unsigned long long cells = am.ncells;
  for (unsigned long long cell = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; cell < cells;
       cell += (unsigned long long)gridDim.x * blockDim.x) {
    const Sec32 r = MULTI ? *cell_ptr<MULTI>(c, (int)(cell / (unsigned long long)c.dimy), (int)(cell % (unsigned long long)c.dimy))
                          : c.top[cell];
    if (r.type == SM_EMPTY) continue;
    const int x = (int)(cell / (unsigned long long)c.dimy), y = (int)(cell % (unsigned long long)c.dimy);
    const Sec32* const pool = MULTI ? c.peer[owner_of_x<MULTI>(c, x)].pool : c.pool;
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
      const Sec32 s = pool[b];
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
// BUDGET: the hydrology's mass budget (HydroScratchBudget::bud, sm_hydro_coop.cuh), for contexts created with SM_FLAG_BUDGET.
// CELLS (with BUDGET): its per-cell maps, SM_HYDRO_CELL_TERMS f64 per cell interleaved (eroded, deposited, cascade_net,
// water_net), cell order x*dimy + y, for contexts created with SM_FLAG_HYDRO_CELL_BUDGET.  The map pointer lives in an
// empty-when-off base, so that HydroBack<BUDGET> keeps its size and layout.
template <bool CELLS> struct HydroCellsRef {
  __device__ __forceinline__ explicit HydroCellsRef(double*) {}
};
template <> struct HydroCellsRef<true> {
  double* hcells;
  __device__ __forceinline__ explicit HydroCellsRef(double* m) : hcells(m) {}
};
// Frequency arrays of every rank of a sharded map.  Rank q's copies are authoritative for the columns of its strip
// only (the batches write wtrack where the particle is, on the rank that owns that column), so the hydrology reads and
// writes each cell's words at the column's owner.  A trailing kernel parameter, as CellMaps, so that DevCtx and
// PeerPtrs keep their layout.
struct FreqPeers {
  float* wfreq[SM_MAX_RANKS];
  float* wtrack[SM_MAX_RANKS];
};
template <bool MULTI> struct FreqPeersRef {
  __device__ __forceinline__ explicit FreqPeersRef(const FreqPeers*) {}
};
template <> struct FreqPeersRef<true> {
  const FreqPeers* fp;
  __device__ __forceinline__ explicit FreqPeersRef(const FreqPeers* f) : fp(f) {}
};
// MULTI: the map is sharded.  Records, pool allocations and frees go to the column's owner (DevBack<true>, steered by
// the focus() calls of sm_hydro_coop.cuh); the active-cell index is one whole-map bitmap on the issuing rank, indexed
// by global cell, as on one context.
template <bool MULTI, bool BUDGET, bool CELLS = false>
struct HydroBack : DevBack<MULTI, BUDGET>, HydroCellsRef<CELLS>, FreqPeersRef<MULTI> {
  static_assert(!CELLS || BUDGET, "the per-cell maps are measured by the budget instantiations");
  static_assert(!(CELLS && MULTI), "the hydrology's per-cell maps are not kept on a sharded map");
  static constexpr bool kHydroHooks = true;
  static constexpr bool kCellBudget = CELLS;
  ActiveMap act;
  bool marking;
  __device__ __forceinline__ HydroBack(const DevCtx& ctx, const SoilDev* ss, const ActiveMap& am, bool mk,
                                       double* cells = nullptr, const FreqPeers* fp = nullptr)
      : DevBack<MULTI, BUDGET>(ctx, ss, 0u), HydroCellsRef<CELLS>(cells), FreqPeersRef<MULTI>(fp), act(am), marking(mk) {}
  // index i = y*dimx + x
  __device__ __forceinline__ float wfreq(int i) const {
    if constexpr (MULTI) return this->fp->wfreq[owner_of_x<true>(this->c, i % this->c.dimx)][i];
    else return this->c.wfreq[i];
  }
  __device__ __forceinline__ float wtrack(int i) const {
    if constexpr (MULTI) return this->fp->wtrack[owner_of_x<true>(this->c, i % this->c.dimx)][i];
    else return this->c.wtrack[i];
  }
  __device__ __forceinline__ void set_wtrack(int i, float v) {
    if constexpr (MULTI) this->fp->wtrack[owner_of_x<true>(this->c, i % this->c.dimx)][i] = v;
    else this->c.wtrack[i] = v;
  }
  // One fire-and-forget f64 reduction (the rounding of `total += d`), as DevBack::cell_budget: the warp does not wait
  // for it.  One lane of one warp issues them in program order, so each cell's additions land in execution order.  The
  // map is device memory; saying so lets the compiler emit the global-space reduction (ATOMG/RED, no result used)
  // instead of a generic-address atomic with a shared-memory fallback branch behind it.
  __device__ __forceinline__ void cell_budget(int term, int x, int y, double d) {
    if constexpr (CELLS) {
      double* const m = this->hcells + ((size_t)x * this->c.dimy + y) * SM_HYDRO_CELL_TERMS + term;
      __builtin_assume(__isGlobal(m));
      atomicAdd(m, d);
    }
  }
  // single writer: only the lane that mutates columns calls these
  __device__ __forceinline__ void air_mark(Sec32* r, int x, int y) {
    if (marking && r->type == SM_AIR) active_mark_block(act, x, y, this->c.dimx, this->c.dimy);
  }
  __device__ __forceinline__ void wet_mark(int x, int y) {
    if (marking) active_set(act, (unsigned long long)x * this->c.dimy + y);
  }
};
// what a hydrology call hands back: its counters, and with BUDGET the eleven budget sums
struct HydroTotals {
  HydroCount hc;
  double bud[SM_HYDRO_BUDGET_SLOTS];
};
template <bool BUDGET, class S> __device__ __forceinline__ void hydro_budget_zero(S& hx, int lane) {
  if constexpr (BUDGET) if (lane == 0)
    for (int k = 0; k < SM_HYDRO_BUDGET_SLOTS; k++) hx.bud[k] = 0.0;
}
template <bool BUDGET, class S> __device__ __forceinline__ void hydro_totals_out(HydroTotals* out, const HydroCount& hc, const S& hx) {
  hydro_count_out(&out->hc, hc);
  if constexpr (BUDGET)
    for (int k = 0; k < SM_HYDRO_BUDGET_SLOTS; k++) out->bud[k] = hx.bud[k];
}
// `hcells`: the per-cell maps with CELLS (HydroBack), `fp`: the ranks' frequency arrays with MULTI; trailing
// parameters so that DevCtx keeps its layout.
// MULTI: the finished particles of a sharded map's last water batch.  A dead particle's final state lives on the rank
// that ran its last step, and only there does `done` hold the dead marker: every rank clears done[0, n) before a
// spawning launch (launch_run), and a rank writes a particle's `done` only while it holds the particle.  So the holder
// is the one rank whose word is 0xFFFFFFFF; the flood reads the state there and leaves SM_DONE_FLOODED there.
// The flood phase over the particles [base0, n) by one warp.  RESUME: the counters and the budget sums continue from
// what *out holds (k_hydro_flood_sweep, several flood phases in one call), else they start from zero.
template <bool MULTI, bool BUDGET, bool CELLS, bool RESUME>
__device__ __forceinline__ void hydro_flood_warp(const DevCtx& c, int base0, int n, HydroTotals* out, double* hcells,
                                                 const FreqPeers& fp) {
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  __shared__ CoopScratch sc;
  __shared__ typename HydroScratchOf<BUDGET>::type hx;
  const int lane = threadIdx.x;
  for (int i = lane; i < c.nsoils; i += 32) s_soils[i] = c.soils[i];
  if constexpr (RESUME && BUDGET) {
    if (lane == 0) for (int k = 0; k < SM_HYDRO_BUDGET_SLOTS; k++) hx.bud[k] = out->bud[k];
  } else {
    hydro_budget_zero<BUDGET>(hx, lane);
  }
  __syncwarp();
  WarpDev w{lane};
  ActiveMap none{};
  HydroBack<MULTI, BUDGET, CELLS> back(c, s_soils, none, false, hcells, &fp);
  CoopWin<HydroBack<MULTI, BUDGET, CELLS> > a(back, &sc);
  HydroCount hc{};
  if constexpr (RESUME) hc = out->hc;
  for (int base = base0; base < n; base += 32) {
    const int i = base + lane;
    bool cand = false;
    int holder = 0;
    if constexpr (MULTI) {
      if (i < n)
        for (int q = 0; q < c.nranks; q++)
          if (c.peer[q].done[i] == 0xFFFFFFFFu) {
            holder = q;
            cand = (c.peer[q].alive[i] == 0) && !(c.peer[q].pb[i].x < SM_MINVOL);
            break;
          }
    } else {
      if (i < n) cand = (c.alive[i] == 0) && !(c.pb[i].x < SM_MINVOL) && c.done[i] != SM_DONE_FLOODED;
    }
    unsigned int m = __ballot_sync(0xFFFFFFFFu, cand);
    while (m) {                                   // warp-uniform
      const int j = base + __ffs((int)m) - 1;
      m &= m - 1u;
      const int q = MULTI ? __shfl_sync(0xFFFFFFFFu, holder, j - base) : 0;
      const float4 pa = MULTI ? c.peer[q].pa[j] : c.pa[j];
      const double2 pb = MULTI ? c.peer[q].pb[j] : c.pb[j];
      WaterP p;
      p.px = pa.x; p.py = pa.y; p.sx = pa.z; p.sy = pa.w;
      p.volume = pb.x; p.sediment = pb.y; p.contains = MULTI ? c.peer[q].pc[j].x : c.pc[j].x;
      hydro_flood_particle_coop(w, a, &hx, p, hc);
      if (lane == 0) {
        if (MULTI) c.peer[q].done[j] = SM_DONE_FLOODED;
        else c.done[j] = SM_DONE_FLOODED;
      }
      __syncwarp();
    }
  }
  if (lane == 0) hydro_totals_out<BUDGET>(out, hc, hx);
}
template <bool MULTI, bool BUDGET, bool CELLS = false>
__global__ void __launch_bounds__(32) k_hydro_flood_w(DevCtx c, int n, HydroTotals* out, double* hcells,
                                                      const __grid_constant__ FreqPeers fp) {
  hydro_flood_warp<MULTI, BUDGET, CELLS, false>(c, 0, n, out, hcells, fp);
}

// ---- sweep floods (sm_water_run_flooding): the batch advances one sweep per launch of k_sweep, and after each sweep
// the particles that stopped in it flood, in ascending index, before the next sweep starts.
// FloodGate: lives on the issuing context's device, zeroed by the host at the start of a call.
//   hi1 / loinv  the flood candidates k_flood_gate found after the last sweep: indices [n - loinv, hi1), 0 = none
//   ended        the batch had no live particle left after an earlier sweep
//   sweeps       sweeps executed so far (a launch that finds no live particle executes none)
struct FloodGate {
  unsigned int hi1, loinv, ended, pad;
  unsigned long long sweeps;
};
// After a sweep: count it, rotate the pool rings (below) and bound the particles that flood() will find (the predicate
// of hydro_flood_warp: dead, volume >= minvol, not flooded yet), so that a sweep nobody stopped in costs no flood scan.
// One pass over n words.
template <bool MULTI>
__global__ void __launch_bounds__(256) k_flood_gate(DevCtx c, int n, FloodGate* g) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    if (!g->ended) g->sweeps++;
    if (c.ctl->alive == 0) g->ended = 1u;     // MULTI: the issuing rank's copy holds the total over the ranks
    // A one-sweep launch advances tag_base by 3, so without this every launch would free into the same ring and pop
    // the same other ring, and the sweeps' frees would never be served again.  One unused tag more per sweep makes
    // launch k free into ring[(t0 + k) % 3] and pop the ring launch k - 2 filled, as consecutive sweeps of one launch
    // do.  Every rank's tags advance alike (the ranks' next launches wait for this kernel).
    if constexpr (MULTI) {
      for (int q = 0; q < c.nranks; q++) c.peer[q].ctl->tag_base += 1u;
    } else {
      c.ctl->tag_base += 1u;
    }
  }
  const int stride = gridDim.x * blockDim.x;
  for (int base = blockIdx.x * blockDim.x; base < n; base += stride) {     // warp-uniform trip count
    const int i = base + (int)threadIdx.x;
    bool cand = false;
    if (i < n) {
      if constexpr (MULTI) {
        for (int q = 0; q < c.nranks; q++)
          if (c.peer[q].done[i] == 0xFFFFFFFFu) {
            cand = (c.peer[q].alive[i] == 0) && !(c.peer[q].pb[i].x < SM_MINVOL);
            break;
          }
      } else {
        cand = (c.alive[i] == 0) && !(c.pb[i].x < SM_MINVOL) && c.done[i] != SM_DONE_FLOODED;
      }
    }
    const unsigned int m = __ballot_sync(0xFFFFFFFFu, cand);
    if ((threadIdx.x & 31) == 0 && m) {
      const int w0 = i;                                   // lane 0's index
      atomicMax(&g->hi1, (unsigned int)(w0 + 32 - __clz((int)m)));
      atomicMax(&g->loinv, (unsigned int)(n - (w0 + __ffs((int)m) - 1)));
    }
  }
}
// The flood phase after one sweep: hydro_flood_warp over the gate's range, counters and budget continuing from *out
// (zeroed by the host at the start of the call); then the gate is cleared for the next sweep.
template <bool MULTI, bool BUDGET, bool CELLS = false>
__global__ void __launch_bounds__(32) k_hydro_flood_sweep(DevCtx c, int n, HydroTotals* out, double* hcells,
                                                          const __grid_constant__ FreqPeers fp, FloodGate* g) {
  const unsigned int hi1 = g->hi1, loinv = g->loinv;
  if (hi1 == 0u) return;
  hydro_flood_warp<MULTI, BUDGET, CELLS, true>(c, (n - (int)loinv) & ~31, (int)hi1, out, hcells, fp);
  if (threadIdx.x == 0) { g->hi1 = 0u; g->loinv = 0u; }
}

template <bool MULTI, bool BUDGET, bool CELLS = false>
__global__ void __launch_bounds__(32) k_hydro_seep_w(DevCtx c, ActiveMap am, HydroTotals* out, double* hcells,
                                                     const __grid_constant__ FreqPeers fp) {
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  __shared__ CoopScratch sc;
  __shared__ typename HydroScratchOf<BUDGET>::type hx;
  const int lane = threadIdx.x;
  for (int i = lane; i < c.nsoils; i += 32) s_soils[i] = c.soils[i];
  hydro_budget_zero<BUDGET>(hx, lane);
  __syncwarp();
  WarpDev w{lane};
  HydroBack<MULTI, BUDGET, CELLS> back(c, s_soils, am, true, hcells, &fp);
  CoopWin<HydroBack<MULTI, BUDGET, CELLS> > a(back, &sc);
  HydroCount hc{};
  const unsigned long long cells = am.ncells;
  for (unsigned long long cell = active_next(am, 0); cell < cells; cell = active_next(am, cell + 1)) {
    hydro_seep_visit_coop(w, a, &hx, (int)(cell / (unsigned long long)c.dimy), (int)(cell % (unsigned long long)c.dimy), hc);
    __syncwarp();
  }
  if (lane == 0) hydro_totals_out<BUDGET>(out, hc, hx);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
struct sm_group;
struct sm_context {
  sm_group* group = nullptr;      // set: this context is a group of rank contexts (sm_create_group, sm_group.cuh)
  sm_config cfg;
  DevCtx d;
  std::string err;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, evt0 = nullptr, evt1 = nullptr;
  size_t cells = 0;        // cells of the whole map (frequency arrays, bins)
  size_t lcells = 0;       // cells of this rank's x-strip (top records); == cells when not sharded
  int nranks = 1, rank = 0, x0 = 0, x1 = 0, share = 1;
  bool peers_attached = false;
  bool hydro_issuer = false;      // sharded: this rank issues the pooling hydrology of the whole map (sm_hydro_issuer)
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
  HydroTotals* d_hydro = nullptr;
  FloodGate* d_gate = nullptr;    // sm_water_run_flooding (allocated on first use)
  double hydro_bud[SM_HYDRO_BUDGET_SLOTS] = {};   // budget of the last successful hydrology call (SM_FLAG_BUDGET)
  bool hydro_bud_valid = false;
  // per-cell budget maps (SM_FLAG_CELL_BUDGET): 3 f64 per cell of the strip, interleaved; every rank's, by rank
  double* d_cells = nullptr;
  CellMaps cells_of = {};
  FreqPeers freq_of = {};         // every rank's frequency arrays, by rank (sharded hydrology)
  int cells_state = 0;           // 0 no batch yet, 1 the maps cover the last batch, 2 it ran on a kernel without them
  // per-cell maps of the hydrology's budget (SM_FLAG_HYDRO_CELL_BUDGET): SM_HYDRO_CELL_TERMS f64 per cell, interleaved
  double* d_hcells = nullptr;
  int hcells_state = 0;           // 0 no hydrology call yet, 1 the maps cover the last call, 2 that call failed
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

#include "sm_group.cuh"

extern "C" {

const char* sm_last_error(const sm_context* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

void sm_destroy(sm_context* ctx) {
  if (!ctx) return;
  if (ctx->group) { grp_destroy(ctx); return; }
  cudaSetDevice(ctx->cfg.device);
  cudaDeviceSynchronize();
  for (int q = 0; q < SM_MAX_RANKS; q++) for (int i = 0; i < SM_PEER_SLOTS; i++) if (ctx->ipc_opened[q][i]) cudaIpcCloseMemHandle(ctx->ipc_opened[q][i]);
  DevCtx& d = ctx->d;
  cudaFree(d.top); cudaFree(d.pool); cudaFree(d.ringbuf[0]); cudaFree(d.ringbuf[1]); cudaFree(d.ringbuf[2]);
  cudaFree(d.wfreq); cudaFree(d.wtrack); cudaFree(d.windfreq); cudaFree(ctx->d_soils);
  cudaFree(d.ctl); cudaFree(d.pa); cudaFree(d.pb); cudaFree(d.pc); cudaFree(d.alive); cudaFree(d.done); cudaFree(d.fin); cudaFree(d.mv); cudaFree(d.bud);
#ifdef SM_AUDIT_HANDOFF
  cudaFree(d.relz);
#endif
  for (int i = 0; i < 3; i++) cudaFree(d.lmask[i]);
  for (int i = 0; i < 2; i++) { cudaFree(d.head[i]); cudaFree(d.node[i]); }
  cudaFree(ctx->d_verts); cudaFree(ctx->d_colors); cudaFree(d.dbg);
  cudaFree(ctx->d_act); cudaFree(ctx->d_hydro); cudaFree(ctx->d_gate); cudaFree(ctx->d_cells); cudaFree(ctx->d_hcells);
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
  if ((cfg->flags & SM_FLAG_CELL_BUDGET) && !(cfg->flags & SM_FLAG_BUDGET)) {
    g_create_err = "sm_create: SM_FLAG_CELL_BUDGET needs SM_FLAG_BUDGET";
    return SM_ERR_INVALID;
  }
  if ((cfg->flags & SM_FLAG_HYDRO_CELL_BUDGET) && !(cfg->flags & SM_FLAG_BUDGET)) {
    g_create_err = "sm_create: SM_FLAG_HYDRO_CELL_BUDGET needs SM_FLAG_BUDGET";
    return SM_ERR_INVALID;
  }
  if ((cfg->flags & SM_FLAG_HYDRO_CELL_BUDGET) && nranks > 1) {
    g_create_err = "sm_create_sharded: SM_FLAG_HYDRO_CELL_BUDGET needs the pooling hydrology, which does not run on a "
                   "sharded context";
    return SM_ERR_INVALID;
  }
  int strip_w, sx0, sx1;
  if (!shard_strip(cfg->dimx, nranks, rank, &strip_w, &sx0, &sx1)) {
    g_create_err = kStripTooNarrow;
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
#ifdef SM_AUDIT_HANDOFF
    CK(cudaMalloc(&d.relz, N * 4)); CK(cudaMemsetAsync(d.relz, 0, N * 4, ctx->stream));
#endif
    for (int i = 0; i < 3; i++) {
      CK(cudaMalloc(&d.lmask[i], (N / 32 + 2) * sizeof(unsigned int)));
      CK(cudaMemsetAsync(d.lmask[i], 0, (N / 32 + 2) * sizeof(unsigned int), ctx->stream));
    }
    if (cfg->flags & SM_FLAG_BUDGET) {
      CK(cudaMalloc(&d.bud, N * SM_BUDGET_SLOTS * sizeof(double)));
      CK(cudaMemsetAsync(d.bud, 0, N * SM_BUDGET_SLOTS * sizeof(double), ctx->stream));
    }
    if (cfg->flags & SM_FLAG_CELL_BUDGET) {
      CK(cudaMalloc(&ctx->d_cells, LC * 3 * sizeof(double)));
      CK(cudaMemsetAsync(ctx->d_cells, 0, LC * 3 * sizeof(double), ctx->stream));
      if (nranks == 1) ctx->cells_of.p[0] = ctx->d_cells;    // sharded: every rank's, at sm_peer_attach
    }
    if (cfg->flags & SM_FLAG_HYDRO_CELL_BUDGET)                // zeroed by every sm_water_flood / sm_seep
      CK(cudaMalloc(&ctx->d_hcells, C * SM_HYDRO_CELL_TERMS * sizeof(double)));
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
int sm_create_group(const sm_config* cfg, int32_t nranks, const int32_t* devices, sm_context** out) {
  return grp_create(cfg, nranks, devices, out);
}
int sm_group_size(sm_context* ctx, int32_t* nranks) {
  if (!nranks) return fail(ctx, SM_ERR_INVALID, "null argument");
  *nranks = ctx->group ? ctx->group->n : 1;
  return SM_OK;
}
int sm_group_rank(sm_context* ctx, int32_t rank, sm_context** rank_ctx) {
  const int n = ctx->group ? ctx->group->n : 1;
  if (!rank_ctx || rank < 0 || rank >= n) return fail(ctx, SM_ERR_INVALID, "sm_group_rank: rank out of range");
  *rank_ctx = ctx->group ? ctx->group->rank[rank] : ctx;
  return SM_OK;
}
int sm_group_layout(const sm_config* cfg, int32_t nranks, int32_t rank, int32_t* x0, int32_t* x1, int64_t* pool_capacity) {
  int w, a, b;
  if (!cfg || nranks < 1 || nranks > SM_MAX_RANKS || rank < 0 || rank >= nranks || cfg->dimx < 2) {
    g_create_err = "sm_group_layout: invalid arguments";
    return SM_ERR_INVALID;
  }
  if (!shard_strip(cfg->dimx, nranks, rank, &w, &a, &b)) {
    g_create_err = kStripTooNarrow;
    return SM_ERR_INVALID;
  }
  if (x0) *x0 = a;
  if (x1) *x1 = b;
  if (pool_capacity) *pool_capacity = nranks == 1 ? cfg->pool_capacity : shard_pool_capacity(cfg->pool_capacity, cfg->dimx, a, b);
  return SM_OK;
}
int sm_shard_range(sm_context* ctx, int32_t* x0, int32_t* x1) {
  if (x0) *x0 = ctx->x0;
  if (x1) *x1 = ctx->x1;
  return SM_OK;
}

// ---- peers of a sharded map ----------------------------------------------------------------------------
// audit builds (-DSM_AUDIT_HANDOFF) exchange one more array, the hand-off records (relz)
#ifdef SM_AUDIT_HANDOFF
#define SM_PEER_USED (SM_PEER_ARRAYS + 1)
#else
#define SM_PEER_USED SM_PEER_ARRAYS
#endif
static void own_ptrs(sm_context* ctx, void** p) {
  DevCtx& d = ctx->d;
  p[0] = d.top; p[1] = d.pool; p[2] = d.ringbuf[0]; p[3] = d.ringbuf[1]; p[4] = d.ctl; p[5] = d.pa; p[6] = d.pb;
  p[7] = d.pc; p[8] = d.alive; p[9] = d.done; p[10] = d.head[0]; p[11] = d.head[1]; p[12] = d.node[0]; p[13] = d.node[1];
  p[14] = d.ringbuf[2]; p[15] = d.bud; p[16] = d.fin; p[17] = d.lmask[0]; p[18] = d.lmask[1]; p[19] = d.lmask[2];
  p[20] = ctx->d_cells;
  p[21] = d.wfreq; p[22] = d.wtrack;    // each its own cudaMalloc (create_impl), as cudaIpcGetMemHandle needs
#ifdef SM_AUDIT_HANDOFF
  p[SM_PEER_ARRAYS] = d.relz;
#endif
}
static void fill_peer(PeerPtrs& P, void* const* p, unsigned long long pool_cap) {
  P.top = (Sec32*)p[0]; P.pool = (Sec32*)p[1]; P.ringbuf[0] = (uint32_t*)p[2]; P.ringbuf[1] = (uint32_t*)p[3];
  P.ctl = (RunCtl*)p[4]; P.pa = (float4*)p[5]; P.pb = (double2*)p[6]; P.pc = (uint2*)p[7];
  P.alive = (unsigned char*)p[8]; P.done = (unsigned int*)p[9]; P.head[0] = (unsigned long long*)p[10];
  P.head[1] = (unsigned long long*)p[11]; P.node[0] = (uint2*)p[12]; P.node[1] = (uint2*)p[13];
  P.ringbuf[2] = (uint32_t*)p[14]; P.bud = (double*)p[15]; P.fin = (unsigned int*)p[16];
  P.lmask[0] = (unsigned int*)p[17]; P.lmask[1] = (unsigned int*)p[18]; P.lmask[2] = (unsigned int*)p[19];
  P.pool_cap = pool_cap;
#ifdef SM_AUDIT_HANDOFF
  P.relz = (unsigned int*)p[SM_PEER_ARRAYS];
#endif
}
int sm_peer_export(sm_context* ctx, sm_peer_blob* out) {
  if (ctx->group) return fail(ctx, SM_ERR_INVALID, "a group manages its ranks' peers itself (sm_group_rank gives the rank contexts)");
  if (!out) return fail(ctx, SM_ERR_INVALID, "null blob");
  CK(cudaSetDevice(ctx->cfg.device));
  memset(out, 0, sizeof(*out));
  void* p[SM_PEER_SLOTS] = {};
  own_ptrs(ctx, p);
  for (int i = 0; i < SM_PEER_USED; i++) {
    out->ptr[i] = (uint64_t)(uintptr_t)p[i];
    if (!p[i]) continue;                      // optional array (mass budget, per-cell maps) not allocated
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
  if (ctx->group) return fail(ctx, SM_ERR_INVALID, "a group manages its ranks' peers itself (sm_group_rank gives the rank contexts)");
  if (!blobs || nblobs != ctx->nranks) return fail(ctx, SM_ERR_INVALID, "sm_peer_attach: one blob per rank");
  for (int q = 0; q < nblobs; q++)   // slot 20: the per-cell budget maps; a step writes into its neighbours' maps
    if ((blobs[q].ptr[20] != 0) != (ctx->d_cells != nullptr))
      return fail(ctx, SM_ERR_INVALID, "sm_peer_attach: the ranks disagree on SM_FLAG_CELL_BUDGET");
  CK(cudaSetDevice(ctx->cfg.device));
  for (int q = 0; q < ctx->nranks; q++) {
    const sm_peer_blob& b = blobs[q];
    if (b.rank != q) return fail(ctx, SM_ERR_INVALID, "sm_peer_attach: blobs must be ordered by rank");
    void* p[SM_PEER_SLOTS] = {};
    if (q != ctx->rank && b.device != ctx->cfg.device) {
      // this rank's kernels dereference the peer's pointers: raw ones of the same process need the access enabled just
      // as IPC mappings do (every rank attaches every other, so both directions get enabled)
      int can = 0;
      CK(cudaDeviceCanAccessPeer(&can, ctx->cfg.device, b.device));
      if (!can) {
        ctx->err = "sm_peer_attach: no peer access between devices " + std::to_string(ctx->cfg.device) + " and " +
                   std::to_string(b.device);
        return SM_ERR_CUDA;
      }
      cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { ctx->err = cudaGetErrorString(e); return SM_ERR_CUDA; }
      cudaGetLastError();      // cudaErrorPeerAccessAlreadyEnabled is sticky until read
    }
    if (q == ctx->rank) {
      own_ptrs(ctx, p);
    } else if (!use_ipc) {
      for (int i = 0; i < SM_PEER_USED; i++) p[i] = (void*)(uintptr_t)b.ptr[i];   // same process
    } else {
      for (int i = 0; i < SM_PEER_USED; i++) {
        if (!b.ptr[i]) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, b.ipc[i], 64);
        CK(cudaIpcOpenMemHandle(&p[i], h, cudaIpcMemLazyEnablePeerAccess));
        ctx->ipc_opened[q][i] = p[i];
      }
    }
    fill_peer(ctx->d.peer[q], p, b.pool_cap);
    ctx->cells_of.p[q] = (double*)p[20];
    ctx->freq_of.wfreq[q] = (float*)p[21];
    ctx->freq_of.wtrack[q] = (float*)p[22];
  }
  ctx->peers_attached = true;
  return SM_OK;
}

int sm_sync(sm_context* ctx) {
  if (ctx->group) return grp_settle(ctx);
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

int sm_set_soils(sm_context* ctx, const sm_soil* soils, int32_t n) {
  if (ctx->group) {
    const int rc = grp_each(ctx, [&](sm_context* c, int) { return sm_set_soils(c, soils, n); });
    if (rc == SM_OK) ctx->nsoils = n;
    return rc;
  }
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
  if (ctx->group) return grp_upload_columns(ctx, offsets, type, size, saturation);
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
  if (ctx->group) {
    int64_t total = 0, part = 0;
    const int rc = grp_settled_each(ctx, [&](sm_context* c, int) { const int rc_ = sm_section_count(c, &part); total += part; return rc_; });
    *n = total;
    return rc;
  }
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
  if (ctx->group) return grp_download_columns(ctx, capacity, offsets, type, size, floor_, saturation);
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
  if (ctx->group) return grp_settled_each(ctx, [&](sm_context* c, int) { return sm_download_height(c, height + (size_t)c->x0 * c->d.dimy); });
  CK(cudaSetDevice(ctx->cfg.device));
  k_heights<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d.top, ctx->d_scratch, nullptr, ctx->lcells);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(height, ctx->d_scratch, ctx->lcells * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

int sm_download_surface(sm_context* ctx, int32_t* surface) {
  if (ctx->group) return grp_settled_each(ctx, [&](sm_context* c, int) { return sm_download_surface(c, surface + (size_t)c->x0 * c->d.dimy); });
  CK(cudaSetDevice(ctx->cfg.device));
  k_heights<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d.top, nullptr, ctx->d_iscratch, ctx->lcells);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(surface, ctx->d_iscratch, ctx->lcells * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

// whole_map: a rank of a sharded map sums every strip through the peer pointers (the caller has settled the ranks)
static int height_sum(sm_context* ctx, bool whole_map, double* sum) {
  CK(cudaSetDevice(ctx->cfg.device));
  if (whole_map) k_height_sum1<true><<<SUM_BLOCKS, 256, 0, ctx->stream>>>(ctx->d, ctx->cells, ctx->d_scratch);
  else k_height_sum1<false><<<SUM_BLOCKS, 256, 0, ctx->stream>>>(ctx->d, ctx->lcells, ctx->d_scratch);
  k_height_sum2<<<1, 256, 0, ctx->stream>>>(ctx->d_scratch, ctx->d_scratch + SUM_BLOCKS);
  ctx->launches += 2;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(sum, ctx->d_scratch + SUM_BLOCKS, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}
int sm_height_sum(sm_context* ctx, double* sum) {
  if (ctx->group) return grp_settled_rank0(ctx, [&](sm_context* c) { return height_sum(c, true, sum); });
  return height_sum(ctx, false, sum);
}

int sm_checksum(sm_context* ctx, uint64_t* out) {
  if (ctx->group) {     // the strips' checksums add up mod 2^64
    if (!out) return fail(ctx, SM_ERR_INVALID, "null argument");
    uint64_t total = 0, part = 0;
    const int rc = grp_settled_each(ctx, [&](sm_context* c, int) { const int rc_ = sm_checksum(c, &part); total += part; return rc_; });
    *out = total;
    return rc;
  }
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
  if (ctx->group) { float* const h[3] = {wf, wt, windf}; return grp_frequency(ctx, false, h); }
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  if (wf) CK(cudaMemcpy(wf, ctx->d.wfreq, ctx->cells * 4, cudaMemcpyDeviceToHost));
  if (wt) CK(cudaMemcpy(wt, ctx->d.wtrack, ctx->cells * 4, cudaMemcpyDeviceToHost));
  if (windf) CK(cudaMemcpy(windf, ctx->d.windfreq, ctx->cells * 4, cudaMemcpyDeviceToHost));
  return SM_OK;
}
int sm_set_frequency(sm_context* ctx, const float* wf, const float* wt, const float* windf) {
  if (ctx->group) { float* const h[3] = {(float*)wf, (float*)wt, (float*)windf}; return grp_frequency(ctx, true, h); }
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  if (wf) CK(cudaMemcpy(ctx->d.wfreq, wf, ctx->cells * 4, cudaMemcpyHostToDevice));
  if (wt) CK(cudaMemcpy(ctx->d.wtrack, wt, ctx->cells * 4, cudaMemcpyHostToDevice));
  if (windf) CK(cudaMemcpy(ctx->d.windfreq, windf, ctx->cells * 4, cudaMemcpyHostToDevice));
  return SM_OK;
}
int sm_frequency_update(sm_context* ctx) {
  if (ctx->group) return grp_each(ctx, [&](sm_context* c, int) { return sm_frequency_update(c); });
  CK(cudaSetDevice(ctx->cfg.device));
  k_frequency_update<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d.wfreq, ctx->d.wtrack, ctx->cells);
  ctx->launches++;
  CK(cudaGetLastError());
  return SM_OK;
}

// ---- single-cell operations -----------------------------------------------------------------------
// calls that read other ranks' strips need the peer pointers
static int peers_ready(sm_context* ctx) {
  if (ctx->nranks > 1 && !ctx->peers_attached) return fail(ctx, SM_ERR_INVALID, "sharded context: call sm_peer_attach first");
  return SM_OK;
}
static int cell_op(sm_context* ctx, const CellOp& o, CellRes* out) {
  if (ctx->group) return grp_cell_op(ctx, o, out);
  if (ctx->nsoils < 1) return fail(ctx, SM_ERR_INVALID, "soil table not set");
  const bool read = o.op == 3 || o.op == 4;
  if (ctx->nranks > 1 && !read) return fail(ctx, SM_ERR_INVALID, "single-cell operations are not available on a sharded context");
  int rc = peers_ready(ctx);
  if (rc != SM_OK) return rc;
  CK(cudaSetDevice(ctx->cfg.device));
  if (!read) k_cell_op<<<1, 1, 0, ctx->stream>>>(ctx->d, o, ctx->d_cellres);
  else if (ctx->nranks > 1) k_cell_read<true><<<1, 1, 0, ctx->stream>>>(ctx->d, o, ctx->d_cellres);
  else k_cell_read<false><<<1, 1, 0, ctx->stream>>>(ctx->d, o, ctx->d_cellres);
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
  if (ctx->group) return grp_settled_rank0(ctx, [&](sm_context* c) { return sm_cell_column(c, x, y, capacity, n, type, size, floor_, saturation); });
  if (!inb(ctx, x, y) || !n || capacity < 0) return fail(ctx, SM_ERR_INVALID, "sm_cell_column: range");
  int rc = peers_ready(ctx);
  if (rc != SM_OK) return rc;
  CK(cudaSetDevice(ctx->cfg.device));
  const int cap = std::min(capacity, 1024);
  Sec32* d_out = nullptr; int* d_n = nullptr;
  CK(cudaMalloc(&d_out, (size_t)std::max(cap, 1) * sizeof(Sec32)));
  if (cudaMalloc(&d_n, sizeof(int)) != cudaSuccess) { cudaFree(d_out); return fail(ctx, SM_ERR_CUDA, "cudaMalloc"); }
  if (ctx->nranks > 1) k_cell_column<true><<<1, 1, 0, ctx->stream>>>(ctx->d, x, y, cap, d_n, d_out);
  else k_cell_column<false><<<1, 1, 0, ctx->stream>>>(ctx->d, x, y, cap, d_n, d_out);
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
  if (ctx->group) return grp_each(ctx, [&](sm_context* c, int) { return sm_set_volume_factor(c, v); });
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
  // Sharded map, new batch: a rank writes a particle's `done` only while it holds the particle, so without this a
  // dead marker of an earlier batch would look like the holder's (the flood finds the holder by it, k_hydro_flood_w).
  // No peer writes into this array before the kernel below has passed its prologue barrier: hand-overs happen in the
  // sweeps, and that barrier waits for every rank.
  if (multi && d_spawn != nullptr && n > 0) CK(cudaMemsetAsync(ctx->d.done, 0, (size_t)n * sizeof(unsigned int), ctx->stream));
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
  // per-cell maps: only the warp kernel keeps them; a batch any of whose launches ran without them has no maps
  if (ctx->d_cells && !use_coop) ctx->cells_state = 2;
  else if (ctx->d_cells && ctx->cells_state == 0) ctx->cells_state = 1;
  if (use_coop) {
    const int sw_warps = kind == KIND_WIND ? SwShape<KIND_WIND>::WARPS : SwShape<KIND_WATER>::WARPS;
    const int cthreads = sw_warps * 32;
    int occ = 0;
    const bool budget = ctx->d.bud != nullptr;
    // SM_EXACT: bit mask of the kinds that use exact footprints (sweep_exact): 1 = water, 2 = wind
    bool exact = false;
    {
      const char* e = getenv("SM_EXACT");
      exact = (((e ? atoi(e) : SM_DEFAULT_EXACT) >> kind) & 1) != 0;
    }
    void* const fns[16] = {(void*)k_sweep<KIND_WATER, false, false, false, false>, (void*)k_sweep<KIND_WIND, false, false, false, false>,
                           (void*)k_sweep<KIND_WATER, true, false, false, false>,  (void*)k_sweep<KIND_WIND, true, false, false, false>,
                           (void*)k_sweep<KIND_WATER, false, true, false, false>,  (void*)k_sweep<KIND_WIND, false, true, false, false>,
                           (void*)k_sweep<KIND_WATER, true, true, false, false>,   (void*)k_sweep<KIND_WIND, true, true, false, false>,
                           (void*)k_sweep<KIND_WATER, false, false, true, false>,  (void*)k_sweep<KIND_WIND, false, false, true, false>,
                           (void*)k_sweep<KIND_WATER, true, false, true, false>,   (void*)k_sweep<KIND_WIND, true, false, true, false>,
                           (void*)k_sweep<KIND_WATER, false, true, true, false>,   (void*)k_sweep<KIND_WIND, false, true, true, false>,
                           (void*)k_sweep<KIND_WATER, true, true, true, false>,    (void*)k_sweep<KIND_WIND, true, true, true, false>};
    // with the per-cell maps (SM_FLAG_CELL_BUDGET, which implies the budget)
    void* const fns_cells[8] = {(void*)k_sweep<KIND_WATER, false, true, false, true>, (void*)k_sweep<KIND_WIND, false, true, false, true>,
                                (void*)k_sweep<KIND_WATER, true, true, false, true>,  (void*)k_sweep<KIND_WIND, true, true, false, true>,
                                (void*)k_sweep<KIND_WATER, false, true, true, true>,  (void*)k_sweep<KIND_WIND, false, true, true, true>,
                                (void*)k_sweep<KIND_WATER, true, true, true, true>,   (void*)k_sweep<KIND_WIND, true, true, true, true>};
    void* fn = ctx->d_cells ? fns_cells[(exact ? 4 : 0) + (multi ? 2 : 0) + (kind == KIND_WATER ? 0 : 1)]
                            : fns[(exact ? 8 : 0) + (budget ? 4 : 0) + (multi ? 2 : 0) + (kind == KIND_WATER ? 0 : 1)];
    // dynamic shared memory: the live mask of the batch and its popcount prefix (2 x n/32 words per block)
    const size_t csmem = (size_t)2 * (((size_t)std::max(n, 1) + 31) / 32) * sizeof(unsigned int);
    if (csmem > 40 * 1024) CK(cudaFuncSetAttribute((const void*)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)csmem));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void*)fn, cthreads, csmem));
    if (occ < 1) return fail(ctx, SM_ERR_CUDA, "sweep kernel does not fit an SM");
    // contexts that share the device must all be resident at once (they meet in the cross-rank barrier)
    const long long maxblocks = std::max<long long>(1, (long long)ctx->num_sms * occ / ctx->share);
    const long long want = ((long long)std::max(n, 1) + sw_warps - 1) / sw_warps;
    const int cblocks = (int)std::max<long long>(1, std::min(maxblocks, want));
    DevCtx dd = ctx->d;
    int ms = max_sweeps;
    if (ms <= 0) ms = -1;
    if (max_sweeps == SM_SWEEPS_NONE) ms = 0;
    CellMaps cm = ctx->cells_of;
    void* cargs[] = {&dd, &n, (void*)&d_spawn, &ms, &cm};
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
  if (ctx->group) return grp_last_stats(ctx, st);
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
  if (h.err & (1u << 6)) return fail(ctx, SM_ERR_REACH, "a waiter acquired a hand-off that was not released (audit build)");
  if (h.err & (1u << 3)) return fail(ctx, SM_ERR_POOL, "section pool exhausted (sections were dropped)");
  return SM_OK;
}

// a new batch (*_run, *_run_device, *_begin): the per-cell maps start from +0.0; *_sweeps adds onto them
static int new_batch(sm_context* ctx, int kind, int n) {
  ctx->cur_kind = kind; ctx->cur_n = n;
  if (ctx->d_cells) {
    ctx->cells_state = 0;
    CK(cudaMemsetAsync(ctx->d_cells, 0, ctx->lcells * 3 * sizeof(double), ctx->stream));
  }
  return SM_OK;
}

static int run_host(sm_context* ctx, int kind, int n, const float* spawn_xy, int max_sweeps, sm_stats* st) {
  if (ctx->group) {
    const int rc = grp_run(ctx, kind, n, spawn_xy, nullptr, max_sweeps, true);
    return rc != SM_OK ? rc : grp_last_stats(ctx, st);
  }
  if (n > 0 && !spawn_xy) return fail(ctx, SM_ERR_INVALID, "null spawn list");
  if (ctx->nranks > 1 && ctx->share > 1)
    return fail(ctx, SM_ERR_INVALID, "contexts sharing a device must use sm_*_run_device on every rank, then sm_last_stats");
  if (n < 0 || n > ctx->max_particles) return fail(ctx, SM_ERR_INVALID, "batch larger than max_particles");
  CK(cudaSetDevice(ctx->cfg.device));
  if (n) CK(cudaMemcpyAsync(ctx->d_spawn, spawn_xy, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  int rc = zero_counters(ctx);
  if (rc != SM_OK) return rc;
  rc = new_batch(ctx, kind, n);
  if (rc != SM_OK) return rc;
  rc = launch_run(ctx, kind, n, ctx->d_spawn, max_sweeps);
  if (rc != SM_OK) return rc;
  return sm_last_stats(ctx, st);
}

// ---- mass budget (SURVEY.md A.7) --------------------------------------------------------------------------
int sm_budget_particles(sm_context* ctx, int32_t n, double* out) {
  if (ctx->group) return grp_budget_particles(ctx, n, out);
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

int sm_last_cell_budget(sm_context* ctx, double* eroded, double* deposited, double* cascade_net) {
  if (ctx->group)
    return grp_settled_each(ctx, [&](sm_context* c, int) {
      const size_t lo = (size_t)c->x0 * c->d.dimy;
      return sm_last_cell_budget(c, eroded ? eroded + lo : nullptr, deposited ? deposited + lo : nullptr,
                                 cascade_net ? cascade_net + lo : nullptr);
    });
  if (!ctx->d_cells) return fail(ctx, SM_ERR_INVALID, "context was created without SM_FLAG_CELL_BUDGET");
  if (ctx->cells_state == 0) return fail(ctx, SM_ERR_INVALID, "no batch yet");
  if (ctx->cells_state == 2)
    return fail(ctx, SM_ERR_INVALID, "the last batch ran on a kernel without the per-cell maps (SM_KERNEL=thread)");
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  std::vector<double> m(ctx->lcells * 3);
  CK(cudaMemcpy(m.data(), ctx->d_cells, m.size() * sizeof(double), cudaMemcpyDeviceToHost));
  double* const out[3] = {eroded, deposited, cascade_net};
  for (int k = 0; k < 3; k++)
    if (out[k]) for (size_t i = 0; i < ctx->lcells; i++) out[k][i] = m[i * 3 + k];
  return SM_OK;
}

int sm_water_run(sm_context* ctx, int32_t n, const float* xy, int32_t max_sweeps, sm_stats* st) {
  return run_host(ctx, KIND_WATER, n, xy, max_sweeps, st);
}
int sm_wind_run(sm_context* ctx, int32_t n, const float* xy, int32_t max_sweeps, sm_stats* st) {
  return run_host(ctx, KIND_WIND, n, xy, max_sweeps, st);
}
int sm_water_run_device(sm_context* ctx, int32_t n, const float* d_xy, int32_t max_sweeps) {
  if (ctx->group) return grp_run(ctx, KIND_WATER, n, nullptr, d_xy, max_sweeps, true);
  int rc = zero_counters(ctx);
  if (rc != SM_OK) return rc;
  rc = new_batch(ctx, KIND_WATER, n);
  if (rc != SM_OK) return rc;
  return launch_run(ctx, KIND_WATER, n, d_xy, max_sweeps);
}
int sm_wind_run_device(sm_context* ctx, int32_t n, const float* d_xy, int32_t max_sweeps) {
  if (ctx->group) return grp_run(ctx, KIND_WIND, n, nullptr, d_xy, max_sweeps, true);
  int rc = zero_counters(ctx);
  if (rc != SM_OK) return rc;
  rc = new_batch(ctx, KIND_WIND, n);
  if (rc != SM_OK) return rc;
  return launch_run(ctx, KIND_WIND, n, d_xy, max_sweeps);
}

// ---- pooling hydrology ----------------------------------------------------------------------------
// SM_HYDRO=warp | thread selects the executor of the flood phase and the seep pass.  A sharded context always runs the
// warp executor (its MULTI instantiations; DESIGN.md section 7).  A context created with
// SM_FLAG_BUDGET runs the warp executor whatever SM_HYDRO says: the hydrology's budget lives only there, as the
// batches' budget lives only in the warp sweep kernel.  SM_FLAG_HYDRO_CELL_BUDGET runs its CELLS instantiations.
static bool hydro_warp() {
  const char* e = getenv("SM_HYDRO");
  if (e && strcmp(e, "warp") == 0) return true;
  if (e && strcmp(e, "thread") == 0) return false;
  return false;     // without a record cache the warp executor's seep pass does not keep up with the one-thread
                    // executor and its shared-memory cache
}
static int hydro_ready(sm_context* ctx) {
  if (ctx->nsoils < 1) return fail(ctx, SM_ERR_INVALID, "soil table not set");
  // Sharded: the call works on the whole map, so exactly one rank may make it, while the others leave the map alone.
  // Ranks usually make the same calls in lockstep; a rank only issues the hydrology once it has been named the issuer,
  // so a symmetric call on every rank is refused instead of running N floods on the same map at once.
  if (ctx->nranks > 1 && !ctx->hydro_issuer)
    return fail(ctx, SM_ERR_INVALID, "pooling hydrology is not available on a sharded context that is not the issuing rank (sm_hydro_issuer)");
  if (ctx->nranks > 1 && !ctx->peers_attached) return fail(ctx, SM_ERR_INVALID, "sharded context: call sm_peer_attach first");
  CK(cudaSetDevice(ctx->cfg.device));
  if (!ctx->d_hydro) {
    CK(cudaMalloc(&ctx->d_hydro, sizeof(HydroTotals)));
    CK(cudaFuncSetAttribute(k_hydro_flood, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_HC_BYTES));
    CK(cudaFuncSetAttribute(k_hydro_seep, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_HC_BYTES));
  }
  // status and drop counter are per call (see zero_counters)
  CK(cudaMemsetAsync(&ctx->d.ctl->err, 0, sizeof(unsigned int), ctx->stream));
  CK(cudaMemsetAsync(&ctx->d.ctl->drops, 0, sizeof(unsigned long long), ctx->stream));
  return SM_OK;
}
static int hydro_finish(sm_context* ctx, sm_hydro_stats* st) {
  HydroTotals tot;
  const HydroCount& hc = tot.hc;
  const bool budget = ctx->d.bud != nullptr;
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(cudaMemcpyAsync(&tot, ctx->d_hydro, budget ? sizeof(tot) : sizeof(hc), cudaMemcpyDeviceToHost, ctx->stream));
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
  if (budget) {
    for (int k = 0; k < SM_HYDRO_BUDGET_SLOTS; k++) ctx->hydro_bud[k] = tot.bud[k];
    ctx->hydro_bud_valid = true;
  }
  if (ctx->d_hcells) ctx->hcells_state = 1;
  return SM_OK;
}
// the per-cell maps start every call at +0.0; until the call has succeeded they are partial
static int hydro_cells_reset(sm_context* ctx) {
  if (!ctx->d_hcells) return SM_OK;
  ctx->hcells_state = 2;
  CK(cudaMemsetAsync(ctx->d_hcells, 0, ctx->cells * SM_HYDRO_CELL_TERMS * sizeof(double), ctx->stream));
  return SM_OK;
}
int sm_hydro_issuer(sm_context* ctx, int32_t on) {
  if (ctx->group) return fail(ctx, SM_ERR_INVALID, "a group issues the pooling hydrology from its rank 0");
  ctx->hydro_issuer = on != 0;
  return SM_OK;
}
int sm_water_flood(sm_context* ctx, sm_hydro_stats* st) {
  if (ctx->group) {
    if (ctx->cur_kind != KIND_WATER) return fail(ctx, SM_ERR_INVALID, "sm_water_flood: the last batch was not a water batch");
    return grp_hydro(ctx, [&](sm_context* c) { return sm_water_flood(c, st); });
  }
  int rc = hydro_ready(ctx);
  if (rc != SM_OK) return rc;
  if (ctx->cur_kind != KIND_WATER) return fail(ctx, SM_ERR_INVALID, "sm_water_flood: the last batch was not a water batch");
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  rc = hydro_cells_reset(ctx);        // inside the call's device time: the maps' whole cost
  if (rc != SM_OK) return rc;
  const FreqPeers& fp = ctx->freq_of;
  if (ctx->nranks > 1) {     // sharded: the warp executor, whatever SM_HYDRO says
    if (ctx->d.bud) k_hydro_flood_w<true, true><<<1, 32, 0, ctx->stream>>>(ctx->d, ctx->cur_n, ctx->d_hydro, nullptr, fp);
    else k_hydro_flood_w<true, false><<<1, 32, 0, ctx->stream>>>(ctx->d, ctx->cur_n, ctx->d_hydro, nullptr, fp);
  }
  else if (ctx->d_hcells) k_hydro_flood_w<false, true, true><<<1, 32, 0, ctx->stream>>>(ctx->d, ctx->cur_n, ctx->d_hydro, ctx->d_hcells, fp);
  else if (ctx->d.bud) k_hydro_flood_w<false, true><<<1, 32, 0, ctx->stream>>>(ctx->d, ctx->cur_n, ctx->d_hydro, nullptr, fp);
  else if (hydro_warp()) k_hydro_flood_w<false, false><<<1, 32, 0, ctx->stream>>>(ctx->d, ctx->cur_n, ctx->d_hydro, nullptr, fp);
  else k_hydro_flood<<<1, 32, SM_HC_BYTES, ctx->stream>>>(ctx->d, ctx->cur_n, &ctx->d_hydro->hc);
  ctx->launches++;
  CK(cudaGetLastError());
  return hydro_finish(ctx, st);
}
int sm_seep(sm_context* ctx, sm_hydro_stats* st) {
  if (ctx->group) return grp_hydro(ctx, [&](sm_context* c) { return sm_seep(c, st); });
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
  rc = hydro_cells_reset(ctx);        // inside the call's device time: the maps' whole cost
  if (rc != SM_OK) return rc;
  CK(cudaMemsetAsync(ctx->d_act, 0, total * sizeof(unsigned long long), ctx->stream));
  CK(cudaEventRecord(ctx->evt0, ctx->stream));
  const FreqPeers& fp = ctx->freq_of;
  if (ctx->nranks > 1) {     // sharded: the whole map, each column read at its owner; then the warp executor
    k_hydro_classify<true><<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, am);
    CK(cudaEventRecord(ctx->evt1, ctx->stream));
    if (ctx->d.bud) k_hydro_seep_w<true, true><<<1, 32, 0, ctx->stream>>>(ctx->d, am, ctx->d_hydro, nullptr, fp);
    else k_hydro_seep_w<true, false><<<1, 32, 0, ctx->stream>>>(ctx->d, am, ctx->d_hydro, nullptr, fp);
  } else {
    k_hydro_classify<false><<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, am);
    CK(cudaEventRecord(ctx->evt1, ctx->stream));
    if (ctx->d_hcells) k_hydro_seep_w<false, true, true><<<1, 32, 0, ctx->stream>>>(ctx->d, am, ctx->d_hydro, ctx->d_hcells, fp);
    else if (ctx->d.bud) k_hydro_seep_w<false, true><<<1, 32, 0, ctx->stream>>>(ctx->d, am, ctx->d_hydro, nullptr, fp);
    else if (hydro_warp()) k_hydro_seep_w<false, false><<<1, 32, 0, ctx->stream>>>(ctx->d, am, ctx->d_hydro, nullptr, fp);
    else k_hydro_seep<<<1, 32, SM_HC_BYTES, ctx->stream>>>(ctx->d, am, &ctx->d_hydro->hc);
  }
  ctx->launches += 2;
  CK(cudaGetLastError());
  int rc2 = hydro_finish(ctx, st);
  if (st) {     // the full-grid classification alone (the HBM-bound part of the pass)
    float cms = 0.f;
    if (cudaEventElapsedTime(&cms, ctx->evt0, ctx->evt1) == cudaSuccess) st->classify_ms = cms;
  }
  return rc2;
}
int sm_last_hydro_budget(sm_context* ctx, sm_hydro_budget* out) {
  if (ctx->group) return grp_rank0(ctx, [&](sm_context* c) { return sm_last_hydro_budget(c, out); });
  if (!out) return fail(ctx, SM_ERR_INVALID, "null argument");
  if (!ctx->d.bud) return fail(ctx, SM_ERR_INVALID, "context was created without SM_FLAG_BUDGET");
  if (!ctx->hydro_bud_valid) return fail(ctx, SM_ERR_INVALID, "no hydrology call yet");
  const double* b = ctx->hydro_bud;
  out->flood_sediment = b[0]; out->flood_cascade_net = b[1]; out->flood_water = b[2]; out->seeped = b[3];
  out->to_particles = b[4]; out->transfer_net = b[5]; out->nested_eroded = b[6]; out->nested_deposited = b[7];
  out->nested_cascade_net = b[8]; out->nested_discarded = b[9]; out->nested_clamped = b[10];
  return SM_OK;
}
int sm_last_hydro_cell_budget(sm_context* ctx, double* eroded, double* deposited, double* cascade_net, double* water_net) {
  if (!ctx->d_hcells) return fail(ctx, SM_ERR_INVALID, "context was created without SM_FLAG_HYDRO_CELL_BUDGET");
  if (ctx->hcells_state == 0) return fail(ctx, SM_ERR_INVALID, "no hydrology call yet (sm_water_flood or sm_seep)");
  if (ctx->hcells_state == 2)
    return fail(ctx, SM_ERR_INVALID, "the last hydrology call failed: its per-cell maps are partial");
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  // de-interleaved through a bounded host buffer (32 MB), not a host copy of the whole map
  const size_t chunk = (size_t)1 << 20;
  std::vector<double> m(std::min(ctx->cells, chunk) * SM_HYDRO_CELL_TERMS);
  double* const out[SM_HYDRO_CELL_TERMS] = {eroded, deposited, cascade_net, water_net};
  for (size_t c0 = 0; c0 < ctx->cells; c0 += chunk) {
    const size_t n = std::min(chunk, ctx->cells - c0);
    CK(cudaMemcpy(m.data(), ctx->d_hcells + c0 * SM_HYDRO_CELL_TERMS, n * SM_HYDRO_CELL_TERMS * sizeof(double),
                  cudaMemcpyDeviceToHost));
    for (int k = 0; k < SM_HYDRO_CELL_TERMS; k++)
      if (out[k]) for (size_t i = 0; i < n; i++) out[k][c0 + i] = m[i * SM_HYDRO_CELL_TERMS + k];
  }
  return SM_OK;
}

// ---- sweep floods: a water batch whose particles flood at the end of the sweep they stop in -------------------------
// Every sweep is one launch of the sweep kernel (max_sweeps = 1; the first spawns, the others resume), followed on the
// issuing context's stream by k_flood_gate and k_hydro_flood_sweep.  Segments are enqueued in rounds; the live count
// is read back once per round, so the host waits once per round, not once per sweep.  A launch after the batch has
// ended finds no live particle and no candidate and returns at once.  DESIGN.md K6 "Sweep floods".
static int flood_phase(sm_context* ctx, int n) {
  const int blocks = (int)std::max<long long>(1, std::min<long long>(((long long)n + 255) / 256, (long long)ctx->num_sms * 4));
  const FreqPeers& fp = ctx->freq_of;
  if (ctx->nranks > 1) {
    k_flood_gate<true><<<blocks, 256, 0, ctx->stream>>>(ctx->d, n, ctx->d_gate);
    if (ctx->d.bud) k_hydro_flood_sweep<true, true><<<1, 32, 0, ctx->stream>>>(ctx->d, n, ctx->d_hydro, nullptr, fp, ctx->d_gate);
    else k_hydro_flood_sweep<true, false><<<1, 32, 0, ctx->stream>>>(ctx->d, n, ctx->d_hydro, nullptr, fp, ctx->d_gate);
  } else {
    k_flood_gate<false><<<blocks, 256, 0, ctx->stream>>>(ctx->d, n, ctx->d_gate);
    if (ctx->d_hcells)
      k_hydro_flood_sweep<false, true, true><<<1, 32, 0, ctx->stream>>>(ctx->d, n, ctx->d_hydro, ctx->d_hcells, fp, ctx->d_gate);
    else if (ctx->d.bud) k_hydro_flood_sweep<false, true><<<1, 32, 0, ctx->stream>>>(ctx->d, n, ctx->d_hydro, nullptr, fp, ctx->d_gate);
    else k_hydro_flood_sweep<false, false><<<1, 32, 0, ctx->stream>>>(ctx->d, n, ctx->d_hydro, nullptr, fp, ctx->d_gate);
  }
  ctx->launches += 2;
  CK(cudaGetLastError());
  return SM_OK;
}
// one sweep of the batch and the floods of the particles that stopped in it
static int flood_segment(sm_context* ctx, int n, const float* h_xy, bool first) {
  if (!ctx->group) {
    const int rc = launch_run(ctx, KIND_WATER, n, first ? ctx->d_spawn : nullptr, 1);
    return rc != SM_OK ? rc : flood_phase(ctx, n);
  }
  sm_group& G = *ctx->group;
  sm_context* const c0 = G.rank[0];
  int rc = first ? grp_run(ctx, KIND_WATER, n, h_xy, nullptr, 1, true)
                 : grp_each(ctx, [&](sm_context* c, int) { return launch_run(c, KIND_WATER, c->cur_n, nullptr, 1); });
  if (rc != SM_OK) return rc;
  // the flood reads and writes every strip: rank 0 waits for every rank's sweep, every rank's next sweep for the flood
  for (int r = 1; r < G.n; r++) {
    sm_context* const c = G.rank[r];
    CK(cudaSetDevice(c->cfg.device));
    CK(cudaEventRecord(c->evt0, c->stream));
    CK(cudaSetDevice(c0->cfg.device));
    CK(cudaStreamWaitEvent(c0->stream, c->evt0, 0));
  }
  rc = flood_phase(c0, n);
  if (rc != SM_OK) return grp_err(ctx, 0, rc);
  CK(cudaEventRecord(G.ev, c0->stream));
  for (int r = 1; r < G.n; r++) {
    sm_context* const c = G.rank[r];
    CK(cudaSetDevice(c->cfg.device));
    CK(cudaStreamWaitEvent(c->stream, G.ev, 0));
  }
  return SM_OK;
}
int sm_water_run_flooding(sm_context* ctx, int32_t n, const float* xy, int32_t max_sweeps, sm_stats* st,
                          sm_hydro_stats* hst) {
  if (!ctx->group && ctx->nranks > 1)
    return fail(ctx, SM_ERR_INVALID, "sm_water_run_flooding: not available on a rank of a sharded map (use a group)");
  if (n < 0 || n > ctx->max_particles) return fail(ctx, SM_ERR_INVALID, "batch larger than max_particles");
  if (n > 0 && !xy) return fail(ctx, SM_ERR_INVALID, "null spawn list");
  sm_context* const c0 = ctx->group ? ctx->group->rank[0] : ctx;
  int rc = hydro_ready(c0);
  if (rc != SM_OK) return ctx->group ? grp_err(ctx, 0, rc) : rc;
  if (!c0->d_gate) CK(cudaMalloc(&c0->d_gate, sizeof(FloodGate)));
  CK(cudaEventRecord(c0->evt0, c0->stream));
  rc = hydro_cells_reset(c0);
  if (rc != SM_OK) return rc;
  CK(cudaMemsetAsync(c0->d_gate, 0, sizeof(FloodGate), c0->stream));
  if (n == 0) CK(cudaMemsetAsync(&c0->d_gate->ended, 1, 1, c0->stream));
  CK(cudaMemsetAsync(c0->d_hydro, 0, sizeof(HydroTotals), c0->stream));
  if (!ctx->group) {
    if (n) CK(cudaMemcpyAsync(ctx->d_spawn, xy, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    rc = zero_counters(ctx);
    if (rc == SM_OK) rc = new_batch(ctx, KIND_WATER, n);
    if (rc != SM_OK) return rc;
  }
  long long done = 0;
  for (int round = 16;; round = std::min(2 * round, 256)) {
    const long long k = max_sweeps > 0 ? std::min<long long>(round, (long long)max_sweeps - done) : round;
    for (long long j = 0; j < k; j++) {
      rc = flood_segment(ctx, n, xy, done + j == 0);
      if (rc != SM_OK) return rc;
    }
    done += k;
    if (max_sweeps > 0 && done >= max_sweeps) break;
    CK(cudaSetDevice(c0->cfg.device));
    CK(cudaMemcpyAsync(&c0->h_ctl->alive, &c0->d.ctl->alive, sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                             c0->stream));
    CK(cudaStreamSynchronize(c0->stream));
    if (c0->h_ctl->alive == 0) break;
  }
  // the batch's sweep count replaces what the last launch counted (sm_last_stats reads it from the issuer's counters)
  CK(cudaSetDevice(c0->cfg.device));
  CK(cudaMemcpyAsync(&c0->d.ctl->sweeps, &c0->d_gate->sweeps, sizeof(unsigned long long), cudaMemcpyDeviceToDevice,
                           c0->stream));
  CK(cudaEventRecord(c0->evt1, c0->stream));
  sm_stats s;
  memset(&s, 0, sizeof(s));
  rc = ctx->group ? grp_last_stats(ctx, &s) : sm_last_stats(ctx, &s);
  sm_hydro_stats h;
  memset(&h, 0, sizeof(h));
  const int hrc = hydro_finish(c0, &h);
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, c0->evt0, c0->evt1));
  s.device_ms = ms;
  h.device_ms = ms;
  h.classify_ms = 0.0;
  if (st) *st = s;
  if (hst) *hst = h;
  if (ctx->group) for (int r = 0; r < ctx->group->n; r++) ctx->group->rank[r]->mesh_valid = false;
  if (rc != SM_OK) return rc;
  return hrc != SM_OK && ctx->group ? grp_err(ctx, 0, hrc) : hrc;
}

// stepping interface: *_begin runs the prologue only (spawn + bins), *_sweeps(k) resumes the batch
int sm_water_begin(sm_context* ctx, int32_t n, const float* xy) {
  return run_host(ctx, KIND_WATER, n, xy, SM_SWEEPS_NONE, nullptr);
}
int sm_wind_begin(sm_context* ctx, int32_t n, const float* xy) {
  return run_host(ctx, KIND_WIND, n, xy, SM_SWEEPS_NONE, nullptr);
}
static int sweeps_k(sm_context* ctx, int kind, int k, sm_stats* st) {
  if (ctx->group) return grp_sweeps(ctx, kind, k, st);
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
  if (ctx->group) return grp_fetch_state(ctx, a, b, c, al);
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
  if (ctx->group) return grp_each(ctx, [&](sm_context* c, int) { return sm_set_soil_colors(c, rgba, n); });
  if (!rgba || n < 1 || n > SM_MAX_SOILS) return fail(ctx, SM_ERR_INVALID, "sm_set_soil_colors: 1..64 soils");
  CK(cudaSetDevice(ctx->cfg.device));
  if (!ctx->d_colors) CK(cudaMalloc(&ctx->d_colors, SM_MAX_SOILS * sizeof(float4)));
  CK(cudaMemcpy(ctx->d_colors, rgba, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice));
  return SM_OK;
}
int sm_mesh_update(sm_context* ctx, int32_t slice, float* host_vertices) {
  if (ctx->group)
    return grp_settled_each(ctx, [&](sm_context* c, int) {
      return sm_mesh_update(c, slice, host_vertices ? host_vertices + (size_t)c->x0 * c->d.dimy * 11 : nullptr);
    });
  if (!ctx->d_colors) return fail(ctx, SM_ERR_INVALID, "sm_mesh_update: soil colours not set");
  int rc = peers_ready(ctx);
  if (rc != SM_OK) return rc;
  CK(cudaSetDevice(ctx->cfg.device));
  if (!ctx->d_verts) CK(cudaMalloc(&ctx->d_verts, ctx->lcells * 11 * sizeof(float)));
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  if (ctx->nranks > 1) k_mesh<true><<<ctx->num_sms * 16, MESH_BLOCK, 0, ctx->stream>>>(ctx->d, slice, ctx->d_colors, ctx->d_verts);
  else k_mesh<false><<<ctx->num_sms * 16, MESH_BLOCK, 0, ctx->stream>>>(ctx->d, slice, ctx->d_colors, ctx->d_verts);
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  ctx->launches++;
  ctx->timing_pending = true;
  ctx->mesh_valid = true;
  CK(cudaGetLastError());
  if (host_vertices) {
    CK(cudaMemcpyAsync(host_vertices, ctx->d_verts, ctx->lcells * 11 * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  return SM_OK;
}
int sm_mesh_device_ptr(sm_context* ctx, void** dptr) {
  if (ctx->group)
    return fail(ctx, SM_ERR_INVALID, "sm_mesh_device_ptr: a group of several ranks has no single device array "
                                     "(sm_group_rank gives the ranks, each with its strip's pointer)");
  if (!ctx->mesh_valid) return fail(ctx, SM_ERR_INVALID, "no mesh yet: call sm_mesh_update");
  *dptr = ctx->d_verts;
  return SM_OK;
}
static int export_maps(sm_context* ctx, float* height, float* bgra) {
  if (!ctx->mesh_valid) return fail(ctx, SM_ERR_INVALID, "no mesh yet: call sm_mesh_update");
  CK(cudaSetDevice(ctx->cfg.device));
  float* d_out = nullptr;
  const size_t n = ctx->lcells * (height ? 1 : 4);
  CK(cudaMalloc(&d_out, n * sizeof(float)));
  k_export<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d_verts, ctx->lcells, ctx->d.scale, height ? d_out : nullptr,
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
  if (ctx->group) return grp_each(ctx, [&](sm_context* c, int) { return sm_export_height(c, height + (size_t)c->x0 * c->d.dimy); });
  return export_maps(ctx, height, nullptr);
}
int sm_export_color(sm_context* ctx, float* bgra) {
  if (!bgra) return fail(ctx, SM_ERR_INVALID, "null buffer");
  if (ctx->group) return grp_each(ctx, [&](sm_context* c, int) { return sm_export_color(c, bgra + (size_t)c->x0 * c->d.dimy * 4); });
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
static int lbm_ready(sm_context* ctx) {
  if (!ctx->lbm.F[0]) return fail(ctx, SM_ERR_INVALID, "no wind field: call sm_lbm_create");
  CK(cudaSetDevice(ctx->cfg.device));
  return SM_OK;
}
int sm_lbm_init(sm_context* ctx) {
  if (ctx->group) return grp_each(ctx, [&](sm_context* c, int) { return sm_lbm_init(c); });
  int rc = lbm_ready(ctx);
  if (rc != SM_OK) return rc;
  ctx->lbm_cur = 0;
  k_lbm_init<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->lbm, 0);
  ctx->launches++;
  CK(cudaGetLastError());
  return SM_OK;
}
int sm_lbm_create(sm_context* ctx, int32_t nx, int32_t ny, int32_t nz) {
  if (ctx->group) return grp_each(ctx, [&](sm_context* c, int) { return sm_lbm_create(c, nx, ny, nz); });
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
  if (ctx->group) {     // from the terrain: every rank reads the whole map
    const int rc = boundary ? SM_OK : grp_settle(ctx);
    return rc != SM_OK ? rc : grp_each(ctx, [&](sm_context* c, int) { return sm_lbm_set_boundary(c, boundary); });
  }
  int rc = lbm_ready(ctx);
  if (rc != SM_OK) return rc;
  const size_t n = (size_t)ctx->lbm.nx * ctx->lbm.ny * ctx->lbm.nz;
  if (boundary) {
    CK(cudaMemcpyAsync(ctx->lbm.B, boundary, n * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  } else {                       // from the terrain of the whole map (every rank of a sharded map builds all of it)
    rc = peers_ready(ctx);
    if (rc != SM_OK) return rc;
    if (ctx->nranks > 1) k_lbm_boundary_from_map<true><<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, ctx->lbm);
    else k_lbm_boundary_from_map<false><<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, ctx->lbm);
    ctx->launches++;
    CK(cudaGetLastError());
  }
  return SM_OK;
}
int sm_lbm_step(sm_context* ctx, int32_t nsteps, double* device_ms) {
  if (ctx->group) {     // every rank steps its copy of the lattice; the slowest rank's time
    double worst = 0.0, ms = 0.0;
    const int rc = grp_each(ctx, [&](sm_context* c, int) { const int rc_ = sm_lbm_step(c, nsteps, &ms); worst = std::max(worst, ms); return rc_; });
    if (device_ms) *device_ms = worst;
    return rc;
  }
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
  if (ctx->group) return grp_rank0(ctx, [&](sm_context* c) { return sm_lbm_get(c, f, rho, v4); });
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
  if (ctx->group) return grp_each(ctx, [&](sm_context* c, int) { return sm_wind_use_lbm(c, on); });
  if (!on) { ctx->d.wind_v4 = nullptr; return SM_OK; }
  int rc = lbm_ready(ctx);
  if (rc != SM_OK) return rc;
  ctx->d.wind_v4 = (const float*)ctx->lbm.V;
  ctx->d.wind_nx = ctx->lbm.nx; ctx->d.wind_ny = ctx->lbm.ny; ctx->d.wind_nz = ctx->lbm.nz;
  return SM_OK;
}
int sm_lbm_advect(sm_context* ctx, int32_t n, float* pos4) {
  if (ctx->group) return grp_rank0(ctx, [&](sm_context* c) { return sm_lbm_advect(c, n, pos4); });
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
  if (ctx->group) return grp_rank0(ctx, [&](sm_context* c) { return sm_timer_start(c); });
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaEventRecord(ctx->evt0, ctx->stream));
  return SM_OK;
}
int sm_timer_stop(sm_context* ctx, double* elapsed_ms) {
  if (ctx->group) return grp_rank0(ctx, [&](sm_context* c) { return sm_timer_stop(c, elapsed_ms); });
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaEventRecord(ctx->evt1, ctx->stream));
  CK(cudaEventSynchronize(ctx->evt1));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, ctx->evt0, ctx->evt1));
  if (elapsed_ms) *elapsed_ms = ms;
  return SM_OK;
}
int sm_launch_count(sm_context* ctx, int64_t* n) {
  *n = ctx->launches;
  if (ctx->group) for (int r = 0; r < ctx->group->n; r++) *n += ctx->group->rank[r]->launches;
  return SM_OK;
}
// debug (only meaningful in a -DSM_PROFILE build): clock64() totals per phase, summed over particles
// -DSM_PROFILE builds of k_sweep: 8 words per sweep - live particles, max step cycles, max wait cycles, max cycles a
// warp spent on its particles, sum of step cycles, steps, globaltimer at the first warp's start, at the last warp's end
int sm_debug_sweeps8(sm_context* ctx, uint64_t* out, int nsweeps) {
  if (ctx->group) return grp_rank0(ctx, [&](sm_context* c) { return sm_debug_sweeps8(c, out, nsweeps); });
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaMemcpy(out, ctx->d.dbg, (size_t)std::min(nsweeps, 16384) * 64, cudaMemcpyDeviceToHost));
  CK(cudaMemset(ctx->d.dbg, 0, 8 * 16384 * sizeof(unsigned long long)));
  return SM_OK;
}
int sm_debug_sweeps(sm_context* ctx, uint64_t* out, int nsweeps) {   // -DSM_PROFILE builds: (clock64, alive) per sweep
  if (ctx->group) return grp_rank0(ctx, [&](sm_context* c) { return sm_debug_sweeps(c, out, nsweeps); });
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaMemcpy(out, ctx->d.dbg, (size_t)std::min(nsweeps, 16384) * 16, cudaMemcpyDeviceToHost));
  return SM_OK;
}
int sm_debug_profile(sm_context* ctx, uint64_t* out16, int reset) {
  if (ctx->group) return grp_rank0(ctx, [&](sm_context* c) { return sm_debug_profile(c, out16, reset); });
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
  if (ctx->group) return grp_rank0(ctx, [&](sm_context* c) { return sm_device_alloc(c, bytes, dptr); });
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaMalloc(dptr, (size_t)bytes));
  return SM_OK;
}
int sm_device_free(sm_context* ctx, void* dptr) {
  if (ctx->group) return grp_rank0(ctx, [&](sm_context* c) { return sm_device_free(c, dptr); });
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaFree(dptr));
  return SM_OK;
}
int sm_device_upload(sm_context* ctx, void* dptr, const void* host, int64_t bytes) {
  if (ctx->group) return grp_rank0(ctx, [&](sm_context* c) { return sm_device_upload(c, dptr, host, bytes); });
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaMemcpyAsync(dptr, host, (size_t)bytes, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

int sm_initialize(sm_context* ctx, int32_t seed, const sm_layer* layers, int32_t nlayers) {
  if (ctx->group) return grp_each(ctx, [&](sm_context* c, int) { return sm_initialize(c, seed, layers, nlayers); });
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

// ---- snapshots (sm_snap.cuh, DESIGN.md section 10) ---------------------------------------------------------------
// A save to host memory packs the records through this much device memory at a time, cell range by cell range.
#define SNAP_STAGE_BYTES (32ull << 20)

namespace {
struct DevTmp {      // device allocations of one snapshot call, freed when the call returns
  int device = 0;
  std::vector<void*> p;
  DevTmp() = default;
  DevTmp(const DevTmp&) = delete;
  DevTmp& operator=(const DevTmp&) = delete;
  ~DevTmp() {
    if (p.empty()) return;
    cudaSetDevice(device);
    for (void* q : p) cudaFree(q);
  }
};
}  // namespace

static int snap_alloc(sm_context* ctx, DevTmp& t, size_t bytes, void** out) {
  t.device = ctx->cfg.device;
  CK(cudaMalloc(out, std::max<size_t>(bytes, 32)));
  t.p.push_back(*out);
  return SM_OK;
}
// in-place exclusive sum of d[0, n)
static int snap_scan(sm_context* ctx, DevTmp& t, unsigned long long* d, size_t n) {
  size_t tb = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, tb, d, d, (int64_t)n, ctx->stream));
  void* tmp = nullptr;
  const int rc = snap_alloc(ctx, t, tb, &tmp);
  if (rc != SM_OK) return rc;
  CK(cub::DeviceScan::ExclusiveSum(tmp, tb, d, d, (int64_t)n, ctx->stream));
  ctx->launches += 2;      // CUB's initialisation and scan kernels
  return SM_OK;
}
// the count pass: *d_off = the offsets of this context's strip on the device, *nsec = its sections
static int snap_count(sm_context* ctx, DevTmp& t, unsigned long long** d_off, uint64_t* nsec) {
  CK(cudaSetDevice(ctx->cfg.device));
  int rc = snap_alloc(ctx, t, (ctx->lcells + 1) * 8, (void**)d_off);
  if (rc != SM_OK) return rc;
  k_snap_count<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, ctx->lcells, *d_off);
  ctx->launches++;
  CK(cudaGetLastError());
  rc = snap_scan(ctx, t, *d_off, ctx->lcells + 1);
  if (rc != SM_OK) return rc;
  unsigned long long n = 0;
  CK(cudaMemcpyAsync(&n, *d_off + ctx->lcells, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  *nsec = n;
  return SM_OK;
}
// the header and the zero gap before the records
static int snap_put_header(sm_context* ctx, const SnapHeader& H, unsigned char* dst, bool dev) {
  const size_t gap0 = H.offsets_at + 8 * (H.ncells + 1), gap = H.records_at - gap0;
  if (!dev) {
    memcpy(dst, &H, sizeof(H));
    memset(dst + gap0, 0, gap);
    return SM_OK;
  }
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaMemcpyAsync(dst, &H, sizeof(H), cudaMemcpyHostToDevice, ctx->stream));
  if (gap) CK(cudaMemsetAsync(dst + gap0, 0, gap, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}
// This context's strip into the snapshot H at dst: its offsets (plus sb, the sections of the snapshot's cells before
// the strip), its records and its frequency columns.  d_off from snap_count.
static int snap_put_strip(sm_context* ctx, DevTmp& t, const SnapHeader& H, uint64_t sb, unsigned char* dst, bool dev,
                          const unsigned long long* d_off) {
  CK(cudaSetDevice(ctx->cfg.device));
  const size_t L = ctx->lcells, dimy = (size_t)ctx->d.dimy;
  unsigned long long* const o_dst = (unsigned long long*)(dst + H.offsets_at) + (size_t)(ctx->x0 - H.x0) * dimy;
  SnapRec* const r_dst = (SnapRec*)(dst + H.records_at) + sb;
  if (dev) {
    k_snap_offsets<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(d_off, L, sb, o_dst);
    k_snap_pack<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, d_off, 0, L, r_dst);
    ctx->launches += 2;
    CK(cudaGetLastError());
  } else {
    CK(cudaMemcpyAsync(o_dst, d_off, (L + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (sb) for (size_t i = 0; i <= L; i++) o_dst[i] += sb;
    SnapRec* stage = nullptr;
    const int rc = snap_alloc(ctx, t, SNAP_STAGE_BYTES, (void**)&stage);
    if (rc != SM_OK) return rc;
    const unsigned long long cap = SNAP_STAGE_BYTES / sizeof(SnapRec);
    for (size_t lo = 0; lo < L;) {     // the longest cell range whose records fit in the staging buffer
      const size_t hi = (size_t)(std::upper_bound(o_dst + lo + 1, o_dst + L + 1, o_dst[lo] + cap) - o_dst) - 1;
      if (hi == lo) return fail(ctx, SM_ERR_INVALID, "sm_snapshot_save: a column longer than the staging buffer");
      k_snap_pack<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, d_off, lo, hi, stage);
      ctx->launches++;
      CK(cudaGetLastError());
      const size_t n = (size_t)(o_dst[hi] - o_dst[lo]);
      if (n) CK(cudaMemcpyAsync(r_dst + (o_dst[lo] - sb), stage, n * sizeof(SnapRec), cudaMemcpyDeviceToHost, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
      lo = hi;
    }
  }
  const float* const src[3] = {ctx->d.wfreq, ctx->d.wtrack, ctx->d.windfreq};
  const size_t w = (size_t)(H.x1 - H.x0);
  for (int k = 0; k < 3; k++)
    CK(cudaMemcpy2DAsync(dst + H.freq_at + (size_t)k * 4 * H.ncells + 4 * (size_t)(ctx->x0 - H.x0), 4 * w,
                         src[k] + ctx->x0, 4 * (size_t)ctx->d.dimx, 4 * (size_t)(ctx->x1 - ctx->x0), dimy,
                         cudaMemcpyDefault, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SM_OK;
}

// Save (dst != NULL) or size (bytes != NULL) the snapshot of this context: its strip, or the whole map of a group.
static int snap_save(sm_context* ctx, int64_t* bytes, void* dst, int64_t capacity, bool dev) {
  const int n = ctx->group ? ctx->group->n : 1;
  sm_context* const* const R = ctx->group ? ctx->group->rank : &ctx;
  if (ctx->group) {
    const int rc = grp_settle(ctx);
    if (rc != SM_OK) return rc;
  } else {
    CK(cudaSetDevice(ctx->cfg.device));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  std::vector<DevTmp> t((size_t)n);
  std::vector<unsigned long long*> d_off((size_t)n, nullptr);
  std::vector<uint64_t> base((size_t)n + 1, 0);
  for (int r = 0; r < n; r++) {       // every rank counts; the rank totals become the section bases
    uint64_t nsec = 0;
    const int rc = snap_count(R[r], t[(size_t)r], &d_off[(size_t)r], &nsec);
    if (rc != SM_OK) return ctx->group ? grp_err(ctx, r, rc) : rc;
    base[(size_t)r + 1] = base[(size_t)r] + nsec;
  }
  SnapHeader H;
  snap_layout(H, ctx->d.dimx, ctx->d.dimy, ctx->group ? 0 : ctx->x0, ctx->group ? ctx->d.dimx : ctx->x1, ctx->nsoils,
              base[(size_t)n]);
  if (bytes) { *bytes = (int64_t)H.total_bytes; return SM_OK; }
  if ((uint64_t)capacity < H.total_bytes) return fail(ctx, SM_ERR_INVALID, "sm_snapshot_save: capacity too small");
  uint64_t sum = 0;
  for (int r = 0; r < n; r++) {       // the strips' checksums add up mod 2^64
    uint64_t part = 0;
    const int rc = sm_checksum(R[r], &part);
    if (rc != SM_OK) return ctx->group ? grp_err(ctx, r, rc) : rc;
    sum += part;
  }
  H.checksum = sum;
  int rc = snap_put_header(R[0], H, (unsigned char*)dst, dev);
  if (rc != SM_OK) return ctx->group ? grp_err(ctx, 0, rc) : rc;
  for (int r = 0; r < n; r++) {
    rc = snap_put_strip(R[r], t[(size_t)r], H, base[(size_t)r], (unsigned char*)dst, dev, d_off[(size_t)r]);
    if (rc != SM_OK) return ctx->group ? grp_err(ctx, r, rc) : rc;
  }
  return SM_OK;
}

int sm_snapshot_bytes(sm_context* ctx, int64_t* bytes) {
  if (!bytes) return fail(ctx, SM_ERR_INVALID, "null argument");
  return snap_save(ctx, bytes, nullptr, 0, false);
}
int sm_snapshot_save(sm_context* ctx, void* dst, int64_t capacity, int32_t dst_on_device) {
  if (!dst) return fail(ctx, SM_ERR_INVALID, "sm_snapshot_save: null destination");
  return snap_save(ctx, nullptr, dst, capacity, dst_on_device != 0);
}

// One context's share of a restore: its slice [lo, lo + lcells) of the snapshot's cells, validated and given its pool
// bases (snap_prepare) before any context's map is written (snap_commit).
struct SnapIn {
  DevTmp t;
  const unsigned long long* off = nullptr;   // device: the slice of the offsets, lcells + 1 of them
  const SnapRec* rec = nullptr;              // device: the record of index off[0]
  unsigned long long* base = nullptr;        // device: each column's first pool slot
  uint64_t need = 0;                         // pool slots (buried sections)
};
static int snap_header(sm_context* ctx, const void* src, int64_t bytes, bool dev, SnapHeader& H) {
  if (!src || bytes < (int64_t)sizeof(H)) return fail(ctx, SM_ERR_INVALID, "snapshot: shorter than its header");
  if (dev) {
    CK(cudaSetDevice(ctx->cfg.device));
    CK(cudaMemcpy(&H, src, sizeof(H), cudaMemcpyDeviceToHost));
  } else {
    memcpy(&H, src, sizeof(H));
  }
  const char* m = snap_check_header(H, bytes, ctx->d.dimx, ctx->d.dimy, ctx->nsoils);
  return m ? fail(ctx, SM_ERR_INVALID, m) : SM_OK;
}
static int snap_prepare(sm_context* ctx, const SnapHeader& H, const unsigned char* src, bool dev, SnapIn& in) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaStreamSynchronize(ctx->stream));
  const size_t dimy = (size_t)ctx->d.dimy, L = ctx->lcells;
  size_t lo;
  if (H.x0 == ctx->x0 && H.x1 == ctx->x1) lo = 0;
  else if (H.x0 == 0 && H.x1 == ctx->d.dimx) lo = (size_t)ctx->x0 * dimy;
  else return fail(ctx, SM_ERR_INVALID, "snapshot: its x-range is neither the whole map nor this context's strip");
  const unsigned long long* const off = (const unsigned long long*)(src + H.offsets_at);
  unsigned long long ends[4];          // off[0], off[ncells], off[lo], off[lo + L]
  const size_t at[4] = {0, (size_t)H.ncells, lo, lo + L};
  for (int i = 0; i < 4; i++) {
    if (dev) CK(cudaMemcpy(&ends[i], off + at[i], 8, cudaMemcpyDeviceToHost));
    else ends[i] = off[at[i]];
  }
  if (!snap_check_ends(ends[0], ends[1], ends[2], ends[3], H.nsections))
    return fail(ctx, SM_ERR_INVALID, "snapshot: offsets do not run from 0 to nsections");
  const size_t nrec = (size_t)(ends[3] - ends[2]);
  const SnapRec* const rec = (const SnapRec*)(src + H.records_at) + ends[2];
  int rc;
  if (dev) {
    in.off = off + lo;
    in.rec = rec;
  } else {             // a host source: the slice's offsets and records are copied to the device first
    void* p;
    if ((rc = snap_alloc(ctx, in.t, (L + 1) * 8, &p)) != SM_OK) return rc;
    CK(cudaMemcpyAsync(p, off + lo, (L + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    in.off = (const unsigned long long*)p;
    if ((rc = snap_alloc(ctx, in.t, nrec * sizeof(SnapRec), &p)) != SM_OK) return rc;
    if (nrec) CK(cudaMemcpyAsync(p, rec, nrec * sizeof(SnapRec), cudaMemcpyHostToDevice, ctx->stream));
    in.rec = (const SnapRec*)p;
  }
  if ((rc = snap_alloc(ctx, in.t, (L + 2) * 8, (void**)&in.base)) != SM_OK) return rc;
  unsigned int* const d_err = (unsigned int*)(in.base + L + 1);
  CK(cudaMemsetAsync(d_err, 0, 4, ctx->stream));
  k_snap_validate<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(in.off, in.rec, L, ctx->nsoils, in.base, d_err);
  ctx->launches++;
  CK(cudaGetLastError());
  unsigned int err = 0;
  CK(cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (err) return fail(ctx, SM_ERR_INVALID, "snapshot: offsets run backwards or a section's soil type is out of range");
  if ((rc = snap_scan(ctx, in.t, in.base, L + 1)) != SM_OK) return rc;
  unsigned long long need = 0;
  CK(cudaMemcpyAsync(&need, in.base + L, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  in.need = need;
  if (need >= SM_NIL - L - (4ull << 20)) return fail(ctx, SM_ERR_POOL, "snapshot: more buried sections than pool slots can address");
  if ((ctx->cfg.pool_capacity > 0 || ctx->nranks > 1) && need > ctx->d.pool_cap)
    return fail(ctx, SM_ERR_POOL, ctx->nranks > 1 ? "sharded context: pool_capacity is fixed at creation and too small"
                                                  : "snapshot: pool_capacity too small");
  return SM_OK;
}
static int snap_commit(sm_context* ctx, const SnapHeader& H, const unsigned char* src, SnapIn& in) {
  CK(cudaSetDevice(ctx->cfg.device));
  if (ctx->cfg.pool_capacity <= 0 && ctx->nranks == 1) {      // grows as sm_upload_columns does
    const int rc = alloc_pool(ctx, in.need + (unsigned long long)ctx->lcells + (4ull << 20));
    if (rc != SM_OK) return rc;
  }
  k_snap_unpack<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, in.off, in.rec, ctx->lcells, in.base);
  ctx->launches++;
  CK(cudaGetLastError());
  float* const dstf[3] = {ctx->d.wfreq, ctx->d.wtrack, ctx->d.windfreq};
  const size_t w = (size_t)(H.x1 - H.x0);
  for (int k = 0; k < 3; k++)
    CK(cudaMemcpy2DAsync(dstf[k] + ctx->x0, 4 * (size_t)ctx->d.dimx,
                         src + H.freq_at + (size_t)k * 4 * H.ncells + 4 * (size_t)(ctx->x0 - H.x0), 4 * w,
                         4 * (size_t)(ctx->x1 - ctx->x0), (size_t)ctx->d.dimy, cudaMemcpyDefault, ctx->stream));
  const int rc = reset_pool_ctl(ctx, in.need);     // synchronises the stream first
  if (rc != SM_OK) return rc;
  ctx->cur_kind = -1; ctx->cur_n = 0;              // no batch to resume or flood, as on a fresh context
  ctx->mesh_valid = false;
  return SM_OK;
}

int sm_snapshot_restore(sm_context* ctx, const void* src_, int64_t bytes, int32_t src_on_device) {
  const bool dev = src_on_device != 0;
  const unsigned char* const src = (const unsigned char*)src_;
  const int n = ctx->group ? ctx->group->n : 1;
  sm_context* const* const R = ctx->group ? ctx->group->rank : &ctx;
  SnapHeader H;
  int rc = snap_header(ctx->group ? R[0] : ctx, src, bytes, dev, H);
  if (rc != SM_OK) return ctx->group ? grp_err(ctx, 0, rc) : rc;
  if (ctx->group) {
    if (H.x0 != 0 || H.x1 != ctx->d.dimx) return fail(ctx, SM_ERR_INVALID, "snapshot: a group restores whole-map snapshots only");
    if ((rc = grp_settle(ctx)) != SM_OK) return rc;
  }
  std::vector<SnapIn> in((size_t)n);
  for (int r = 0; r < n; r++)            // every rank validates its slice before any rank writes
    if ((rc = snap_prepare(R[r], H, src, dev, in[(size_t)r])) != SM_OK) return ctx->group ? grp_err(ctx, r, rc) : rc;
  if (ctx->group) { ctx->group->dirty = true; ctx->cur_kind = -1; ctx->cur_n = 0; }
  for (int r = 0; r < n; r++)
    if ((rc = snap_commit(R[r], H, src, in[(size_t)r])) != SM_OK) return ctx->group ? grp_err(ctx, r, rc) : rc;
  // the map now holds what the snapshot describes; its checksum is checked where this context holds all it covers
  if (ctx->group || (H.x0 == ctx->x0 && H.x1 == ctx->x1)) {
    uint64_t sum = 0, part = 0;
    for (int r = 0; r < n; r++) {
      if ((rc = sm_checksum(R[r], &part)) != SM_OK) return ctx->group ? grp_err(ctx, r, rc) : rc;
      sum += part;
    }
    if (sum != H.checksum) return fail(ctx, SM_ERR_INVALID, "snapshot: the restored columns do not match the header's checksum");
  }
  return SM_OK;
}

// ---- layer rasters (sm_layer.cuh, DESIGN.md section 11) ----------------------------------------------------------
// One context's share of sm_apply_layer: its strip of the raster, checked and counted (layer_check) before any context's
// map is written (layer_launch, layer_finish).
struct LayerIn {
  DevTmp t;
  const double* delta = nullptr;             // device: the strip's raster
  double* left = nullptr;                    // device: where k_layer_apply writes the leftovers (null: nowhere)
  unsigned long long* d_out = nullptr;       // device: pushed, touched, error, emptied
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  sm_layer_stats st = {};
  ~LayerIn() {
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
  }
};
// src: the strip's raster, on the host or (dev) on this context's device; src_dev0: a raster on `dev0` (a group's rank 0)
// that is copied over after ev0 on that device's stream.  want_left: k_layer_apply writes leftovers (into `left_dev`
// when given, a device buffer on this context's device, else into a staging buffer).
static int layer_check(sm_context* ctx, const double* src, bool dev, const double* src_dev0, int dev0, cudaEvent_t ev0,
                       int32_t type, bool want_left, double* left_dev, LayerIn& in) {
  if (ctx->nsoils < 1) return fail(ctx, SM_ERR_INVALID, "soil table not set");
  if (type < 0 || type >= ctx->nsoils) return fail(ctx, SM_ERR_INVALID, "sm_apply_layer: type out of range");
  CK(cudaSetDevice(ctx->cfg.device));
  const size_t L = ctx->lcells;
  int rc;
  if ((rc = snap_alloc(ctx, in.t, 4 * 8, (void**)&in.d_out)) != SM_OK) return rc;
  CK(cudaMemsetAsync(in.d_out, 0, 4 * 8, ctx->stream));
  if (src_dev0) {
    void* p;
    if ((rc = snap_alloc(ctx, in.t, L * 8, &p)) != SM_OK) return rc;
    CK(cudaStreamWaitEvent(ctx->stream, ev0, 0));
    CK(cudaMemcpyPeerAsync(p, ctx->cfg.device, src_dev0, dev0, L * 8, ctx->stream));
    in.delta = (const double*)p;
  } else if (!dev) {            // a host raster is staged: L x 8 bytes of device memory
    void* p;
    if ((rc = snap_alloc(ctx, in.t, L * 8, &p)) != SM_OK) return rc;
    CK(cudaMemcpyAsync(p, src, L * 8, cudaMemcpyHostToDevice, ctx->stream));
    in.delta = (const double*)p;
  } else {
    in.delta = src;
  }
  if (want_left) {
    if (left_dev) in.left = left_dev;
    else if ((rc = snap_alloc(ctx, in.t, L * 8, (void**)&in.left)) != SM_OK) return rc;
  }
  CK(cudaEventCreate(&in.e0));
  CK(cudaEventCreate(&in.e1));
  CK(cudaEventRecord(in.e0, ctx->stream));
  k_layer_check<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, in.delta, L, type, in.d_out);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(in.e1, ctx->stream));
  unsigned long long out[3];
  RunCtl h;                     // the pool's state: bump counter and rings, as the last call left them
  CK(cudaMemcpyAsync(out, in.d_out, 3 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(&h.bump, &ctx->d.ctl->bump, sizeof(h.bump) + sizeof(h.ring), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, in.e0, in.e1));
  const unsigned long long cap = ctx->d.pool_cap;
  in.st.cells = (int64_t)out[1];
  in.st.pushed = (int64_t)out[0];
  in.st.free_slots = (int64_t)((h.ring[1].tail - h.ring[1].head) + (cap - std::min(h.bump, cap)));
  in.st.device_ms = ms;
  if (out[2]) return fail(ctx, SM_ERR_INVALID, "sm_apply_layer: a raster entry is not finite");
  if (in.st.pushed > in.st.free_slots)
    return fail(ctx, SM_ERR_POOL, "sm_apply_layer: the raster pushes more sections than the pool has free slots");
  return SM_OK;
}
// the apply kernel of a checked strip, left in flight
static int layer_launch(sm_context* ctx, uint32_t type, LayerIn& in) {
  CK(cudaSetDevice(ctx->cfg.device));
  CK(cudaEventRecord(in.e0, ctx->stream));
  k_layer_apply<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(ctx->d, in.delta, ctx->lcells, type, in.left, in.d_out + 3);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(in.e1, ctx->stream));
  return SM_OK;
}
// wait for the apply; left_host: copy the leftovers there; left_dev0: copy them to that buffer on device dev0
static int layer_finish(sm_context* ctx, LayerIn& in, double* left_host, double* left_dev0, int dev0) {
  CK(cudaSetDevice(ctx->cfg.device));
  const size_t L = ctx->lcells;
  unsigned long long emptied = 0;
  CK(cudaMemcpyAsync(&emptied, in.d_out + 3, 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (left_host) CK(cudaMemcpyAsync(left_host, in.left, L * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (left_dev0) CK(cudaMemcpyPeerAsync(left_dev0, dev0, in.left, ctx->cfg.device, L * 8, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, in.e0, in.e1));
  in.st.emptied = (int64_t)emptied;
  in.st.device_ms += ms;
  return SM_OK;
}

int sm_apply_layer(sm_context* ctx, const double* delta, int32_t type, double* leftover, int32_t on_device,
                   int32_t check_only, sm_layer_stats* stats) {
  if (!delta) return fail(ctx, SM_ERR_INVALID, "sm_apply_layer: null raster");
  const bool dev = on_device != 0, want_left = leftover != nullptr && !check_only;
  const int n = ctx->group ? ctx->group->n : 1;
  sm_context* const* const R = ctx->group ? ctx->group->rank : &ctx;
  int rc;
  if (ctx->group && (rc = grp_settle(ctx)) != SM_OK) return rc;
  sm_context* const c0 = R[0];
  if (ctx->group && dev) {      // the ranks' slices of a device raster are copied from rank 0's device after its stream
    CK(cudaSetDevice(c0->cfg.device));
    CK(cudaEventRecord(ctx->group->ev, c0->stream));
  }
  std::vector<LayerIn> in((size_t)n);
  sm_layer_stats tot = {};
  auto add = [&](const sm_layer_stats& s) {
    tot.cells += s.cells; tot.pushed += s.pushed; tot.free_slots += s.free_slots; tot.emptied += s.emptied;
    tot.device_ms = std::max(tot.device_ms, s.device_ms);
  };
  int bad = -1, bad_rc = SM_OK;
  for (int r = 0; r < n; r++) {     // every rank checks its strip before any rank writes
    sm_context* const c = R[r];
    const size_t off = ctx->group ? (size_t)c->x0 * ctx->d.dimy : 0;
    const bool peer = ctx->group && dev && r > 0;
    double* const ldev = (want_left && dev && !peer) ? leftover + off : nullptr;
    rc = layer_check(c, peer ? nullptr : delta + off, dev, peer ? delta + off : nullptr, c0->cfg.device,
                     ctx->group ? ctx->group->ev : nullptr, type, want_left, ldev, in[(size_t)r]);
    add(in[(size_t)r].st);
    if (rc != SM_OK && bad < 0) { bad = r; bad_rc = rc; }
    if (rc != SM_OK && rc != SM_ERR_POOL) break;     // the other ranks' counts only matter for a pool refusal
  }
  if (bad >= 0 || check_only) {
    if (stats) *stats = tot;
    if (bad >= 0) return ctx->group ? grp_err(ctx, bad, bad_rc) : bad_rc;
    return SM_OK;
  }
  if (ctx->group) ctx->group->dirty = true;
  for (int r = 0; r < n; r++)       // every rank's apply is in flight before any is waited for
    if ((rc = layer_launch(R[r], (uint32_t)type, in[(size_t)r])) != SM_OK) return ctx->group ? grp_err(ctx, r, rc) : rc;
  tot = {};
  for (int r = 0; r < n; r++) {
    sm_context* const c = R[r];
    const size_t off = ctx->group ? (size_t)c->x0 * ctx->d.dimy : 0;
    const bool peer = ctx->group && dev && r > 0;
    rc = layer_finish(c, in[(size_t)r], want_left && !dev ? leftover + off : nullptr,
                      want_left && peer ? leftover + off : nullptr, c0->cfg.device);
    if (rc != SM_OK) return ctx->group ? grp_err(ctx, r, rc) : rc;
    add(in[(size_t)r].st);
  }
  if (stats) *stats = tot;
  return SM_OK;
}

// ---- slope relaxation (sm_relax.cuh, DESIGN.md section 12) -------------------------------------------------------
// One rank's share of a relax call: its stale bitmap and counter block, its timing events, and `ev`, recorded after
// each of its phase launches, which every rank's next phase waits for.
struct RelaxRank {
  DevTmp t;
  cudaEvent_t e0 = nullptr, e1 = nullptr, ev = nullptr;
  unsigned long long cnt[SM_RELAX_CNT] = {};
  ~RelaxRank() {
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    if (ev) cudaEventDestroy(ev);
  }
};

int sm_relax(sm_context* ctx, int32_t max_passes, int32_t transferloop, sm_relax_stats* stats) {
  if (transferloop < 0 || transferloop > 3 || max_passes < 1)
    return fail(ctx, SM_ERR_INVALID, "sm_relax: range (transferloop 0..3, max_passes >= 1)");
  if (!ctx->group && ctx->nranks > 1)
    return fail(ctx, SM_ERR_INVALID, "sm_relax is not available on a rank of a sharded map (every phase needs every "
                                     "rank's previous phase); a group (sm_create_group) offers it");
  const int n = ctx->group ? ctx->group->n : 1;
  sm_context* const* const R = ctx->group ? ctx->group->rank : &ctx;
  if (R[0]->nsoils < 1) return fail(ctx, SM_ERR_INVALID, "soil table not set");
  int rc;
  if (ctx->group && (rc = grp_settle(ctx)) != SM_OK) return rc;
  std::vector<RelaxRank> rk((size_t)n);
  RelaxMaps m = {};
  for (int r = 0; r < n; r++) {     // every cell stale, counters zero
    sm_context* const c = R[r];
    RelaxRank& k = rk[(size_t)r];
    const size_t words = (c->lcells + 31) / 32;
    if ((rc = snap_alloc(c, k.t, words * 4, (void**)&m.stale[r])) != SM_OK ||
        (rc = snap_alloc(c, k.t, SM_RELAX_CNT * 8, (void**)&m.cnt[r])) != SM_OK)
      return ctx->group ? grp_err(ctx, r, rc) : rc;
    CK(cudaSetDevice(c->cfg.device));
    CK(cudaMemsetAsync(m.stale[r], 0xFF, words * 4, c->stream));
    CK(cudaMemsetAsync(m.cnt[r], 0, SM_RELAX_CNT * 8, c->stream));
    CK(cudaEventCreate(&k.e0));
    CK(cudaEventCreate(&k.e1));
    CK(cudaEventCreateWithFlags(&k.ev, cudaEventDisableTiming));
    CK(cudaEventRecord(k.e0, c->stream));
  }
  if (ctx->group) ctx->group->dirty = true;
  const int P = relax_period(transferloop);
  sm_relax_stats st = {};
  unsigned long long changed = 0;
  unsigned int j = 0;               // launch index of the call: its pool parity
  for (int pass = 1; pass <= max_passes; pass++) {
    for (int p = 0; p < P * P; p++, j++) {
      // every rank's phase p - 1 is complete before any rank's phase p starts (only neighbours share columns, but the
      // stop flag of a pool drop reaches every rank)
      for (int r = 0; r < n; r++) {
        sm_context* const c = R[r];
        CK(cudaSetDevice(c->cfg.device));
        if (n > 1 && j > 0)
          for (int q = 0; q < n; q++) CK(cudaStreamWaitEvent(c->stream, rk[(size_t)q].ev, 0));
        const size_t cells = (size_t)((c->x1 - c->x0 + P - 1) / P) * (size_t)((c->d.dimy + P - 1) / P);
        const int blocks = (int)std::min<size_t>((cells + 255) / 256, (size_t)c->num_sms * 8);
        if (n > 1) k_relax_phase<true><<<blocks, 256, 0, c->stream>>>(c->d, p / P, p % P, transferloop, j & 1u, m);
        else k_relax_phase<false><<<blocks, 256, 0, c->stream>>>(c->d, p / P, p % P, transferloop, j & 1u, m);
        c->launches++;
        CK(cudaGetLastError());
      }
      if (n > 1)
        for (int r = 0; r < n; r++) {
          CK(cudaSetDevice(R[r]->cfg.device));
          CK(cudaEventRecord(rk[(size_t)r].ev, R[r]->stream));
        }
    }
    for (int r = 0; r < n; r++) {   // one counter block per rank and pass decides whether the call goes on
      sm_context* const c = R[r];
      CK(cudaSetDevice(c->cfg.device));
      CK(cudaEventRecord(rk[(size_t)r].e1, c->stream));
      CK(cudaMemcpyAsync(rk[(size_t)r].cnt, m.cnt[r], SM_RELAX_CNT * 8, cudaMemcpyDeviceToHost, c->stream));
    }
    unsigned long long tot[SM_RELAX_CNT] = {};
    for (int r = 0; r < n; r++) {
      CK(cudaSetDevice(R[r]->cfg.device));
      CK(cudaStreamSynchronize(R[r]->stream));
      for (int k = 0; k < SM_RELAX_CNT; k++) tot[k] += rk[(size_t)r].cnt[k];
    }
    st.passes = pass;
    st.visits = (int64_t)tot[0];
    st.transfers = (int64_t)tot[2];
    st.pool_drops = (int64_t)tot[3];
    st.stable = tot[1] == changed;
    changed = tot[1];
    if (st.pool_drops || st.stable) break;
  }
  if (ctx->group) ctx->group->dirty = false;    // every rank's stream was synchronised after the last pass
  for (int r = 0; r < n; r++) {
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, rk[(size_t)r].e0, rk[(size_t)r].e1));
    st.device_ms = std::max(st.device_ms, (double)ms);
  }
  if (stats) *stats = st;
  if (st.pool_drops) return fail(ctx, SM_ERR_POOL, "sm_relax: pool exhausted, sections dropped (the call stopped)");
  return SM_OK;
}

}  // extern "C"

// ---- strata views (sm_strata.cuh, DESIGN.md section 13) ----------------------------------------------------------
namespace {
struct StrataEvents {      // one kernel's timing events, destroyed with the call
  int device = 0;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  StrataEvents() = default;
  StrataEvents(const StrataEvents&) = delete;
  StrataEvents& operator=(const StrataEvents&) = delete;
  ~StrataEvents() {
    if (!e0 && !e1) return;
    cudaSetDevice(device);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
  }
};
}  // namespace

// One context's part of a view: n cells, `planes` planes of esize-byte entries.  launch(lo, hi, out, stride, nsec)
// enqueues the kernel that writes cells [lo, hi) of every plane to out[plane * stride + (cell - lo)].  dst: where cell 0
// of plane 0 of this part goes, dpitch: the bytes from one plane to the next there.  direct: dst is on this context's
// device and the kernel writes it in place; otherwise the planes go through a staging buffer of at most
// SNAP_STAGE_BYTES, range by range, with 2-D copies to dst (host memory or another device).  Returns when dst is
// written; st gets the sections read and the kernels' event time.
template <class F>
static int strata_part(sm_context* ctx, size_t n, size_t planes, size_t esize, unsigned char* dst, size_t dpitch,
                       bool direct, F launch, sm_view_stats& st) {
  CK(cudaSetDevice(ctx->cfg.device));
  DevTmp t;
  unsigned long long* d_n = nullptr;
  int rc = snap_alloc(ctx, t, 8, (void**)&d_n);
  if (rc != SM_OK) return rc;
  CK(cudaMemsetAsync(d_n, 0, 8, ctx->stream));
  const size_t chunk = direct ? std::max<size_t>(n, 1) : std::max<size_t>(1, SNAP_STAGE_BYTES / (planes * esize));
  unsigned char* stage = nullptr;
  if (!direct && (rc = snap_alloc(ctx, t, std::min(chunk, std::max<size_t>(n, 1)) * planes * esize, (void**)&stage)) != SM_OK)
    return rc;
  std::vector<StrataEvents> ev((n + chunk - 1) / chunk);
  for (size_t lo = 0, j = 0; lo < n; lo += chunk, j++) {
    const size_t hi = std::min(n, lo + chunk);
    StrataEvents& e = ev[j];
    e.device = ctx->cfg.device;
    CK(cudaEventCreate(&e.e0));
    CK(cudaEventCreate(&e.e1));
    CK(cudaEventRecord(e.e0, ctx->stream));
    launch(lo, hi, direct ? dst : stage, direct ? dpitch / esize : hi - lo, d_n);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaEventRecord(e.e1, ctx->stream));
    if (!direct) {      // the next range's kernel rewrites the staging buffer after this copy, in stream order
      CK(cudaMemcpy2DAsync(dst + lo * esize, dpitch, stage, (hi - lo) * esize, (hi - lo) * esize, planes, cudaMemcpyDefault,
                           ctx->stream));
    }
  }
  unsigned long long nsec = 0;
  CK(cudaMemcpyAsync(&nsec, d_n, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  double ms = 0.0;
  for (const StrataEvents& e : ev) {
    float m = 0.f;
    CK(cudaEventElapsedTime(&m, e.e0, e.e1));
    ms += m;
  }
  st.cells += (int64_t)n;
  st.sections += (int64_t)nsec;
  st.bytes_out += (int64_t)(n * planes * esize);
  st.device_ms = std::max(st.device_ms, ms);
  return SM_OK;
}

// the ranks of ctx and whether rank r's kernels write device output in place (rank 0's device)
static bool strata_direct(sm_context* ctx, sm_context* c, bool dev) {
  return dev && (!ctx->group || c->cfg.device == ctx->group->rank[0]->cfg.device);
}

extern "C" {

int sm_composition(sm_context* ctx, const int32_t* types, int32_t ntypes, double lo, double hi, int32_t flags,
                   double* out, int32_t on_device, sm_view_stats* stats) {
  const int n = ctx->group ? ctx->group->n : 1;
  sm_context* const* const R = ctx->group ? ctx->group->rank : &ctx;
  const int nsoils = R[0]->nsoils;
  if (nsoils < 1) return fail(ctx, SM_ERR_INVALID, "soil table not set");
  if (!types || !out) return fail(ctx, SM_ERR_INVALID, "sm_composition: null argument");
  if (ntypes < 1 || ntypes > nsoils) return fail(ctx, SM_ERR_INVALID, "sm_composition: ntypes outside 1..nsoils");
  if (std::isnan(lo) || std::isnan(hi) || lo > hi)
    return fail(ctx, SM_ERR_INVALID, "sm_composition: the window needs lo <= hi, neither NaN");
  if (flags & ~(SM_COMP_BELOW_SURFACE | SM_COMP_PORE_WATER)) return fail(ctx, SM_ERR_INVALID, "sm_composition: unknown flags");
  StrataSel sel;
  memset(sel.slot, -1, sizeof(sel.slot));
  for (int i = 0; i < ntypes; i++) {
    if (types[i] < 0 || types[i] >= nsoils) return fail(ctx, SM_ERR_INVALID, "sm_composition: type out of range");
    if (sel.slot[types[i]] >= 0) return fail(ctx, SM_ERR_INVALID, "sm_composition: type repeated");
    sel.slot[types[i]] = (signed char)i;
  }
  int rc;
  if (ctx->group && (rc = grp_settle(ctx)) != SM_OK) return rc;
  const bool dev = on_device != 0;
  const size_t N = ctx->lcells;       // the cells of one plane: the whole map on a group, the strip on a rank
  sm_view_stats st = {};
  for (int r = 0; r < n; r++) {
    sm_context* const c = R[r];
    const size_t off = ctx->group ? (size_t)c->x0 * ctx->d.dimy : 0;
    auto launch = [&](size_t a, size_t b, unsigned char* o, size_t stride, unsigned long long* d_n) {
      k_strata_compose<<<c->num_sms * 8, 256, 0, c->stream>>>(c->d, sel, ntypes, lo, hi, flags, a, b, (double*)o, stride,
                                                              d_n);
    };
    sm_view_stats part = {};
    rc = strata_part(c, c->lcells, (size_t)ntypes, 8, (unsigned char*)(out + off), N * 8, strata_direct(ctx, c, dev),
                     launch, part);
    if (rc != SM_OK) return ctx->group ? grp_err(ctx, r, rc) : rc;
    st.cells += part.cells; st.sections += part.sections; st.bytes_out += part.bytes_out;
    st.device_ms = std::max(st.device_ms, part.device_ms);
  }
  if (ctx->group) ctx->group->dirty = false;     // every rank's stream was synchronised
  if (stats) *stats = st;
  return SM_OK;
}

int sm_voxelize(sm_context* ctx, int32_t x0, int32_t x1, int32_t y0, int32_t y1, double z0, double dz, int32_t nz,
                uint8_t* out, int32_t on_device, sm_view_stats* stats) {
  const int n = ctx->group ? ctx->group->n : 1;
  sm_context* const* const R = ctx->group ? ctx->group->rank : &ctx;
  if (!out) return fail(ctx, SM_ERR_INVALID, "sm_voxelize: null argument");
  if (!(x0 < x1 && y0 < y1 && x0 >= ctx->x0 && x1 <= ctx->x1 && y0 >= 0 && y1 <= ctx->d.dimy))
    return fail(ctx, SM_ERR_INVALID, "sm_voxelize: the window is empty or outside the map (or this rank's strip)");
  if (!std::isfinite(z0) || !std::isfinite(dz) || !(dz > 0))
    return fail(ctx, SM_ERR_INVALID, "sm_voxelize: z0 and dz must be finite, dz > 0");
  if (nz < 1 || nz > SM_VOXEL_MAX_NZ) return fail(ctx, SM_ERR_INVALID, "sm_voxelize: nz outside 1..65536");
  int rc;
  if (ctx->group && (rc = grp_settle(ctx)) != SM_OK) return rc;
  const bool dev = on_device != 0;
  const double rdz = 1.0 / dz;      // the kernels estimate sample indices with it; the exact comparisons decide
  const int wy = y1 - y0;
  const size_t W = (size_t)(x1 - x0) * (size_t)wy;
  sm_view_stats st = {};
  for (int r = 0; r < n; r++) {
    sm_context* const c = R[r];
    const int xs = std::max(x0, c->x0), xe = std::min(x1, c->x1);
    if (xs >= xe) continue;       // the window does not reach this rank's strip
    auto launch = [&](size_t a, size_t b, unsigned char* o, size_t stride, unsigned long long* d_n) {
      k_strata_voxel<<<c->num_sms * 8, 256, 0, c->stream>>>(c->d, c->x0, xs, y0, wy, z0, dz, rdz, (uint32_t)nz, a, b, o,
                                                            stride, d_n);
    };
    sm_view_stats part = {};
    rc = strata_part(c, (size_t)(xe - xs) * (size_t)wy, (size_t)nz, 1, out + (size_t)(xs - x0) * (size_t)wy, W,
                     strata_direct(ctx, c, dev), launch, part);
    if (rc != SM_OK) return ctx->group ? grp_err(ctx, r, rc) : rc;
    st.cells += part.cells; st.sections += part.sections; st.bytes_out += part.bytes_out;
    st.device_ms = std::max(st.device_ms, part.device_ms);
  }
  if (ctx->group) ctx->group->dirty = false;
  if (stats) *stats = st;
  return SM_OK;
}

}  // extern "C"

// ---- drainage (sm_drain.cuh, DESIGN.md section 14) ------------------------------------------------------------------
// Every phase works on whole-map rasters in cell order x*dimy + y on the computing device.  The two relaxations run on
// tiles of DRAIN_T x DRAIN_T cells: a block loads its tile and a one-cell halo into shared memory, relaxes it to local
// stability, writes back what changed and marks for the next pass the neighbour tiles whose halo it changed.
#define DRAIN_T 32
#define DRAIN_S (DRAIN_T + 2)
#define DRAIN_BATCH 4          // relaxation passes launched between two reads of their mark counters

// H of every cell of the whole map, each column read from its owner (MULTI: through the peer pointers); the fill
// starts from W = H on the border, +inf inside.
template <bool MULTI>
__global__ void __launch_bounds__(256) k_drain_heights(DevCtx c, int ground, double* __restrict__ H, double* __restrict__ W) {
  const size_t n = (size_t)c.dimx * c.dimy;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i / (size_t)c.dimy), y = (int)(i % (size_t)c.dimy);
    const StrataPool a{MULTI ? c.peer[owner_of_x<MULTI>(c, x)].pool : c.pool};
    const double h = drain_column_height(a, *cell_ptr<MULTI>(c, x, y), ground != 0);
    H[i] = h;
    W[i] = (x == 0 || y == 0 || x == c.dimx - 1 || y == c.dimy - 1) ? h : (double)INFINITY;
  }
}

// One pass of a tiled relaxation.  DIST = false: the fill, W(c) = max(H(c), min_n W(n)) on interior cells.  DIST =
// true: the flat distances, on cells whose D is not SM_DRAIN_NOT_FLAT.  Tile t runs when act_cur[t] is set and clears
// it; *marks counts the tiles it sets in act_next.
template <bool DIST>
__global__ void __launch_bounds__(256) k_drain_relax(const double* __restrict__ H, double* W, int32_t* D, int dimx, int dimy,
                                                     int ntx, int nty, unsigned int* act_cur, unsigned int* act_next,
                                                     unsigned long long* marks) {
  __shared__ double sw[DRAIN_S][DRAIN_S];
  __shared__ int32_t sd[DIST ? DRAIN_S : 1][DIST ? DRAIN_S : 1];
  __shared__ unsigned int s_on, s_dirs;
  const int tile = blockIdx.x, tid = threadIdx.y * DRAIN_T + threadIdx.x;
  if (tid == 0) {
    s_on = act_cur[tile];
    if (s_on) act_cur[tile] = 0;
    s_dirs = 0;
  }
  __syncthreads();
  if (!s_on) return;
  const int TX = tile / nty, TY = tile % nty, X0 = TX * DRAIN_T, Y0 = TY * DRAIN_T;
  for (int i = tid; i < DRAIN_S * DRAIN_S; i += blockDim.x * blockDim.y) {
    const int lx = i / DRAIN_S, ly = i % DRAIN_S, gx = X0 - 1 + lx, gy = Y0 - 1 + ly;
    const bool in = gx >= 0 && gx < dimx && gy >= 0 && gy < dimy;
    const size_t g = (size_t)gx * dimy + gy;
    sw[lx][ly] = in ? W[g] : (double)INFINITY;
    if (DIST) sd[DIST ? lx : 0][DIST ? ly : 0] = in ? D[g] : SM_DRAIN_FAR;
  }
  __syncthreads();
  constexpr int R = DRAIN_T * DRAIN_T / 256;
  double h[R];
  bool live[R];
  const int ly = threadIdx.x, Y = Y0 + ly;
#pragma unroll
  for (int j = 0; j < R; j++) {
    const int lx = threadIdx.y + j * (256 / DRAIN_T), X = X0 + lx;
    live[j] = X > 0 && X < dimx - 1 && Y > 0 && Y < dimy - 1;
    if (DIST) live[j] = live[j] && sd[DIST ? lx + 1 : 0][DIST ? ly + 1 : 0] != SM_DRAIN_NOT_FLAT;
    h[j] = !live[j] ? 0.0 : (DIST ? sw[lx + 1][ly + 1] : H[(size_t)X * dimy + Y]);
  }
  bool mine = false;
  SM_UNROLL1
  for (;;) {
    bool ch = false;
#pragma unroll
    for (int j = 0; j < R; j++) {
      if (!live[j]) continue;
      const int lx = threadIdx.y + j * (256 / DRAIN_T) + 1, cy = ly + 1;
      double wn[8];
#pragma unroll
      for (int k = 0; k < 8; k++) wn[k] = sw[lx + drain_dx(k)][cy + drain_dy(k)];
      if (!DIST) {
        const double v = drain_fill_value(h[j], wn);
        if (v < sw[lx][cy]) { sw[lx][cy] = v; ch = true; }
      } else {
        int32_t dn[8];
#pragma unroll
        for (int k = 0; k < 8; k++) dn[k] = sd[DIST ? lx + drain_dx(k) : 0][DIST ? cy + drain_dy(k) : 0];
        const int32_t dc = sd[DIST ? lx : 0][DIST ? cy : 0];
        const int32_t v = drain_dist_value(h[j], dc, wn, dn);
        if (v < dc) { sd[DIST ? lx : 0][DIST ? cy : 0] = v; ch = true; }
      }
    }
    mine |= ch;
    if (!__syncthreads_or(ch)) break;
  }
  if (mine) {       // write back what changed; the neighbour tiles whose halo holds a changed cell run again
    unsigned int dirs = 0;
#pragma unroll
    for (int j = 0; j < R; j++) {
      if (!live[j]) continue;
      const int lx = threadIdx.y + j * (256 / DRAIN_T);
      const size_t g = (size_t)(X0 + lx) * dimy + Y;
      bool changed;
      if (!DIST) {
        changed = sw[lx + 1][ly + 1] != W[g];
        if (changed) W[g] = sw[lx + 1][ly + 1];
      } else {
        const int32_t v = sd[DIST ? lx + 1 : 0][DIST ? ly + 1 : 0];
        changed = v != D[g];
        if (changed) D[g] = v;
      }
      if (!changed) continue;
      const int ax = lx == 0 ? -1 : 0, bx = lx == DRAIN_T - 1 ? 1 : 0;
      const int ay = ly == 0 ? -1 : 0, by = ly == DRAIN_T - 1 ? 1 : 0;
      for (int dx = ax; dx <= bx; dx++)
        for (int dy = ay; dy <= by; dy++)
          if (dx || dy) dirs |= 1u << ((dx + 1) * 3 + (dy + 1));
    }
    if (dirs) atomicOr(&s_dirs, dirs);
  }
  __syncthreads();
  if (tid == 0 && s_dirs) {
    unsigned long long n = 0;
    for (int b = 0; b < 9; b++) {
      if (!(s_dirs & (1u << b))) continue;
      const int tx = TX + b / 3 - 1, ty = TY + b % 3 - 1;
      if (tx < 0 || tx >= ntx || ty < 0 || ty >= nty) continue;
      act_next[tx * nty + ty] = 1u;
      n++;
    }
    if (n) atomicAdd(marks, n);
  }
}

// the 3x3 window of a whole-map raster around the interior cell (x, y), neighbours in the order n[k]
template <class T>
__device__ __forceinline__ void drain_window(const T* __restrict__ a, int x, int y, int dimy, T* out) {
#pragma unroll
  for (int k = 0; k < 8; k++) out[k] = a[(size_t)(x + drain_dx(k)) * dimy + (y + drain_dy(k))];
}
__device__ __forceinline__ bool drain_border(int x, int y, int dimx, int dimy) {
  return x == 0 || y == 0 || x == dimx - 1 || y == dimy - 1;
}

// after the fill: D = SM_DRAIN_NOT_FLAT on drained and border cells, SM_DRAIN_FAR on flat ones.  cnt[0] += flat
// cells, cnt[1] += cells with W > H.
__global__ void __launch_bounds__(256) k_drain_classify(const double* __restrict__ H, const double* __restrict__ W,
                                                        int32_t* __restrict__ D, int dimx, int dimy,
                                                        unsigned long long* __restrict__ cnt) {
  const size_t n = (size_t)dimx * dimy;
  unsigned long long flat = 0, dep = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i / (size_t)dimy), y = (int)(i % (size_t)dimy);
    bool f = false;
    if (!drain_border(x, y, dimx, dimy)) {
      double wn[8];
      drain_window(W, x, y, dimy, wn);
      f = !drain_drained(W[i], wn);
    }
    D[i] = f ? SM_DRAIN_FAR : SM_DRAIN_NOT_FLAT;
    flat += f;
    dep += W[i] > H[i];
  }
  block_add_u64(flat, &cnt[0]);
  block_add_u64(dep, &cnt[1]);
}

// receivers: dir (k or -1), rcv (the receiver's cell or -1), in-degrees, area = 1 (area may be null).  cnt[2] +=
// interior cells without a receiver (none at the fixed point).
__global__ void __launch_bounds__(256) k_drain_receivers(const double* __restrict__ W, const int32_t* __restrict__ D,
                                                         int dimx, int dimy, int8_t* __restrict__ dir, int32_t* __restrict__ rcv,
                                                         int32_t* indeg, unsigned long long* __restrict__ area,
                                                         unsigned long long* __restrict__ cnt) {
  const size_t n = (size_t)dimx * dimy;
  unsigned long long bad = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i / (size_t)dimy), y = (int)(i % (size_t)dimy);
    int k = -1;
    if (!drain_border(x, y, dimx, dimy)) {
      double wn[8];
      int32_t dn[8];
      drain_window(W, x, y, dimy, wn);
      drain_window(D, x, y, dimy, dn);
      k = drain_receiver(W[i], D[i], wn, dn);
      bad += k < 0;
    }
    dir[i] = (int8_t)k;
    if (area) area[i] = 1ull;
    if (k < 0) {
      rcv[i] = -1;
    } else {
      const int r = (x + drain_dx(k)) * dimy + (y + drain_dy(k));
      rcv[i] = r;
      atomicAdd(&indeg[r], 1);
    }
  }
  block_add_u64(bad, &cnt[2]);
}

// cnt[3] += border cells with a donor (area > 1)
__global__ void __launch_bounds__(256) k_drain_outlets(const int32_t* __restrict__ indeg, int dimx, int dimy,
                                                       unsigned long long* __restrict__ cnt) {
  const size_t n = (size_t)dimx * dimy;
  unsigned long long o = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i / (size_t)dimy), y = (int)(i % (size_t)dimy);
    o += drain_border(x, y, dimx, dimy) && indeg[i] > 0;
  }
  block_add_u64(o, &cnt[3]);
}

// Upstream area: one walker per cell without donors carries its area downstream.  At each receiver it adds its area,
// fences, and takes one from rem (a copy of the in-degrees); the walker that takes the last one owns the receiver's
// complete area and goes on from there.  Every cell is passed on exactly once, with integer sums.  *longest = the
// most receivers one walker visited.
__global__ void __launch_bounds__(256) k_drain_area(const int32_t* __restrict__ rcv, const int32_t* __restrict__ indeg,
                                                    int32_t* rem, unsigned long long* area, size_t n,
                                                    unsigned long long* __restrict__ longest) {
  unsigned long long most = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (indeg[i] != 0) continue;
    unsigned long long a = 1ull, hops = 0;
    int32_t r = rcv[i];
    SM_UNROLL1
    while (r >= 0) {
      atomicAdd(&area[r], a);
      __threadfence();
      hops++;
      if (atomicSub(&rem[r], 1) != 1) break;
      __threadfence();
      a = atomicAdd(&area[r], 0ull);
      r = rcv[r];
    }
    most = hops > most ? hops : most;
  }
  if (most) atomicMax(longest, most);
}

// basins: nxt = the receiver, or the cell itself on the border; then jumps nxt = nxt[nxt] until nothing changes
__global__ void __launch_bounds__(256) k_drain_basin_init(const int32_t* __restrict__ rcv, int32_t* __restrict__ nxt, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    nxt[i] = rcv[i] < 0 ? (int32_t)i : rcv[i];
}
__global__ void __launch_bounds__(256) k_drain_jump(int32_t* nxt, size_t n, unsigned long long* __restrict__ changed) {
  unsigned long long c = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int32_t a = nxt[i], b = nxt[a];
    if (a != b) { nxt[i] = b; c++; }
  }
  block_add_u64(c, changed);
}
// basin[i] = nxt[i] as int64, cells [c0, c0 + m)
__global__ void __launch_bounds__(256) k_drain_basin_out(const int32_t* __restrict__ nxt, size_t c0, size_t m,
                                                         int64_t* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (size_t)gridDim.x * blockDim.x)
    out[i] = (int64_t)nxt[c0 + i];
}

namespace {
struct DrainTimer {        // CUDA-event time of each phase's launches, summed per phase
  StrataEvents e;
  double ms[6] = {};
};
// the counters of one call, in one device array
enum { DC_FLAT, DC_DEPRESSED, DC_BAD, DC_OUTLETS, DC_LONGEST, DC_JUMP, DC_MARKS = 8, DC_N = DC_MARKS + DRAIN_BATCH };
}  // namespace

// One tiled relaxation, pass after pass until a pass marks no tile.  Returns the passes.
template <bool DIST>
static int drain_relax(sm_context* ctx, DrainTimer& tm, int phase, const double* H, double* W, int32_t* D,
                       unsigned int* act, unsigned long long* d_marks, int64_t* passes) {
  const int dimx = ctx->d.dimx, dimy = ctx->d.dimy;
  const int ntx = (dimx + DRAIN_T - 1) / DRAIN_T, nty = (dimy + DRAIN_T - 1) / DRAIN_T;
  const size_t nt = (size_t)ntx * nty;
  std::vector<unsigned int> ones(nt, 1u);
  CK(cudaMemcpyAsync(act, ones.data(), nt * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(act + nt, 0, nt * 4, ctx->stream));
  unsigned long long h_marks[DRAIN_BATCH];
  *passes = 0;
  for (int64_t p = 0;; p += DRAIN_BATCH) {
    CK(cudaMemsetAsync(d_marks, 0, sizeof(h_marks), ctx->stream));
    CK(cudaEventRecord(tm.e.e0, ctx->stream));
    for (int b = 0; b < DRAIN_BATCH; b++) {
      const int64_t q = p + b;
      k_drain_relax<DIST><<<(unsigned)nt, dim3(DRAIN_T, 256 / DRAIN_T), 0, ctx->stream>>>(
          H, W, D, dimx, dimy, ntx, nty, act + (q & 1) * nt, act + ((q + 1) & 1) * nt, d_marks + b);
      ctx->launches++;
    }
    CK(cudaGetLastError());
    CK(cudaEventRecord(tm.e.e1, ctx->stream));
    CK(cudaMemcpyAsync(h_marks, d_marks, sizeof(h_marks), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    float m = 0.f;
    CK(cudaEventElapsedTime(&m, tm.e.e0, tm.e.e1));
    tm.ms[phase] += m;
    for (int b = 0; b < DRAIN_BATCH; b++) {
      ++*passes;
      if (h_marks[b] == 0) return SM_OK;
    }
  }
}

extern "C" {

int sm_drainage(sm_context* ctx, int32_t flags, double* spill, int8_t* dir, int64_t* area, int64_t* basin,
                int32_t on_device, sm_drain_stats* stats) {
  if (flags & ~SM_DRAIN_GROUND) return fail(ctx, SM_ERR_INVALID, "sm_drainage: unknown flags");
  if (!spill && !dir && !area && !basin) return fail(ctx, SM_ERR_INVALID, "sm_drainage: no output requested");
  int rc;
  sm_context* c = ctx;       // the computing context: rank 0 of a group
  if (ctx->group) {
    if ((rc = grp_settle(ctx)) != SM_OK) return rc;
    c = ctx->group->rank[0];
  } else if ((rc = peers_ready(ctx)) != SM_OK) {
    return rc;
  }
  const bool multi = c->nranks > 1;
  const int dimx = c->d.dimx, dimy = c->d.dimy;
  const size_t N = (size_t)dimx * dimy;
  // the cells this call writes: the whole map, or a rank's strip
  const size_t c0 = ctx->group ? 0 : (size_t)c->x0 * dimy, m = ctx->group ? N : c->lcells;
  const bool want_rcv = dir || area || basin;
  const int ntx = (dimx + DRAIN_T - 1) / DRAIN_T, nty = (dimy + DRAIN_T - 1) / DRAIN_T;
  const size_t nt = (size_t)ntx * nty;
  sm_context* const ectx = ctx;         // errors are reported on the caller's handle
  ctx = c;                              // CK writes ctx->err: the computing context's
  auto done = [&](int r) { return ectx->group ? grp_err(ectx, 0, r) : r; };
  CK(cudaSetDevice(c->cfg.device));
  DevTmp t;
  // about 37 B per cell: H, W, D, rcv, indeg, dir, area
  double *H = nullptr, *W = nullptr;
  int32_t *D = nullptr, *rcv = nullptr, *indeg = nullptr;
  int8_t* dir8 = nullptr;
  unsigned long long *A = nullptr, *cnt = nullptr;
  unsigned int* act = nullptr;
  if ((rc = snap_alloc(c, t, N * 8, (void**)&H)) != SM_OK || (rc = snap_alloc(c, t, N * 8, (void**)&W)) != SM_OK ||
      (rc = snap_alloc(c, t, N * 4, (void**)&D)) != SM_OK || (rc = snap_alloc(c, t, nt * 8, (void**)&act)) != SM_OK ||
      (rc = snap_alloc(c, t, DC_N * 8, (void**)&cnt)) != SM_OK)
    return done(rc);
  if (want_rcv && ((rc = snap_alloc(c, t, N * 4, (void**)&rcv)) != SM_OK ||
                   (rc = snap_alloc(c, t, N * 4, (void**)&indeg)) != SM_OK || (rc = snap_alloc(c, t, N, (void**)&dir8)) != SM_OK))
    return done(rc);
  if (area && (rc = snap_alloc(c, t, N * 8, (void**)&A)) != SM_OK) return done(rc);
  CK(cudaMemsetAsync(cnt, 0, DC_N * 8, c->stream));
  DrainTimer tm;
  tm.e.device = c->cfg.device;
  CK(cudaEventCreate(&tm.e.e0));
  CK(cudaEventCreate(&tm.e.e1));
  const int G = c->num_sms * 8;
  // the nl launches enqueued by f, timed as phase `ph`
  auto timed = [&](int ph, int nl, auto f) -> int {
    CK(cudaEventRecord(tm.e.e0, c->stream));
    f();
    c->launches += nl;
    CK(cudaGetLastError());
    CK(cudaEventRecord(tm.e.e1, c->stream));
    CK(cudaEventSynchronize(tm.e.e1));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, tm.e.e0, tm.e.e1));
    tm.ms[ph] += ms;
    return SM_OK;
  };
  sm_drain_stats st = {};
  const int ground = (flags & SM_DRAIN_GROUND) ? 1 : 0;
  if ((rc = timed(0, 1, [&] {
         if (multi) k_drain_heights<true><<<G, 256, 0, c->stream>>>(c->d, ground, H, W);
         else k_drain_heights<false><<<G, 256, 0, c->stream>>>(c->d, ground, H, W);
       })) != SM_OK)
    return done(rc);
  if ((rc = drain_relax<false>(c, tm, 1, H, W, nullptr, act, cnt + DC_MARKS, &st.fill_passes)) != SM_OK) return done(rc);
  if ((rc = timed(2, 1, [&] { k_drain_classify<<<G, 256, 0, c->stream>>>(H, W, D, dimx, dimy, cnt); })) != SM_OK)
    return done(rc);
  if (want_rcv) {
    if ((rc = drain_relax<true>(c, tm, 2, nullptr, W, D, act, cnt + DC_MARKS, &st.dist_passes)) != SM_OK) return done(rc);
    CK(cudaMemsetAsync(indeg, 0, N * 4, c->stream));
    if ((rc = timed(3, 2, [&] {
           k_drain_receivers<<<G, 256, 0, c->stream>>>(W, D, dimx, dimy, dir8, rcv, indeg, A, cnt);
           k_drain_outlets<<<G, 256, 0, c->stream>>>(indeg, dimx, dimy, cnt);
         })) != SM_OK)
      return done(rc);
    if (area) {
      CK(cudaMemcpyAsync(D, indeg, N * 4, cudaMemcpyDeviceToDevice, c->stream));     // D is free now: the walkers' rem
      if ((rc = timed(4, 1, [&] { k_drain_area<<<G, 256, 0, c->stream>>>(rcv, indeg, D, A, N, cnt + DC_LONGEST); })) != SM_OK)
        return done(rc);
    }
    if (basin) {      // indeg is free now: the jump pointers
      if ((rc = timed(5, 1, [&] { k_drain_basin_init<<<G, 256, 0, c->stream>>>(rcv, indeg, N); })) != SM_OK) return done(rc);
      for (;;) {
        unsigned long long ch = 0;
        CK(cudaMemsetAsync(cnt + DC_JUMP, 0, 8, c->stream));
        if ((rc = timed(5, 1, [&] { k_drain_jump<<<G, 256, 0, c->stream>>>(indeg, N, cnt + DC_JUMP); })) != SM_OK) return done(rc);
        CK(cudaMemcpy(&ch, cnt + DC_JUMP, 8, cudaMemcpyDeviceToHost));
        st.jump_passes++;
        if (!ch) break;
      }
    }
  }
  unsigned long long h_cnt[DC_N] = {};
  CK(cudaMemcpy(h_cnt, cnt, sizeof(h_cnt), cudaMemcpyDeviceToHost));
  if (h_cnt[DC_BAD]) return done(fail(c, SM_ERR_CUDA, "sm_drainage: a cell without a receiver after the fill (internal error)"));
  // outputs: the cells [c0, c0 + m) of the whole-map rasters
  const cudaMemcpyKind kind = cudaMemcpyDefault;
  if (spill) CK(cudaMemcpyAsync(spill, W + c0, m * 8, kind, c->stream));
  if (dir) CK(cudaMemcpyAsync(dir, dir8 + c0, m, kind, c->stream));
  if (area) CK(cudaMemcpyAsync(area, A + c0, m * 8, kind, c->stream));
  if (basin) {
    int64_t* b64 = (int64_t*)H;      // H is free now
    k_drain_basin_out<<<G, 256, 0, c->stream>>>(indeg, c0, m, b64);
    c->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(basin, b64, m * 8, kind, c->stream));
  }
  CK(cudaStreamSynchronize(c->stream));
  if (ectx->group) ectx->group->dirty = false;
  st.flat_cells = (int64_t)h_cnt[DC_FLAT];
  st.depressed_cells = (int64_t)h_cnt[DC_DEPRESSED];
  st.outlets = (int64_t)h_cnt[DC_OUTLETS];
  st.longest_walk = (int64_t)h_cnt[DC_LONGEST];
  for (int i = 0; i < 6; i++) {
    st.phase_ms[i] = tm.ms[i];
    st.device_ms += tm.ms[i];
  }
  if (stats) *stats = st;
  return SM_OK;
}

}  // extern "C"
