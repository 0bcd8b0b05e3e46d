// sm_device.cuh -- device-side data layout and the accessor the sweep kernels hand to sm_core.cuh.
//
// HBM layout (DESIGN.md section 3):
//   top[x*dimy+y]      Sec32 (32 B = one DRAM sector): the TOP section of every column, so
//                      height()/surface() (43-89 calls per particle-step in the reference) are one
//                      sector read and >92 % of add()/remove() calls are one sector write.
//   pool[slot]         Sec32: buried sections, chained by `below`; two free rings keyed by sweep
//                      parity so that slots freed in sweep s are reused from sweep s+1 on without
//                      any lock (frees append to ring[s&1], allocations pop ring[(s+1)&1]).
//   wfreq/wtrack/windfreq  f32[y*dimx+x]   (water.h:53,349; wind.h:50)
//   particle SoA       16-byte vectors per particle (pa/pb/pc)
//   bins               per-sweep cell-bin lists of live particles used for the id-ordered
//                      conflict detection (head[parity][bin] = tag<<32 | particle, next/key per
//                      particle); tags make clearing unnecessary.
#pragma once
#include <cuda_runtime.h>
#include "sm_core.cuh"

#ifdef SM_PROFILE
#define SM_PROF_DECL unsigned long long prof_[16] = {0}; long long pt_ = clock64();
#define SM_PROF(i) { long long t_ = clock64(); prof_[i] += (unsigned long long)(t_ - pt_); pt_ = t_; }
#define SM_PROF_FLUSH(ctl) { for (int i_ = 0; i_ < 16; i_++) if (prof_[i_]) atomicAdd(&(ctl)->prof[i_], prof_[i_]); }
#else
#define SM_PROF_DECL
#define SM_PROF(i)
#define SM_PROF_FLUSH(ctl)
#endif

struct PoolRing {
  unsigned long long head;  // next entry to hand out (advanced only in sweeps of the other parity)
  unsigned long long tail;  // next entry to write   (advanced only in sweeps of this parity)
};

struct RunCtl {
  unsigned int barrier;         // monotone arrival counter of the grid barrier
  unsigned int alive_slot[3];   // live-particle totals, rotated per sweep
  unsigned int tag_base;        // first unused sweep tag
  unsigned int err;             // SM_ERR_* bits raised on device
  unsigned long long steps, sweeps, exit_oob, exit_evap, exit_stall, drops, alive;
  unsigned long long bump;      // pool high-water mark
  PoolRing ring[3];             // k_sweep: frees of sweep s go to ring[s%3], allocations pop ring[(s+1)%3] (filled in sweep s-2)
  unsigned long long prof[16];  // clock64() phase totals (built with -DSM_PROFILE only)
  unsigned long long marks[8];  // finer marks inside interact()
  // sharded maps: cross-rank barrier (every rank writes its arrival into every peer's copy)
  unsigned int xflag[8];        // xflag[r] = last global barrier epoch rank r arrived at
  unsigned int xalive[2][8];    // live particles rank r reported with that arrival (by epoch parity)
  unsigned int alive_total[2];  // sum over ranks, for the local blocks
  unsigned int release;         // global epoch the local blocks may pass
  unsigned int epoch_base;      // global epoch at the start of the next launch (never reset)
  // k_sweep's cross-rank barrier: xw[ge & 1][r] = (global epoch ge << 32) | live particles of rank r, written by
  // rank r into the copy of every rank it synchronises with at that epoch (its own included)
  unsigned long long xw[2][8];
  unsigned int ticket[3];       // k_sweep: next unclaimed live-particle rank beyond the first nslots, by sweep number mod 3
};

// Pointers of one rank's arrays, as seen from this rank (own arrays, same-process contexts, or CUDA-IPC
// mappings of a peer GPU's memory over NVLink).
#define SM_MAX_RANKS 8
struct PeerPtrs {
  Sec32* top;                    // that rank's strip of top records
  Sec32* pool;
  uint32_t* ringbuf[3];
  unsigned long long pool_cap;
  RunCtl* ctl;
  float4* pa; double2* pb; uint2* pc;
  unsigned char* alive;
  unsigned int* done;
  unsigned long long* head[2];
  uint2* node[2];
  double* bud;
  unsigned int* fin;
  unsigned int* lmask[3];
#ifdef SM_AUDIT_HANDOFF
  unsigned int* relz;
#endif
};

struct DevCtx {
  Sec32* top;
  Sec32* pool;
  uint32_t* ringbuf[3];
  unsigned long long pool_cap;
  float* wfreq;
  float* wtrack;
  float* windfreq;
  const SoilDev* soils;
  int nsoils;
  int dimx, dimy, scale;
  double volume_factor;          // WaterParticle::volumeFactor (water.h:368), default 0.015
  const float* wind_v4;          // lattice velocity field coupled to the wind particles (null: constant pspeed)
  int wind_nx, wind_ny, wind_nz;
  RunCtl* ctl;
  // particle batch
  float4* pa;        // water: px,py,sx,sy        | wind: px,py,sx,sy
  double2* pb;       // water: volume,sediment    | wind: sediment,height
  uint2* pc;         // water: contains,-         | wind: contains, bits(sz)
  unsigned char* alive;
  unsigned int* done;            // tag of the last sweep this particle completed (0xFFFFFFFF = dead)
  unsigned int* fin;             // exact kernel: tag of the last sweep whose map writes are complete
  unsigned long long* mv;        // exact kernel: tag<<32 | npos.x<<16 | npos.y, published right after move()
  unsigned int* lmask[3];        // k_sweep: live-particle bit masks (bit pid), rotated by sweep number mod 3
  double* bud;                   // mass budget: SM_BUDGET_SLOTS f64 accumulators per particle (contexts created with SM_FLAG_BUDGET)
  unsigned long long* head[2];   // bin heads per sweep parity
  uint2* node[2];                // per particle: .x = next particle in the bin list, .y = ipos x<<16|y
  int nbx, nby;                  // allocated bin grid (for the smallest bin edge)
  // sharding by x-strips: rank q owns the columns x in [q*strip_w, min((q+1)*strip_w, dimx)); its `top`
  // holds only that strip.  nranks == 1: one strip = the whole map.
  int nranks, rank, strip_w;
  unsigned long long* dbg;       // -DSM_PROFILE: per-sweep (clock64, live particles) of the last launch
  PeerPtrs peer[SM_MAX_RANKS];
#ifdef SM_AUDIT_HANDOFF
  unsigned int* relz;            // audit builds: tag of the last sweep whose hand-off this particle released
#endif
};

template <bool MULTI> __device__ __forceinline__ int owner_of_x(const DevCtx& c, int x) {
  if (!MULTI) return 0;
  const int q = x / c.strip_w;
  return q < c.nranks ? q : c.nranks - 1;
}
// top record of the global cell (x, y)
template <bool MULTI> __device__ __forceinline__ Sec32* cell_ptr(const DevCtx& c, int x, int y) {
  if (!MULTI) return &c.top[(size_t)x * c.dimy + y];
  const int q = owner_of_x<true>(c, x);
  return c.peer[q].top + (size_t)(x - q * c.strip_w) * c.dimy + y;
}

// ---- memory helpers: everything mutable is read through L2 (the TU is compiled -dlcm=cg) ----------
__device__ __forceinline__ unsigned int ld_volatile_u32(const unsigned int* p) {
  return *((const volatile unsigned int*)p);
}
__device__ __forceinline__ void st_volatile_u32(unsigned int* p, unsigned int v) {
  *((volatile unsigned int*)p) = v;
}
// acquire / release at gpu scope (the hand-off between dependent particle-steps)
__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(unsigned int* p, unsigned int v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// one release for several flag words: fence.acq_rel, then relaxed stores (the pattern st.release expands to)
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void st_relaxed_u32(unsigned int* p, unsigned int v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// relaxed polls: a spin loop reads with relaxed loads (an acquire load drags an L1 invalidation along on every
// iteration - CCTL.IVALL was 12 % of all stall samples of the first warp-kernel profile, and the poll traffic slows
// every other L2 access down) and acquires ONCE when the value it waited for has arrived
__device__ __forceinline__ unsigned int ld_relaxed_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned int ld_relaxed_sys_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
#ifndef SM_POLL_NS
#define SM_POLL_NS 0          // back-off between two polls of a spin loop, ns (0 = none)
#endif
__device__ __forceinline__ void poll_backoff() { if (SM_POLL_NS > 0) __nanosleep(SM_POLL_NS); }
// system scope: the other end may be a different GPU
__device__ __forceinline__ unsigned int ld_acquire_sys_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u32(unsigned int* p, unsigned int v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Grid-wide barrier for a co-resident (cooperative) grid: one arrival per block on a monotone
// counter.  `epoch` is a per-thread copy of how many barriers this launch has passed.
__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int& epoch) {
  __syncthreads();
  epoch++;
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    const unsigned int target = epoch * gridDim.x;
    while ((int)(ld_relaxed_u32(counter) - target) < 0) poll_backoff();
    __threadfence();
  }
  __syncthreads();
}

// Barrier across the blocks of EVERY rank of a sharded map.  Local blocks arrive on the local counter
// (reset by the host before each launch); block 0's thread 0 then publishes this rank's arrival and its
// live-particle count into every peer's RunCtl, waits for all peers, sums the counts and releases the
// local blocks.  Cross-rank words use a global epoch that is never reset, so no rank can erase another
// rank's arrival.  Returns the number of live particles over all ranks.
__device__ __forceinline__ unsigned int grid_barrier_multi(const DevCtx& c, unsigned int& epoch, unsigned int gbase,
                                                           unsigned int local_alive_slot) {
  // Only the rank leader (block 0, thread 0) uses system scope: the other blocks synchronise with it at
  // gpu scope (release: fence + arrival; acquire: the `release` word), and causality composes across the
  // two scopes, so their peer writes are ordered before the leader's system-scope flag.
  RunCtl* ctl = c.ctl;
  __syncthreads();
  epoch++;
  const unsigned int ge = gbase + epoch;           // global epoch of this barrier
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(&ctl->barrier, 1u);
    if (blockIdx.x == 0) {
      const unsigned int target = epoch * gridDim.x;
      while ((int)(ld_acquire_u32(&ctl->barrier) - target) < 0) { }
      const unsigned int mine = ld_volatile_u32(&ctl->alive_slot[local_alive_slot]);
#ifdef SM_XBAR_FENCES
      for (int q = 0; q < c.nranks; q++) st_volatile_u32(&c.peer[q].ctl->xalive[ge & 1u][c.rank], mine);
      __threadfence_system();
      for (int q = 0; q < c.nranks; q++) st_volatile_u32(&c.peer[q].ctl->xflag[c.rank], ge);
      unsigned int total = 0;
      for (int q = 0; q < c.nranks; q++) {
        while ((int)(ld_volatile_u32(&ctl->xflag[q]) - ge) < 0) { }
      }
      __threadfence_system();
      for (int q = 0; q < c.nranks; q++) total += ld_volatile_u32(&ctl->xalive[ge & 1u][q]);
#else
      // one system-scope release store per peer (orders the live count and every peer write of this rank
      // before the flag), one acquire poll per peer; no separate system fences
      for (int q = 0; q < c.nranks; q++) st_volatile_u32(&c.peer[q].ctl->xalive[ge & 1u][c.rank], mine);
      for (int q = 0; q < c.nranks; q++) st_release_sys_u32(&c.peer[q].ctl->xflag[c.rank], ge);
      unsigned int total = 0;
      for (int q = 0; q < c.nranks; q++) {
        while ((int)(ld_acquire_sys_u32(&ctl->xflag[q]) - ge) < 0) { }
        total += ld_volatile_u32(&ctl->xalive[ge & 1u][q]);
      }
#endif
      st_volatile_u32(&ctl->alive_total[ge & 1u], total);
      st_release_u32(&ctl->release, ge);
    } else {
      while ((int)(ld_acquire_u32(&ctl->release) - ge) < 0) { }
    }
  }
  __syncthreads();
  return ld_volatile_u32(&ctl->alive_total[ge & 1u]);
}

// ---- accessor: direct global records ------------------------------------------------------------
struct DevAccess {
  const DevCtx& c;
  const SoilDev* s_soils;   // shared-memory copy of the soil table
  unsigned int phase;       // sweep parity for the pool rings
  __device__ __forceinline__ DevAccess(const DevCtx& ctx, const SoilDev* ss, unsigned int ph)
      : c(ctx), s_soils(ss), phase(ph & 1u) {}
  __device__ __forceinline__ int dimx() const { return c.dimx; }
  __device__ __forceinline__ int dimy() const { return c.dimy; }
  __device__ __forceinline__ int scale() const { return c.scale; }
  __device__ __forceinline__ SoilDev soil(uint32_t t) const { return s_soils[t]; }
  __device__ __forceinline__ Sec32* rec(int x, int y) { return &c.top[(size_t)x * c.dimy + y]; }
  __device__ __forceinline__ double height(int x, int y) { return rec_height(*rec(x, y)); }
  __device__ __forceinline__ uint32_t surface_of(int x, int y) { return rec_surface(*rec(x, y)); }
  __device__ __forceinline__ void query(int x, int y, double& h, uint32_t& t) { const Sec32* r = rec(x, y); h = rec_height(*r); t = rec_surface(*r); }
  __device__ __forceinline__ void begin(int, int) {}
  __device__ __forceinline__ void target(int, int) {}
  __device__ __forceinline__ void dirty(int, int) {}
  __device__ __forceinline__ void dirty_rec(Sec32*, int, int) {}
  __device__ __forceinline__ void cascade_prefetch(int, int) {}
  __device__ __forceinline__ void mark(int) {}
  __device__ __forceinline__ void note_transfer() {}
  __device__ __forceinline__ void wet_mark(int, int) {}
  __device__ __forceinline__ double volume_factor() const { return c.volume_factor; }
  __device__ __forceinline__ void focus(int, int) {}
  __device__ __forceinline__ Sec32 pool_load(uint32_t i) { return c.pool[i]; }
  __device__ __forceinline__ void pool_store(uint32_t i, const Sec32& r) { c.pool[i] = r; }
  __device__ uint32_t pool_alloc() {
    // Pop from the ring that was filled during the previous phase (its tail is stable now).  No CAS
    // loop: under contention a CAS loop lets only one popper succeed per L2 round trip.  Instead every
    // popper takes a ticket with one atomicAdd; tickets >= tail are overshoots, undone with an
    // atomicMin(head, tail) (the head never drops below tail, so tickets < tail are unique), and served
    // from the bump allocator.
    PoolRing* R = &c.ctl->ring[phase ^ 1u];
    const unsigned long long t = R->tail;
    if (*((volatile unsigned long long*)&R->head) < t) {
      const unsigned long long h = atomicAdd(&R->head, 1ull);
      if (h < t) return c.ringbuf[phase ^ 1u][h % c.pool_cap];
      atomicMin(&R->head, t);
    }
    unsigned long long b = atomicAdd(&c.ctl->bump, 1ull);
    if (b < c.pool_cap) return (uint32_t)b;
    atomicOr(&c.ctl->err, 1u << 3);   // SM_ERR_POOL
    atomicAdd(&c.ctl->drops, 1ull);
    return SM_NIL;
  }
  __device__ void pool_free(uint32_t i) {
    PoolRing* R = &c.ctl->ring[phase];
    unsigned long long t = atomicAdd(&R->tail, 1ull);
    c.ringbuf[phase][t % c.pool_cap] = i;
  }
  __device__ __forceinline__ void track_add(int ind, double v) {     // water.h:348-351
    c.wtrack[ind] = (float)(c.wtrack[ind] + v);
  }
  __device__ __forceinline__ float water_frequency(int ind) { return c.wfreq[ind]; }
  __device__ __forceinline__ void wind_frequency_touch(int ind) {    // wind.h:49-52
    c.windfreq[ind] = (float)(0.5 * c.windfreq[ind] + 0.5f);
  }
};


// ---- accessor: shared-memory window ---------------------------------------------------------------
// The records a particle-step touches are staged in shared memory: patch A = the 3x3 block around
// ipos (slots 0-8; move() reads its plus-shaped subset), patch B = the 3x3 block around the new
// position (slots 9-17; bilinear height + cascade).  A cell inside both patches always resolves to
// patch A.  Records are pulled from L2 with cp.async (16-byte .cg copies straight into shared
// memory, all in flight at once), modified in place and written back once at the end of the step.
// Cells outside both patches (only the re-cascade of a wind step reaches them) are accessed in
// global memory directly.
#define SM_WIN_SLOTS 18
#define SM_WIN_BYTES (SM_WIN_SLOTS * 32)
#define SM_PLUS_MASK 186u   // (1<<1)|(1<<3)|(1<<4)|(1<<5)|(1<<7): the 5-point stencil inside a 3x3 patch

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  unsigned int d = (unsigned int)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

template <int KIND_, bool MULTI = false>
struct WinAccess {
  const DevCtx& c;
  const SoilDev* s_soils;
  Sec32* win;               // SM_WIN_SLOTS records in shared memory, private to this particle
  unsigned int phase;
  int ax, ay, bx, by;
  uint32_t valid, dirtym;
  bool has_b;
  float f_freq, f_track;    // water: frequency/track at ipos | wind: wind frequency at ipos
  int cur_q = 0;            // owner rank of the column the next col_* call works on (focus())
  long long t_begin = 0, t_target0 = 0, t_target1 = 0;
#ifdef SM_PROFILE
  long long t_last = 0; unsigned long long t_mark[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  __device__ __forceinline__ void mark(int i) { long long t = clock64(); t_mark[i] += (unsigned long long)(t - t_last); t_last = t; }
  unsigned int n_transfers = 0;
  __device__ __forceinline__ void note_transfer() { n_transfers++; }
#else
  __device__ __forceinline__ void mark(int) {}
  __device__ __forceinline__ void note_transfer() {}
#endif
  __device__ __forceinline__ WinAccess(const DevCtx& ctx, const SoilDev* ss, unsigned int ph, Sec32* w)
      : c(ctx), s_soils(ss), win(w), phase(ph & 1u), ax(0), ay(0), bx(0), by(0), valid(0), dirtym(0),
        has_b(false), f_freq(0.f), f_track(0.f) {}
  __device__ __forceinline__ int dimx() const { return c.dimx; }
  __device__ __forceinline__ int dimy() const { return c.dimy; }
  __device__ __forceinline__ int scale() const { return c.scale; }
  __device__ __forceinline__ SoilDev soil(uint32_t t) const { return s_soils[t]; }

  // issue the copies for the wanted cells of one patch (no wait)
  __device__ __forceinline__ void issue_patch(int ox, int oy, int base, uint32_t want) {
    uint32_t got = 0;
#pragma unroll
    for (int k = 0; k < 9; k++) {
      const int x = ox + k / 3 - 1, y = oy + k % 3 - 1;
      bool need = ((want >> k) & 1u) && !((valid >> (base + k)) & 1u) && x >= 0 && y >= 0 &&
                  x < c.dimx && y < c.dimy;
      if (base == 9 && need) {
        const int dx = x - ax + 1, dy = y - ay + 1;
        if ((unsigned)dx < 3u && (unsigned)dy < 3u) need = false;   // resolves to patch A
      }
      if (need) {
        const Sec32* src = cell_ptr<MULTI>(c, x, y);
        cp_async16(&win[base + k], src);
        cp_async16(((char*)&win[base + k]) + 16, ((const char*)src) + 16);
        got |= 1u << k;
      }
    }
    valid |= got << base;
  }
  __device__ __forceinline__ void begin(int ix, int iy) {
    ax = ix; ay = iy; has_b = false; valid = 0; dirtym = 0;
    issue_patch(ix, iy, 0, KIND_ == 1 ? 0x1FFu : SM_PLUS_MASK);   // wind cascades around ipos almost every step: fetch the whole patch at once
    const int ind = iy * c.dimx + ix;
    if (KIND_ == 0) { f_freq = c.wfreq[ind]; f_track = c.wtrack[ind]; }
    else { f_freq = c.windfreq[ind]; }
    cp_async_wait_all();
#ifdef SM_PROFILE
    t_begin = clock64();
#endif
  }
  __device__ __forceinline__ void target(int nx, int ny) {
    bx = nx; by = ny; has_b = true;
#ifdef SM_PROFILE
    t_target0 = clock64();
#endif
    issue_patch(nx, ny, 9, 0x1FFu);
    cp_async_wait_all();
#ifdef SM_PROFILE
    t_target1 = clock64(); t_last = t_target1;
#endif
  }
  __device__ __forceinline__ void cascade_prefetch(int cx, int cy) {
    if (cx == ax && cy == ay) { issue_patch(ax, ay, 0, 0x1FFu); cp_async_wait_all(); }
    else if (has_b && cx == bx && cy == by) { issue_patch(bx, by, 9, 0x1FFu); cp_async_wait_all(); }
  }
  __device__ __forceinline__ int slot_of(int x, int y) const {
    int dx = x - ax + 1, dy = y - ay + 1;
    if ((unsigned)dx < 3u && (unsigned)dy < 3u) return dx * 3 + dy;
    if (has_b) {
      dx = x - bx + 1; dy = y - by + 1;
      if ((unsigned)dx < 3u && (unsigned)dy < 3u) return 9 + dx * 3 + dy;
    }
    return -1;
  }
  __device__ __forceinline__ Sec32* rec(int x, int y) {
    const int s = slot_of(x, y);
    Sec32* g = cell_ptr<MULTI>(c, x, y);
    if (s < 0) return g;
    if (!((valid >> s) & 1u)) { win[s] = *g; valid |= 1u << s; }
    return &win[s];
  }
  __device__ __forceinline__ void dirty(int x, int y) {
    const int s = slot_of(x, y);
    if (s >= 0) dirtym |= 1u << s;
  }
  // mark a record obtained from rec() dirty without looking its slot up again
  __device__ __forceinline__ void dirty_rec(Sec32* r, int, int) {
    const long off = r - win;
    if (off >= 0 && off < SM_WIN_SLOTS) dirtym |= 1u << (int)off;
  }
  // read-only queries served from the window with shared-memory loads (no generic pointer is formed)
  // (measured: -5 % on the water kernel, +11 % on the wind kernel, so wind keeps the pointer path)
  __device__ __forceinline__ double height(int x, int y) {
    if (KIND_ == 1) return rec_height(*rec(x, y));
    const int s = slot_of(x, y);
    if (s >= 0) {
      if (!((valid >> s) & 1u)) { win[s] = *cell_ptr<MULTI>(c, x, y); valid |= 1u << s; }
      const double sz = win[s].size, fl = win[s].floor;
      return win[s].type == SM_EMPTY ? 0.0 : (fl + sz);
    }
    return rec_height(*cell_ptr<MULTI>(c, x, y));
  }
  // height and surface type of one cell with a single slot lookup
  __device__ __forceinline__ void query(int x, int y, double& h, uint32_t& t) {
    if (KIND_ == 1) { const Sec32* r = rec(x, y); h = rec_height(*r); t = rec_surface(*r); return; }
    const int s = slot_of(x, y);
    if (s >= 0) {
      if (!((valid >> s) & 1u)) { win[s] = *cell_ptr<MULTI>(c, x, y); valid |= 1u << s; }
      const double sz = win[s].size, fl = win[s].floor;
      const uint32_t ty = win[s].type;
      h = (ty == SM_EMPTY) ? 0.0 : (fl + sz);
      t = (ty == SM_EMPTY) ? 0u : ty;
      return;
    }
    const Sec32 r = *cell_ptr<MULTI>(c, x, y);
    h = rec_height(r); t = rec_surface(r);
  }
  __device__ __forceinline__ uint32_t surface_of(int x, int y) {
    if (KIND_ == 1) return rec_surface(*rec(x, y));
    const int s = slot_of(x, y);
    if (s >= 0) {
      if (!((valid >> s) & 1u)) { win[s] = *cell_ptr<MULTI>(c, x, y); valid |= 1u << s; }
      const uint32_t t = win[s].type;
      return t == SM_EMPTY ? 0u : t;
    }
    return rec_surface(*cell_ptr<MULTI>(c, x, y));
  }
  // write the modified records back (end of step)
  __device__ __forceinline__ void flush() {
    uint32_t m = dirtym;
    while (m) {
      const int s = __ffs(m) - 1;
      m &= m - 1;
      int x, y;
      if (s < 9) { x = ax + s / 3 - 1; y = ay + s % 3 - 1; }
      else { x = bx + (s - 9) / 3 - 1; y = by + (s - 9) % 3 - 1; }
      *cell_ptr<MULTI>(c, x, y) = win[s];
    }
    dirtym = 0;
  }
  __device__ __forceinline__ void focus(int x, int) { if (MULTI) cur_q = owner_of_x<true>(c, x); }
  __device__ __forceinline__ Sec32 pool_load(uint32_t i) { return MULTI ? c.peer[cur_q].pool[i] : c.pool[i]; }
  __device__ __forceinline__ void pool_store(uint32_t i, const Sec32& r) {
    if (MULTI) c.peer[cur_q].pool[i] = r; else c.pool[i] = r;
  }
  __device__ uint32_t pool_alloc() {
    if (!MULTI) { DevAccess d(c, s_soils, phase); return d.pool_alloc(); }
    // same ticket pop as DevAccess::pool_alloc, on the owner's rings / bump counter
    const PeerPtrs& P = c.peer[cur_q];
    PoolRing* R = &P.ctl->ring[phase ^ 1u];
    const unsigned long long t = *((volatile unsigned long long*)&R->tail);
    if (*((volatile unsigned long long*)&R->head) < t) {
      const unsigned long long h = atomicAdd(&R->head, 1ull);
      if (h < t) return P.ringbuf[phase ^ 1u][h % P.pool_cap];
      atomicMin(&R->head, t);
    }
    unsigned long long b = atomicAdd(&P.ctl->bump, 1ull);
    if (b < P.pool_cap) return (uint32_t)b;
    atomicOr(&c.ctl->err, 1u << 3);
    atomicAdd(&c.ctl->drops, 1ull);
    return SM_NIL;
  }
  __device__ void pool_free(uint32_t i) {
    if (!MULTI) { DevAccess d(c, s_soils, phase); d.pool_free(i); return; }
    const PeerPtrs& P = c.peer[cur_q];
    PoolRing* R = &P.ctl->ring[phase];
    unsigned long long t = atomicAdd(&R->tail, 1ull);
    P.ringbuf[phase][t % P.pool_cap] = i;
  }
  __device__ __forceinline__ void track_add(int ind, double v) {     // water.h:348-351
    c.wtrack[ind] = (float)(f_track + v);
  }
  __device__ __forceinline__ float water_frequency(int) { return f_freq; }
  __device__ __forceinline__ void wind_frequency_touch(int ind) {    // wind.h:49-52
    c.windfreq[ind] = (float)(0.5 * f_freq + 0.5f);
  }
};
