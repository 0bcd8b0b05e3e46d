// sm_core.cuh -- column operations and particle-step arithmetic of the hot path.
//
// Everything here is written against an "accessor" A that hands out mutable top-of-column
// records, so the same arithmetic runs (a) inside the sm_90a sweep kernels on records staged in
// shared memory / read through L2, and (b) on the host inside the facade's single-cell calls.
// The arithmetic is a type-exact transcription of the reference expressions: every float/double
// promotion, association order and narrowing is kept, FMA contraction must be OFF
// (nvcc -fmad=false, gcc -ffp-contract=off) and division / sqrt must be IEEE (nvcc defaults).
//
// Reference map:  Layermap::add/remove/height/normal/surface  source/layermap.h:230-439
//                 Particle::cascade                             source/particle/particle.h:24-101
//                 WaterParticle::move/interact                  source/particle/water.h:43-121
//                 WindParticle::move/interact                   source/particle/wind.h:54-136
//                 GLM semantics (normalize, mix, cross, round)  SURVEY.md section 8c
#pragma once
#include <stdint.h>
#include <math.h>

#if defined(__CUDACC__)
#define SM_HD __host__ __device__ __forceinline__
#define SM_HD_NOINLINE __host__ __device__ __noinline__
#define SM_UNROLL1 _Pragma("unroll 1")
#else
#define SM_HD inline
#define SM_HD_NOINLINE inline
#define SM_UNROLL1
#endif

#if defined(__CUDA_ARCH__)
#define SM_FFS(x) __ffs((int)(x))
#else
#define SM_FFS(x) __builtin_ffs((int)(x))
#endif
#define SM_NIL 0xFFFFFFFFu
#define SM_EMPTY 0xFFFFFFFFu   // Sec32::type of an empty column (dat[] == NULL, layermap.h:176)
#define SM_AIR 0u              // soilmap["Air"] (surface.h:53-57)

// One run of a column ("sec", layermap.h:37-62) as a 32-byte record = one DRAM sector.
// The TOP section of every cell lives in DevMap::top[x*dimy+y]; buried sections live in the pool
// and are chained through `below` (the reference's `prev`).
struct
#if defined(__CUDACC__)
    __align__(32)
#else
    alignas(32)
#endif
        Sec32 {
  double size;        // run length              (sec::size)
  double floor;       // cumulative height below (sec::floor)
  double saturation;  // (sec::saturation) carried, only hydrology changes it
  uint32_t type;      // SurfType, SM_EMPTY = no section
  uint32_t below;     // pool slot of the section underneath, SM_NIL = none
};

// the SurfParam fields the path reads (surface.h:11-39)
struct SoilDev {
  float friction, solubility, equrate, erosionrate, maxdiff, settling, suspension, porosity;
  uint32_t transports, erodes, cascades, abrades;
};

struct WaterP {  // WaterParticle state that survives a step (water.h:27-41, particle.h:16-18)
  float px, py, sx, sy;
  double volume, sediment;
  uint32_t contains;
};
struct WindP {  // WindParticle state (wind.h:29-40)
  float px, py;
  float sx, sy, sz;
  double sediment, height;
  uint32_t contains;
};

enum { SM_ALIVE = 0, SM_EXIT_OOB = 1, SM_EXIT_STALL = 2, SM_EXIT_EVAP = 3 };

// Accessor contract used below: rec(x,y) -> mutable top record; focus(x,y) names the column whose pool
// the next col_* call may touch (columns of different owners keep their buried sections in different
// pools when the map is sharded); dirty(x,y); begin/target/cascade_prefetch are staging hints; mark(i)
// is a profiling hook.
// ------------------------------------------------------------------------------------------------
// record-level column operations
// ------------------------------------------------------------------------------------------------
SM_HD double rec_height(const Sec32& r) {  // Layermap::height(ivec2), layermap.h:422-425
  return r.type == SM_EMPTY ? 0.0 : (r.floor + r.size);
}
SM_HD uint32_t rec_surface(const Sec32& r) {  // Layermap::surface, layermap.h:417-420
  return r.type == SM_EMPTY ? 0u : r.type;
}
SM_HD void rec_set_empty(Sec32& r) {
  r.size = 0.0; r.floor = 0.0; r.saturation = 0.0; r.type = SM_EMPTY; r.below = SM_NIL;
}

// dat[] = E->prev; pool.unget(E)   (layermap.h:318-320, 332-334)
template <class A> SM_HD void col_pop(A& a, Sec32& r) {
  uint32_t b = r.below;
  if (b == SM_NIL) {
    rec_set_empty(r);
  } else {
    r = a.pool_load(b);
    a.pool_free(b);
  }
}
// E->prev = dat[]; E->floor = height(pos); dat[] = E   (layermap.h:302-305)
template <class A> SM_HD void col_push(A& a, Sec32& r, double size, uint32_t type, double sat) {
  uint32_t slot = a.pool_alloc();
  if (slot == SM_NIL) return;  // pool exhausted: the reference drops the section (layermap.h:92-95,232-234)
  a.pool_store(slot, r);
  double fl = r.floor + r.size;
  r.size = size; r.floor = fl; r.saturation = sat; r.type = type; r.below = slot;
}

// Layermap::add(pos, E) with E = sec(size,type) carrying `sat`  (layermap.h:230-307)
template <class A> SM_HD void col_add(A& a, Sec32& r, double size, uint32_t type, double sat = 0.0) {
  if (size <= 0) return;                       // :237-240
  if (r.type == SM_EMPTY) {                    // :243-246
    r.size = size; r.floor = 0.0; r.saturation = sat; r.type = type; r.below = SM_NIL;
    return;
  }
  if (r.type == type) {                        // :249-253
    r.size += size;
    return;
  }
  if (r.type == SM_AIR) {                      // :258-275  insert under the water section
    double wsize = r.size, wsat = r.saturation;
    uint32_t b = r.below;
    if (b == SM_NIL) rec_set_empty(r);
    else { r = a.pool_load(b); a.pool_free(b); }
    // add(pos, E): the section under water is never Air (adjacent equal types merge)
    if (r.type == SM_EMPTY) {
      r.size = size; r.floor = 0.0; r.saturation = sat; r.type = type; r.below = SM_NIL;
    } else if (r.type == type) {
      r.size += size;
    } else {
      col_push(a, r, size, type, sat);
    }
    // add(pos, top): the water section goes back on with a recomputed floor (:302-305)
    if (wsize <= 0) return;
    if (r.type == SM_AIR) r.size += wsize;    // only reachable when `type` could not be pushed
    else col_push(a, r, wsize, SM_AIR, wsat);
    return;
  }
  col_push(a, r, size, type, sat);             // :302-305
}

// Layermap::remove(pos, h) -> leftover   (layermap.h:310-339)
template <class A> SM_HD double col_remove(A& a, Sec32& r, double h) {
  if (r.type == SM_EMPTY) return 0.0;          // :313-314
  if (r.size <= 0.0) {                         // :317-322
    col_pop(a, r);
    return 0.0;
  }
  if (h <= 0.0) return 0.0;                    // :325-326
  double diff = h - r.size;                    // :328-329
  r.size -= h;
  if (diff >= 0.0) {                           // :331-336
    col_pop(a, r);
    return diff;
  }
  return 0.0;
}

// ------------------------------------------------------------------------------------------------
// queries through the accessor
// ------------------------------------------------------------------------------------------------
// read-only queries go through the accessor so that it can serve them from its staged copy without
// forming a generic pointer (shared-memory loads instead of generic ones on the device)
template <class A> SM_HD double map_height(A& a, int x, int y) { return a.height(x, y); }

// Layermap::height(vec2), layermap.h:427-439 (weights cross-wired exactly as upstream)
template <class A> SM_HD double map_height_bilinear(A& a, float px, float py) {
  float fx = floorf(px), fy = floorf(py);
  int ix = (int)fx, iy = (int)fy;
  float wx = px - fx, wy = py - fy;            // fract = x - floor(x)
  double h = 0.0;
  h += (1.0 - wx) * (1.0 - wy) * map_height(a, ix, iy);
  h += (1.0 - wx) * wy * map_height(a, ix + 1, iy);
  h += wx * (1.0 - wy) * map_height(a, ix, iy + 1);
  h += wx * wy * map_height(a, ix + 1, iy + 1);   // wx*wy is a float product
  return h;
}

struct sm_f3 { float x, y, z; };
SM_HD sm_f3 f3_sub(sm_f3 a, sm_f3 b) { return sm_f3{a.x - b.x, a.y - b.y, a.z - b.z}; }
SM_HD sm_f3 f3_cross(sm_f3 x, sm_f3 y) {
  return sm_f3{x.y * y.z - y.y * x.z, x.z * y.x - y.z * x.x, x.x * y.y - y.x * x.y};
}

// Layermap::normal(ivec2), layermap.h:341-377
template <class A> SM_HD sm_f3 map_normal(A& a, int x, int y) {
  const int SCALE = a.scale();
  const int dimx = a.dimx(), dimy = a.dimy();
  sm_f3 n{0.0f, 0.0f, 0.0f};
  sm_f3 p{(float)x, (float)(SCALE * map_height(a, x, y)), (float)y};
  int k = 0;
  // the four neighbour heights are shared by the quadrants; each is read once
  float hxm = 0.0f, hxp = 0.0f, hym = 0.0f, hyp = 0.0f;
  if (x > 0) hxm = (float)(SCALE * map_height(a, x - 1, y));
  if (x < dimx - 1) hxp = (float)(SCALE * map_height(a, x + 1, y));
  if (y > 0) hym = (float)(SCALE * map_height(a, x, y - 1));
  if (y < dimy - 1) hyp = (float)(SCALE * map_height(a, x, y + 1));
  if (x > 0 && y > 0) {
    sm_f3 b{(float)(x - 1), hxm, (float)y};
    sm_f3 c{(float)x, hym, (float)(y - 1)};
    sm_f3 r = f3_cross(f3_sub(c, p), f3_sub(b, p));
    n.x += r.x; n.y += r.y; n.z += r.z;
    k++;
  }
  if (x > 0 && y < dimy - 1) {
    sm_f3 b{(float)(x - 1), hxm, (float)y};
    sm_f3 c{(float)x, hyp, (float)(y + 1)};
    sm_f3 r = f3_cross(f3_sub(c, p), f3_sub(b, p));
    n.x -= r.x; n.y -= r.y; n.z -= r.z;
    k++;
  }
  if (x < dimx - 1 && y > 0) {
    sm_f3 b{(float)(x + 1), hxp, (float)y};
    sm_f3 c{(float)x, hym, (float)(y - 1)};
    sm_f3 r = f3_cross(f3_sub(c, p), f3_sub(b, p));
    n.x -= r.x; n.y -= r.y; n.z -= r.z;
    k++;
  }
  if (x < dimx - 1 && y < dimy - 1) {
    sm_f3 b{(float)(x + 1), hxp, (float)y};
    sm_f3 c{(float)x, hyp, (float)(y + 1)};
    sm_f3 r = f3_cross(f3_sub(c, p), f3_sub(b, p));
    n.x += r.x; n.y += r.y; n.z += r.z;
    k++;
  }
  float fk = (float)k;
  n.x = n.x / fk; n.y = n.y / fk; n.z = n.z / fk;               // n/(float)k
  float d = n.x * n.x + n.y * n.y + n.z * n.z;                  // normalize = v * (1/sqrt(dot))
  float inv = 1.0f / sqrtf(d);
  return sm_f3{n.x * inv, n.y * inv, n.z * inv};
}

// ------------------------------------------------------------------------------------------------
// Particle::cascade, particle.h:24-101.  DEPTH = how many nested re-cascades are compiled in.
// ------------------------------------------------------------------------------------------------
template <int DEPTH, class A> struct Cascade {
  static SM_HD void run(A& a, int cx, int cy, int transferloop) {
    const int dimx = a.dimx(), dimy = a.dimy();
    const int SCALE = a.scale();
    a.cascade_prefetch(cx, cy);
    a.mark(3);
    // Neighbour k = 0..7 in the order of particle.h:30-39; with kk = k + (k >= 4) the offset is
    // (kk/3 - 1, kk%3 - 1).  The reference sorts the in-bounds neighbours by their height BEFORE any
    // transfer, highest first, with std::sort = stable insertion sort on <= 8 elements
    // (particle.h:58-60).  (height desc, k asc) is a total order, so the sorted sequence is unique:
    // rank[k] = #{j : h[j] > h[k] or (h[j] == h[k] and j < k)}, all in registers.
    double h[8];
    uint32_t nty[8];
    int num = 0;
    unsigned int inb = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const int kk = k + (k >= 4 ? 1 : 0);
      const int nx = cx + kk / 3 - 1, ny = cy + kk % 3 - 1;
      const bool in = !(nx >= dimx || ny >= dimy || nx < 0 || ny < 0);   // :51-52
      h[k] = -1.0e300;                                                   // out of bounds sorts last
      nty[k] = 0u;
      if (in) {
        a.query(nx, ny, h[k], nty[k]);
        inb |= 1u << k;
        num++;
      }
    }
    a.mark(4);
    // Speculative pass (all eight neighbours at once, instruction-level parallel): which
    // neighbours would transfer if the loop below met them with the map in its CURRENT state?
    // Until the first transfer happens nothing changes, so the loop may skip the others; after a
    // transfer every neighbour is evaluated exactly as the reference does.
    unsigned int active = 0;
    {
      double hc;
      uint32_t cty;
      a.query(cx, cy, hc, cty);
      const float cmax = a.soil(cty).maxdiff;
#pragma unroll
      for (int k = 0; k < 8; k++) {
        // diff = (float)(dd / 80.0f); its sign is dd's.  |dd| < 80*maxdiff*(1 - 2^-20) already proves
        // |diff| <= maxdiff (rounding is monotone), i.e. no excess: the IEEE double division is only
        // paid for neighbours near or above the threshold.
        const double dd = (hc - h[k]) * (float)SCALE;
        const float md = (dd > 0) ? cmax : a.soil(nty[k]).maxdiff;
        if (!(fabs(dd) < 80.0 * (double)md * (1.0 - 9.5367431640625e-07))) {
          const float diff = (float)(dd / 80.0f);
          const float excess = fabsf(diff) - md;
          if (((inb >> k) & 1u) && !(diff == 0) && !(excess <= 0)) active |= 1u << k;
        }
      }
    }
    a.mark(5);
    if (active == 0) return;
    int rank[8];
#pragma unroll
    for (int k = 0; k < 8; k++) rank[k] = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
#pragma unroll
      for (int j = k + 1; j < 8; j++) {
        const bool j_first = h[j] > h[k];          // strictly higher goes first; ties keep k before j
        rank[k] += j_first ? 1 : 0;
        rank[j] += j_first ? 0 : 1;
      }
    }
    unsigned int order = 0;                         // nibble i = neighbour with rank i
#pragma unroll
    for (int k = 0; k < 8; k++) order |= (unsigned int)k << (4 * rank[k]);

    // Ranks still to be looked at, as a bit mask over the sorted order.  Until the first transfer only the
    // neighbours the speculative pass found active matter; after a transfer every later rank is evaluated,
    // exactly as the reference loop does.  Iterating over the set bits (instead of over all ranks with
    // `continue`) keeps the trip count of a warp at the LARGEST per-lane count rather than at the union of
    // the ranks any lane needs - the lanes of a warp carry different particles.
    unsigned int todo = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int k = (int)((order >> (4 * i)) & 7u);
      if (i < num && ((active >> k) & 1u)) todo |= 1u << i;
    }
    const unsigned int allranks = (num >= 8) ? 0xFFu : ((1u << num) - 1u);
    Sec32* const pc = a.rec(cx, cy);                // the centre record: one lookup for the whole loop
    SM_UNROLL1
    while (todo) {
      const int i = SM_FFS(todo) - 1;
      todo &= todo - 1u;
      const int k = (int)((order >> (4 * i)) & 7u);
      const int kk = k + (k >= 4 ? 1 : 0);
      const int nx = cx + kk / 3 - 1, ny = cy + kk % 3 - 1;
      Sec32* const pn = a.rec(nx, ny);              // one lookup per neighbour and iteration
      // :66  full height difference, narrowed to float.  Same division-free proof as in the speculative
      // pass, on the CURRENT heights: |dd| < 80*maxdiff*(1 - 2^-20) => diff == 0 or excess <= 0 => continue.
      const double dd2 = (rec_height(*pc) - rec_height(*pn)) * (float)SCALE;
      Sec32* const tr = (dd2 > 0) ? pc : pn;        // :71-72 the higher cell ...
      Sec32* const br = (dd2 > 0) ? pn : pc;        //        ... and the lower one
      const uint32_t type = rec_surface(*tr);       // :74-75
      const SoilDev sp = a.soil(type);
      if (fabs(dd2) < 80.0 * (double)sp.maxdiff * (1.0 - 9.5367431640625e-07)) continue;
      float diff = (float)(dd2 / 80.0f);
      if (diff == 0) continue;
      const int tx = (diff > 0) ? cx : nx, ty = (diff > 0) ? cy : ny;
      const int bx = (diff > 0) ? nx : cx, by = (diff > 0) ? ny : cy;
      float excess = fabsf(diff) - sp.maxdiff;                      // :78
      if (excess <= 0) continue;
      float transfer = sp.settling * excess / 2.0f;                 // :83
      double tsize = (tr->type == SM_EMPTY) ? 0.0 : tr->size;
      if (transfer > tsize) transfer = (float)tsize;                // :87-88 (f64 -> f32 narrowing)
      bool recascade = false;
      todo |= allranks & ~((2u << i) - 1u);          // from now on every later rank is evaluated
      a.note_transfer();
      a.focus(tx, ty);
      if (col_remove(a, *tr, (double)transfer) != 0) recascade = true;   // :90-91
      a.dirty_rec(tr, tx, ty);
      a.focus(bx, by);
      col_add(a, *br, (double)transfer, sp.cascades);               // :92
      a.dirty_rec(br, bx, by);
      if constexpr (DEPTH > 0) {
        if (recascade && transferloop > 0) {                        // :96-97
          --transferloop;
          Cascade<DEPTH - 1, A>::run(a, nx, ny, transferloop);
        }
      }
    }
  }
};

// ------------------------------------------------------------------------------------------------
// WaterParticle  (water.h)
// ------------------------------------------------------------------------------------------------
#define SM_SQRT2F 1.41421354f   // sqrt(2.0f) rounded to float (water.h:61)

// A NaN with the bits the reference's x86 build gives it.  SSE returns the default NaN 0xFFC00000 for an invalid
// operation and carries that NaN through the arithmetic after it; CUDA returns 0x7FFFFFFF for every NaN result.
// water.h:60-62 makes one when mix(n.xz, speed, friction) is the zero vector (friction 1 on a particle at rest:
// normalize is 0 * inf); the particle then leaves the map, but its speed and position stay in its state.
SM_HD float host_nan(float v) {
  union { uint32_t u; float f; } nan = {0xFFC00000u};
  return v == v ? v : nan.f;
}

// ctor body water.h:14-17 / wind.h:17-20: what the particle transports
template <class A> SM_HD uint32_t spawn_contains(A& a, float px, float py) {
  int ix = (int)roundf(px), iy = (int)roundf(py);
  return a.soil(rec_surface(*a.rec(ix, iy))).transports;
}

// one move() && interact().  `a` must cover plus(ipos) and the 3x3 around the new position.
// What move() hands to interact() of the same step (the friction-modified `param` copy of water.h:48-54
// is only read for solubility and equrate afterwards).
struct WaterMid {
  float freq, solubility, equrate;
  double evaprate;
  int ix, iy;
};

// WaterParticle::move, water.h:43-73.  `a` must cover plus(ipos).  Returns SM_ALIVE when interact() follows.
template <class A> SM_HD int water_move(A& a, WaterP& p, WaterMid& m) {
  const int dimx = a.dimx(), dimy = a.dimy();
  const int ix = (int)roundf(p.px), iy = (int)roundf(p.py);        // :45
  a.begin(ix, iy);
  sm_f3 n = map_normal(a, ix, iy);                                  // :46
  Sec32* ir = a.rec(ix, iy);
  uint32_t surface = rec_surface(*ir);                              // :47
  SoilDev param = a.soil(surface);                                  // :48
  double evaprate = 0.01;                                           // :49
  const int ind = iy * dimx + ix;
  a.track_add(ind, p.volume);                                       // :50, 348-351
  const float freq = a.water_frequency(ind);
  param.friction = param.friction * (1.0f - freq);                  // :53
  evaprate = evaprate * (1.0f - 0.2f * freq);                       // :54
  m.freq = freq; m.solubility = param.solubility; m.equrate = param.equrate; m.evaprate = evaprate;
  m.ix = ix; m.iy = iy;
  {
    float vx = n.x * param.friction, vz = n.z * param.friction;     // :56
    float len = sqrtf(vx * vx + vz * vz);
    if (len < 1E-5) return SM_EXIT_STALL;
  }
  {
    float f = param.friction;                                       // :60 mix(n.xz, speed, friction)
    float mx = n.x * (1.0f - f) + p.sx * f;
    float my = n.z * (1.0f - f) + p.sy * f;
    float inv = 1.0f / sqrtf(mx * mx + my * my);                    // :61 sqrt(2)*normalize
    p.sx = host_nan(SM_SQRT2F * (mx * inv));
    p.sy = host_nan(SM_SQRT2F * (my * inv));
  }
  p.px = host_nan(p.px + p.sx);                                     // :62
  p.py = host_nan(p.py + p.sy);
  if (!(p.px >= 0.0f && p.py >= 0.0f) ||                            // :65-69
      !(p.px < (float)dimx - 1.0f && p.py < (float)dimy - 1.0f)) {
    p.volume = 0.0;
    return SM_EXIT_OOB;
  }
  return SM_ALIVE;
}

// WaterParticle::interact, water.h:75-121.  `a` must still hold the record of ipos; the 3x3 block around
// the new position is staged here.
template <class A> SM_HD int water_interact(A& a, WaterP& p, const WaterMid& m) {
  const int SCALE = a.scale();
  const int ix = m.ix, iy = m.iy;
  const float freq = m.freq;
  const double evaprate = m.evaprate;
  Sec32* ir = a.rec(ix, iy);
  const int nx = (int)roundf(p.px), ny = (int)roundf(p.py);
  a.target(nx, ny);
  double c_eq = m.solubility * (rec_height(*ir) - map_height_bilinear(a, p.px, p.py)) *
                (double)SCALE / 80.0;                               // :78
  if (c_eq < 0.0) c_eq = 0.0;
  if (c_eq > 1.0) c_eq = 1.0;
  a.mark(1);
  if ((double)(a.soil(p.contains).erosionrate) < freq)              // :83-84
    p.contains = a.soil(p.contains).erodes;
  double cdiff = c_eq - p.sediment;                                 // :87
  if (cdiff > 0) {                                                  // :91-101
    p.sediment += m.equrate * cdiff;
    p.contains = a.soil(rec_surface(*ir)).transports;
    a.focus(ix, iy);
    double diff = col_remove(a, *ir, m.equrate * cdiff * p.volume);
    SM_UNROLL1
    while (fabs(diff) > 1E-8) diff = col_remove(a, *ir, diff);
    a.dirty(ix, iy);
  } else if (cdiff < 0) {                                           // :105-110
    const float eq = a.soil(p.contains).equrate;
    p.sediment += eq * cdiff;
    a.focus(ix, iy);
    col_add(a, *ir, -eq * cdiff * p.volume, p.contains);
    a.dirty(ix, iy);
  }
  a.mark(2);
  Cascade<0, A>::run(a, nx, ny, 0);                                 // :113
  a.mark(6);
  p.sediment /= (1.0 - evaprate);                                   // :116-119
  if (p.sediment > 1.0) p.sediment = 1.0;
  p.volume *= (1.0 - evaprate);
  return (p.volume > 0.01) ? SM_ALIVE : SM_EXIT_EVAP;
}

// one move() && interact().  `a` must cover plus(ipos) and the 3x3 around the new position.
template <class A> SM_HD int water_step(A& a, WaterP& p) {
  WaterMid m;
  const int r = water_move(a, p, m);
  if (r != SM_ALIVE) return r;
  return water_interact(a, p, m);
}

// ------------------------------------------------------------------------------------------------
// WindParticle  (wind.h)
// ------------------------------------------------------------------------------------------------
// What WindParticle::move hands to interact() of the same step.
struct WindMid {
  float suspension;      // param.suspension of the surface at ipos
  uint32_t transports;   // param.transports
  int ix, iy;
};

// WindParticle::move, wind.h:54-92
template <class A> SM_HD int wind_move(A& a, WindP& p, WindMid& m) {
  const int dimx = a.dimx(), dimy = a.dimy();
  const int SCALE = a.scale();
  if (a.soil(p.contains).suspension == 0.0) return SM_EXIT_OOB;     // :56-57
  const int ix = (int)roundf(p.px), iy = (int)roundf(p.py);         // :60
  a.begin(ix, iy);
  sm_f3 n = map_normal(a, ix, iy);                                  // :61
  Sec32* ir = a.rec(ix, iy);
  const SoilDev param = a.soil(rec_surface(*ir));                   // :62-63
  m.suspension = param.suspension; m.transports = param.transports; m.ix = ix; m.iy = iy;
  a.wind_frequency_touch(iy * dimx + ix);                           // :64, 49-52
  double sheight = rec_height(*ir) * (float)SCALE / 80.0f;          // :67
  if (p.height < sheight) p.height = sheight;                       // :68-70
  if (p.height > sheight) {                                         // :73-74
    p.sy = (float)(p.sy - 0.25);
  } else {                                                          // :76 mix(speed, cross(cross(speed,n),n), 0.8)
    sm_f3 s{p.sx, p.sy, p.sz};
    sm_f3 v = f3_cross(f3_cross(s, n), n);
    const double w = 0.8;
    p.sx = (float)((double)s.x * (1.0 - w) + (double)v.x * w);
    p.sy = (float)((double)s.y * (1.0 - w) + (double)v.y * w);
    p.sz = (float)((double)s.z * (1.0 - w) + (double)v.z * w);
  }
  {                                                                 // :78 mix(speed, pspeed, 0.2)
    const double w = 0.2;
    p.sx = (float)((double)p.sx * (1.0 - w) + (double)(-2.0f) * w);
    p.sy = (float)((double)p.sy * (1.0 - w) + (double)(0.0f) * w);
    p.sz = (float)((double)p.sz * (1.0 - w) + (double)(1.0f) * w);
  }
  p.px += p.sx;                                                     // :79
  p.py += p.sz;
  p.height += p.sy;                                                 // :80
  if (!(p.px >= 0.0f && p.py >= 0.0f) ||                            // :83-85
      !((int)p.px < dimx - 1 && (int)p.py < dimy - 1))
    return SM_EXIT_OOB;
  if (sqrtf(p.sx * p.sx + p.sy * p.sy + p.sz * p.sz) < 0.01)        // :87-88
    return SM_EXIT_OOB;
  return SM_ALIVE;
}

// WindParticle::interact, wind.h:94-136 (always returns true upstream)
template <class A> SM_HD int wind_interact(A& a, WindP& p, const WindMid& m) {
  const int SCALE = a.scale();
  const int ix = m.ix, iy = m.iy;
  Sec32* ir = a.rec(ix, iy);
  const int nx = (int)roundf(p.px), ny = (int)roundf(p.py);         // :99
  a.target(nx, ny);
  int ncascade = 0;
  if (p.height <= map_height_bilinear(a, p.px, p.py) * (float)SCALE / 80.0f) {   // :102
    if (m.transports == p.contains) {                               // :105
      float len = sqrtf(p.sx * p.sx + p.sy * p.sy + p.sz * p.sz);
      double force = len * (map_height(a, nx, ny) - p.height) * (float)SCALE / 80.0f *
                     (1.0f - p.sediment);                           // :107
      a.focus(ix, iy);
      double diff = col_remove(a, *ir, m.suspension * force);       // :109
      a.dirty(ix, iy);
      p.sediment += (m.suspension * force - diff);                  // :110
      ncascade = 1;                                                 // :112 cascade(ipos, 1)
    }
  } else if (m.suspension > 0.0) {                                  // :119
    const float sc = a.soil(p.contains).suspension;
    p.sediment -= sc * p.sediment;                                  // :121
    a.focus(nx, ny);
    col_add(a, *a.rec(nx, ny), 0.5f * sc * p.sediment, p.contains); // :123
    a.dirty(nx, ny);
    a.focus(ix, iy);
    col_add(a, *ir, 0.5f * sc * p.sediment, p.contains);            // :124
    a.dirty(ix, iy);
    ncascade = 2;                                                   // :126,129 cascade(ipos,1); cascade(npos,1)
  }
  a.mark(2);
  SM_UNROLL1
  for (int q = 0; q < ncascade; q++)                                // one call site for both
    Cascade<1, A>::run(a, q == 0 ? ix : nx, q == 0 ? iy : ny, 1);
  return SM_ALIVE;
}

template <class A> SM_HD int wind_step(A& a, WindP& p) {
  WindMid m;
  const int r = wind_move(a, p, m);
  if (r != SM_ALIVE) return r;
  return wind_interact(a, p, m);
}
