// sm_strata.cuh -- whole-map views of what lies under the surface (sm_composition, sm_voxelize, DESIGN.md section 13):
// the per-cell logic.
//
// Both views walk one column's chain top -> bottom (the top record, then `below` through the pool) and change nothing.
// A composition cell sums, per requested soil type, the overlap of every section with a height window (or that overlap
// times the section's pore water); a voxel cell gives, at a ladder of sample heights z_k = z0 + k*dz, the type of the
// first section met top -> bottom that contains z_k.  Every section of the chain is visited: a restored snapshot keeps
// `floor` verbatim, so floors need not be running sums and a walk may not stop early.  Everything below is SM_HD so that
// the host compiles it as a test tool (tests/strata/host_strata.cpp); the kernels in sm_engine.cu call it one thread per
// cell.
#pragma once
#include "../../include/soilmachine_b200.h"     // SM_MAX_SOILS, SM_COMP_*, SM_VOXEL_NONE, SM_VOXEL_MAX_NZ
#include "sm_core.cuh"

// read-only accessor over a pool array
struct StrataPool {
  const Sec32* pool;
  SM_HD Sec32 pool_load(uint32_t i) const { return pool[i]; }
};

// One composition cell.  slot[t] = the output slot of soil type t (-1: not requested), for t < SM_MAX_SOILS; porosity[t]
// = soils[t].porosity.  Writes out[i * stride] for every slot i < ntypes; returns the sections read.
template <class A>
SM_HD uint32_t strata_compose_cell(const A& a, const Sec32& top, double lo, double hi, int flags, const signed char* slot,
                                   int ntypes, const float* porosity, double* out, size_t stride) {
  SM_UNROLL1
  for (int i = 0; i < ntypes; i++) out[(size_t)i * stride] = 0.0;
  if (top.type == SM_EMPTY) return 0;
  double wa = lo, wb = hi;
  if (flags & SM_COMP_BELOW_SURFACE) {
    const double H = rec_height(top);
    wa = H - hi;
    wb = H - lo;
  }
  const bool pore = (flags & SM_COMP_PORE_WATER) != 0;
  uint32_t n = 0;
  Sec32 s = top;
  SM_UNROLL1
  for (;;) {
    n++;
    const double t = s.floor + s.size;
    const double ov = (t < wb ? t : wb) - (s.floor > wa ? s.floor : wa);
    const int i = s.type < SM_MAX_SOILS ? (int)slot[s.type] : -1;
    if (ov > 0 && i >= 0) out[(size_t)i * stride] += pore ? ov * s.saturation * (double)porosity[s.type] : ov;
    if (s.below == SM_NIL) break;
    s = a.pool_load(s.below);
  }
  return n;
}

// z_k = z0 + (double)k * dz is non-decreasing in k (both roundings are monotone), so {k : v <= z_k} is [first, nz).
// The smallest k in [0, nz] with v <= z_k (nz when there is none): the ceiling of the quotient (v - z0) / dz, taken as a
// product with rdz = 1.0 / dz (computed once per call: a device division per section would cost a slow-path call), then
// corrected with the exact comparison in both directions, so the answer does not depend on the estimate.
SM_HD uint32_t strata_first_sample(double z0, double dz, double rdz, uint32_t nz, double v) {
  const double t = (v - z0) * rdz;
  uint32_t k;
  if (!(t > 0.0)) k = 0;                       // NaN included
  else if (t >= (double)nz) k = nz;
  else k = (uint32_t)ceil(t);
  SM_UNROLL1
  while (k > 0 && z0 + (double)(k - 1) * dz >= v) k--;
  SM_UNROLL1
  while (k < nz && z0 + (double)k * dz < v) k++;
  return k;
}

// The samples section s contains: [*k0, *k1) = {k : s.floor <= z_k < s.floor + s.size}
SM_HD void strata_sample_range(double z0, double dz, double rdz, uint32_t nz, const Sec32& s, uint32_t* k0,
                               uint32_t* k1) {
  *k0 = strata_first_sample(z0, dz, rdz, nz, s.floor);
  *k1 = strata_first_sample(z0, dz, rdz, nz, s.floor + s.size);
  if (*k1 < *k0) *k1 = *k0;
}

// One voxel cell: out[k * stride] for k < nz (rdz = 1.0 / dz).  One walk; a sample is written by the first section met
// that contains it.  Ranges disjoint from every range written before (a column whose floors are running sums) are stored without looking;
// only a range that meets an earlier one reads its samples back.  Returns the sections read.
template <class A>
SM_HD uint32_t strata_voxel_cell(const A& a, const Sec32& top, double z0, double dz, double rdz, uint32_t nz,
                                 unsigned char* out, size_t stride) {
  SM_UNROLL1
  for (uint32_t k = 0; k < nz; k++) out[(size_t)k * stride] = SM_VOXEL_NONE;
  if (top.type == SM_EMPTY) return 0;
  uint32_t n = 0, hlo = nz, hhi = 0;           // [hlo, hhi): hull of the samples written so far
  Sec32 s = top;
  SM_UNROLL1
  for (;;) {
    n++;
    uint32_t k0, k1;
    strata_sample_range(z0, dz, rdz, nz, s, &k0, &k1);
    if (k0 < k1) {
      const unsigned char t = (unsigned char)s.type;
      if (k1 <= hlo || k0 >= hhi) {
        SM_UNROLL1
        for (uint32_t k = k0; k < k1; k++) out[(size_t)k * stride] = t;
      } else {
        SM_UNROLL1
        for (uint32_t k = k0; k < k1; k++)
          if (out[(size_t)k * stride] == SM_VOXEL_NONE) out[(size_t)k * stride] = t;
      }
      hlo = k0 < hlo ? k0 : hlo;
      hhi = k1 > hhi ? k1 : hhi;
    }
    if (s.below == SM_NIL) break;
    s = a.pool_load(s.below);
  }
  return n;
}
