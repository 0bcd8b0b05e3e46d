// sm_drain.cuh -- how the map drains (sm_drainage, DESIGN.md section 14): the per-cell logic.
//
// The view reads one height H per cell (the top of the column, or with SM_DRAIN_GROUND the top of the first section
// that is not Air, walking the chain as sm_strata.cuh does), fills it to the spill height W (the least, over all
// 8-connected paths to a border cell, of the highest H on the path), measures the distance of every flat cell to the
// edge of its flat, and picks one receiver per cell: the steepest lower neighbour, else the next cell towards the edge
// of the flat.  Everything below is SM_HD so that the host compiles it as a test tool (tests/drainage/host_drain.cpp);
// the kernels in sm_engine.cu apply it to tiles of the whole-map rasters.
//
// A 3x3 window is passed as the centre value and the eight neighbours in the order n[k] of the reference's
// water.h:155-164: (dx, dy) = (-1,-1), (-1,0), (-1,1), (0,-1), (0,1), (1,-1), (1,0), (1,1).
#pragma once
#include "../../include/soilmachine_b200.h"     // SM_DRAIN_GROUND
#include "sm_core.cuh"

#define SM_DRAIN_NOT_FLAT 0           // dist of a drained or border cell
#define SM_DRAIN_FAR 0x7fffffff       // dist of a flat cell not reached yet
// sqrt(2.0), correctly rounded
#define SM_DRAIN_SQRT2 1.4142135623730951
// the 3x3 loops are unrolled on the device, so that the windows stay in registers
#ifdef __CUDACC__
#define SM_DRAIN_UNROLL _Pragma("unroll")
#else
#define SM_DRAIN_UNROLL
#endif

SM_HD int drain_dx(int k) { return k < 3 ? -1 : (k < 5 ? 0 : 1); }
SM_HD int drain_dy(int k) { return (k == 0 || k == 3 || k == 5) ? -1 : ((k == 1 || k == 6) ? 0 : 1); }
SM_HD bool drain_diagonal(int k) { return k == 0 || k == 2 || k == 5 || k == 7; }

// H of one column.  ground = false: top.floor + top.size, 0.0 for an empty column (sm_download_height).  ground = true:
// floor + size of the first section met top -> bottom whose type is not Air (0), 0.0 if there is none.
template <class A>
SM_HD double drain_column_height(const A& a, const Sec32& top, bool ground) {
  if (top.type == SM_EMPTY) return 0.0;
  if (!ground) return top.floor + top.size;
  Sec32 s = top;
  SM_UNROLL1
  for (;;) {
    if (s.type != 0) return s.floor + s.size;
    if (s.below == SM_NIL) return 0.0;
    s = a.pool_load(s.below);
  }
}

// One relaxation of the fill at an interior cell: max(h, min over the eight neighbours' current values).  Applied to
// upper bounds of W it gives an upper bound of W no larger than the neighbours allow; at the fixed point it is W.
SM_HD double drain_fill_value(double h, const double* wn) {
  double m = wn[0];
  SM_DRAIN_UNROLL
  for (int k = 1; k < 8; k++) m = wn[k] < m ? wn[k] : m;
  return h > m ? h : m;
}

// A cell with a neighbour of lower spill height drains; an interior cell that does not lies on a flat.
SM_HD bool drain_drained(double wc, const double* wn) {
  bool d = false;
  SM_DRAIN_UNROLL
  for (int k = 0; k < 8; k++) d |= wn[k] < wc;
  return d;
}

// One relaxation of the flat distances at a flat cell: the least of its own value and dist(n) + 1 over the neighbours
// of equal W.  Drained and border cells hold SM_DRAIN_NOT_FLAT and are never relaxed.
SM_HD int32_t drain_dist_value(double wc, int32_t dc, const double* wn, const int32_t* dn) {
  int32_t m = dc;
  SM_DRAIN_UNROLL
  for (int k = 0; k < 8; k++)
    if (wn[k] == wc && dn[k] != SM_DRAIN_FAR && dn[k] + 1 < m) m = dn[k] + 1;
  return m;
}

// The receiver k of an interior cell with spill height wc and flat distance dc.  Drained: the largest
// (wc - wn[k]) / d, d = 1.0 or sqrt(2.0), ties to the lower k.  Flat: the lowest k with wn[k] == wc and
// dn[k] == dc - 1.  -1 when neither exists (not at the fixed point).
SM_HD int drain_receiver(double wc, int32_t dc, const double* wn, const int32_t* dn) {
  int best = -1;
  double bs = 0.0;
  SM_DRAIN_UNROLL
  for (int k = 0; k < 8; k++) {
    if (!(wn[k] < wc)) continue;
    const double s = (wc - wn[k]) / (drain_diagonal(k) ? SM_DRAIN_SQRT2 : 1.0);
    if (best < 0 || s > bs) { best = k; bs = s; }
  }
  if (best >= 0) return best;
  SM_DRAIN_UNROLL
  for (int k = 0; k < 8; k++)
    if (wn[k] == wc && dn[k] == dc - 1) return k;
  return -1;
}
