// sm_layer.cuh -- one layer raster applied to the map (sm_apply_layer, DESIGN.md section 11): the per-cell logic.
//
// A raster holds one f64 per cell.  delta > 0 deposits that much of one soil type on the cell, exactly as
// Layermap::add(pos, new sec(delta, type)) (layermap.h:230-307, col_add); delta < 0 strips -delta of height with the
// reference's own Layermap::remove (layermap.h:310-339, col_remove) called until that much is gone or the column is
// empty; delta == +-0.0 leaves the cell alone.  Each cell touches its own column only, and pool slot numbers never
// influence values, so the result is the same in any cell order.  Everything below is SM_HD so that the host compiles
// it as a test tool (tests/layer/host_layer.cpp); the kernels in sm_engine.cu call it one thread per cell.
#pragma once
#include "sm_core.cuh"

// A raster entry and the soil type are accepted when the entry is finite and the type names a soil of the table.
SM_HD bool layer_input_ok(double delta, int32_t type, int nsoils) {
  return isfinite(delta) && type >= 0 && type < nsoils;
}

// The pool slots layer_apply_cell allocates on the column whose top record is `top`, provided every allocation
// succeeds: col_add's branches, counted.  0 for an empty column or an equal-type top, 1 for an ordinary push; on an
// Air top the water comes off, the deposit goes onto the record underneath (a push unless that record is missing or of
// the deposited type), and the water goes back on as a push unless its size is <= 0.  A strip allocates nothing.
template <class A> SM_HD uint32_t layer_pushes(A& a, const Sec32& top, double delta, uint32_t type) {
  if (delta <= 0) return 0;                                     // col_add's `size <= 0` guard; strips and zeros
  if (top.type == SM_EMPTY || top.type == type) return 0;
  if (top.type != SM_AIR) return 1;
  const uint32_t under = top.below == SM_NIL ? SM_EMPTY : a.pool_load(top.below).type;
  return ((under == SM_EMPTY || under == type) ? 0u : 1u) + (top.size <= 0 ? 0u : 1u);
}

// Strip h of height: the reference's remove() until h is used up or the column is empty.  A zero-size top is popped
// without using up height; any other call leaves a partial top (returns 0) or pops the top and returns the rest.
// Returns the height that could not be taken (non-zero only where the column ran empty).
template <class A> SM_HD double layer_strip(A& a, Sec32& r, double h) {
  double left = h;
  SM_UNROLL1
  while (left > 0 && r.type != SM_EMPTY) {
    const bool empty_top = r.size <= 0.0;
    const double rest = col_remove(a, r, left);
    if (!empty_top) left = rest;
  }
  return left;
}

// One cell of the raster on its top record `r`; returns the cell's leftover.
template <class A> SM_HD double layer_apply_cell(A& a, Sec32& r, double delta, uint32_t type) {
  if (delta > 0) {
    col_add(a, r, delta, type);
    return 0.0;
  }
  if (delta < 0) return layer_strip(a, r, -delta);
  return 0.0;
}
