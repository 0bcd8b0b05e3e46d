// tests/strata/host_strata.cpp -- the strata views' per-cell logic (soilmachine_b200/csrc/sm_strata.cuh) compiled for
// the host, driven the way k_strata_compose and k_strata_voxel drive it.  TEST TOOL ONLY.
//
// hstrata_compose  every cell of a top / pool image, planar output out[i * ncells + cell]
// hstrata_voxel    the cells of a window, planar output out[k * ncells + j] for window cell j
// hstrata_range    the sample range [k0, k1) of a list of (floor, size) pairs
#include <stdint.h>
#include <string.h>
#include "../../soilmachine_b200/csrc/sm_strata.cuh"

extern "C" {
// types[0..ntypes) (distinct, < SM_MAX_SOILS), porosity[SM_MAX_SOILS].  Returns the sections read.
int64_t hstrata_compose(int64_t ncells, const Sec32* top, const Sec32* pool, double lo, double hi, int32_t flags,
                        const int32_t* types, int32_t ntypes, const float* porosity, double* out) {
  signed char slot[SM_MAX_SOILS];
  memset(slot, -1, sizeof(slot));
  for (int i = 0; i < ntypes; i++) slot[types[i]] = (signed char)i;
  const StrataPool a{pool};
  int64_t n = 0;
  for (int64_t c = 0; c < ncells; c++)
    n += strata_compose_cell(a, top[c], lo, hi, flags, slot, ntypes, porosity, out + c, (size_t)ncells);
  return n;
}
// cells[j]: the top record index of window cell j.  Returns the sections read.
int64_t hstrata_voxel(int64_t ncells, const int64_t* cells, const Sec32* top, const Sec32* pool, double z0, double dz,
                      int32_t nz, uint8_t* out) {
  const StrataPool a{pool};
  int64_t n = 0;
  for (int64_t j = 0; j < ncells; j++)
    n += strata_voxel_cell(a, top[cells[j]], z0, dz, 1.0 / dz, (uint32_t)nz, out + j, (size_t)ncells);
  return n;
}
void hstrata_range(int64_t n, const double* floor_, const double* size, double z0, double dz, int32_t nz, uint32_t* k0,
                   uint32_t* k1) {
  for (int64_t i = 0; i < n; i++) {
    Sec32 s = {};
    s.size = size[i];
    s.floor = floor_[i];
    strata_sample_range(z0, dz, 1.0 / dz, (uint32_t)nz, s, k0 + i, k1 + i);
  }
}
}
