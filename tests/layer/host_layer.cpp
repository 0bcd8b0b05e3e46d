// tests/layer/host_layer.cpp -- the layer raster's per-cell logic (soilmachine_b200/csrc/sm_layer.cuh) compiled for the
// host, driven the way k_layer_check and k_layer_apply drive it.  TEST TOOL ONLY.
//
// hlayer_run   the check pass over every cell (input, push count, pool preflight), then, when it accepts, the apply
//              pass in a given cell order on a top / pool image with the device's pool discipline: frees go to a list
//              the call never reuses (ring 0), allocations pop `ring1` first, then the bump counter up to pool_cap
#include <stdint.h>
#include <vector>
#include "../../soilmachine_b200/csrc/sm_layer.cuh"

namespace {
struct HostPool {
  Sec32* pool;
  int64_t cap, bump;
  const uint32_t* ring1;
  int64_t nring1, head = 0;
  int64_t allocs = 0;                  // pool_alloc calls of the current cell
  std::vector<uint32_t> freed;         // ring 0
  Sec32 pool_load(uint32_t i) { return pool[i]; }
  void pool_store(uint32_t i, const Sec32& r) { pool[i] = r; }
  uint32_t pool_alloc() {
    allocs++;
    if (head < nring1) return ring1[head++];
    if (bump < cap) return (uint32_t)bump++;
    return SM_NIL;
  }
  void pool_free(uint32_t i) { freed.push_back(i); }
};
}  // namespace

extern "C" {
// 0: applied; 1: refused, an entry is not finite or the type is out of range; 3: refused, the raster pushes more than
// nring1 + pool_cap - bump sections.  Refused calls write nothing but stats.  pushes[c]: the push-count predicate of cell
// c; allocs[c]: the pool_alloc calls cell c made (-1 where it did not run).  stats: cells, pushed, free_slots, emptied.
int hlayer_run(int64_t ncells, Sec32* top, Sec32* pool, int64_t pool_cap, int64_t* bump, const uint32_t* ring1,
               int64_t nring1, const double* delta, int32_t type, int32_t nsoils, const int64_t* order,
               double* leftover, int64_t* pushes, int64_t* allocs, int64_t* stats) {
  HostPool a{pool, pool_cap, *bump, ring1, nring1};
  int64_t pushed = 0, touched = 0;
  bool bad = false;
  for (int64_t c = 0; c < ncells; c++) {
    pushes[c] = 0;
    allocs[c] = -1;
    if (!layer_input_ok(delta[c], type, nsoils)) { bad = true; continue; }
    touched += delta[c] != 0.0;
    if (delta[c] > 0) pushes[c] = layer_pushes(a, top[c], delta[c], (uint32_t)type);
    pushed += pushes[c];
  }
  stats[0] = touched; stats[1] = pushed; stats[2] = nring1 + pool_cap - *bump; stats[3] = 0;
  if (bad) return 1;
  if (pushed > stats[2]) return 3;
  for (int64_t k = 0; k < ncells; k++) {
    const int64_t c = order[k];
    a.allocs = 0;
    double left = 0.0;
    if (delta[c] != 0.0) left = layer_apply_cell(a, top[c], delta[c], (uint32_t)type);
    allocs[c] = a.allocs;
    leftover[c] = left;
    stats[3] += left > 0;
  }
  *bump = a.bump;
  return 0;
}
}
