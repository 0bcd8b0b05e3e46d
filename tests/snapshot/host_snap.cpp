// tests/snapshot/host_snap.cpp -- the snapshot's per-cell logic (soilmachine_b200/csrc/sm_snap.cuh) compiled for the
// host, driven the way the kernels and the restore's host checks drive it.  TEST TOOL ONLY.
//
// hsnap_pack         the count pass, the exclusive scan and the pack pass of a save over a top / pool image
// hsnap_validate     a restore's checks, in its order: header, offset ends, every cell of the slice
// hsnap_unpack       a restore's buried-count scan and unpack of the slice of a snapshot one strip takes
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../soilmachine_b200/csrc/sm_snap.cuh"

extern "C" {
// off[ncells + 1] and (rec != NULL) the records of the cells' columns.  broken = 1: a faulty pack that never writes a
// column's deepest buried section (its record stays zero) - the negative control of the tests.
void hsnap_pack(int64_t ncells, const Sec32* top, const Sec32* pool, uint64_t* off, SnapRec* rec, int broken) {
  uint64_t n = 0;
  for (int64_t c = 0; c < ncells; c++) {
    off[c] = n;
    n += snap_count_cell(top[c], pool);
  }
  off[ncells] = n;
  if (!rec) return;
  for (int64_t c = 0; c < ncells; c++) {
    const uint64_t k = off[c + 1] - off[c];
    if (!broken || k < 2) { snap_pack_cell(top[c], pool, k, rec + off[c]); continue; }
    Sec32 r = top[c];
    for (uint64_t i = k; i-- > 1;) {       // stops above the deepest section
      snap_rec_of(rec[off[c] + i], r);
      r = pool[r.below];
    }
  }
}

// 0: the slice [x0, x1) of the snapshot passes every check of a restore; 1: the header, 2: the offsets' ends, 3: a cell
int hsnap_validate(const unsigned char* buf, int64_t bytes, int dimx, int dimy, int nsoils, int x0, int x1) {
  SnapHeader H;
  if (bytes < (int64_t)sizeof(H)) return 1;
  memcpy(&H, buf, sizeof(H));
  if (snap_check_header(H, bytes, dimx, dimy, nsoils)) return 1;
  const uint64_t* off = (const uint64_t*)(buf + H.offsets_at);
  const uint64_t lo = (uint64_t)(x0 - H.x0) * dimy, cells = (uint64_t)(x1 - x0) * dimy;
  if (!snap_check_ends(off[0], off[H.ncells], off[lo], off[lo + cells], H.nsections)) return 2;
  const SnapRec* rec = (const SnapRec*)(buf + H.records_at) + off[lo];
  for (uint64_t c = 0; c < cells; c++)
    if (!snap_valid_cell(off + lo, rec, cells, c, nsoils)) return 3;
  return 0;
}

// the strip [x0, x1) of a (validated) snapshot into top[(x1 - x0)*dimy] and pool[*need]; returns *need, the pool slots
// used.  pool must hold the snapshot's nsections records.
void hsnap_unpack(const unsigned char* buf, int x0, int x1, Sec32* top, Sec32* pool, int64_t* need) {
  SnapHeader H;
  memcpy(&H, buf, sizeof(H));
  const uint64_t* off = (const uint64_t*)(buf + H.offsets_at);
  const uint64_t lo = (uint64_t)(x0 - H.x0) * H.dimy, cells = (uint64_t)(x1 - x0) * H.dimy;
  const SnapRec* rec = (const SnapRec*)(buf + H.records_at) + off[lo];
  std::vector<uint64_t> base(cells + 1);
  uint64_t b = 0;
  for (uint64_t c = 0; c < cells; c++) { base[c] = b; b += snap_buried(off + lo, c); }
  for (uint64_t c = 0; c < cells; c++) snap_unpack_cell(off + lo, rec, c, (uint32_t)base[c], top[c], pool);
  *need = (int64_t)b;
}
}
