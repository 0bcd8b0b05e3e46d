// sm_snap.cuh -- the snapshot format (version 1) and its per-cell logic: count, pack, validate, unpack.
//
// A snapshot is one little-endian byte image of the columns of an x-range [x0, x1) of the map and of the three
// frequency arrays over the same columns (DESIGN.md section 10):
//   header   128 B   SnapHeader
//   offsets          u64[ncells + 1], cell order (x - x0)*dimy + y, offsets[0] = 0 (the CSR of sm_download_columns)
//   records          at records_at (32-B aligned): nsections x SnapRec, bottom -> top within each column
//   frequency        f32 water_frequency, water_track, wind_frequency, each [dimy][x1 - x0]
// The image is canonical: it holds values only, never pool slot numbers, so equal columns give equal bytes whatever
// the pool's history and whatever the sharding.  Everything below is SM_HD so that the host compiles it as a test tool
// (tests/snapshot/host_snap.cpp); the kernels in sm_engine.cu call it one thread per cell.
#pragma once
#include "sm_core.cuh"

#define SM_SNAP_VERSION 1u
#define SM_SNAP_HEADER 128u

struct SnapHeader {
  char magic[8];                  // "SMSNAP\0\0"
  uint32_t version, header_bytes;
  int32_t dimx, dimy, x0, x1, nsoils, reserved;
  uint64_t ncells, nsections, offsets_at, records_at, freq_at, total_bytes;
  uint64_t checksum;              // sm_checksum of the covered columns (global cell indices)
  unsigned char pad[SM_SNAP_HEADER - 96];
};
static_assert(sizeof(SnapHeader) == SM_SNAP_HEADER, "snapshot header is 128 bytes");

struct SnapRec {                  // one section; floor is stored verbatim
  double size, floor, saturation;
  uint32_t type, reserved;
};
static_assert(sizeof(SnapRec) == 32, "snapshot record is 32 bytes");

// where each part lies for a snapshot of ncells cells and nsections sections
SM_HD void snap_layout(SnapHeader& h, int dimx, int dimy, int x0, int x1, int nsoils, uint64_t nsections) {
  for (unsigned i = 0; i < SM_SNAP_HEADER; i++) ((unsigned char*)&h)[i] = 0;
  const char m[8] = {'S', 'M', 'S', 'N', 'A', 'P', 0, 0};
  for (int i = 0; i < 8; i++) h.magic[i] = m[i];
  h.version = SM_SNAP_VERSION; h.header_bytes = SM_SNAP_HEADER;
  h.dimx = dimx; h.dimy = dimy; h.x0 = x0; h.x1 = x1; h.nsoils = nsoils;
  h.ncells = (uint64_t)(x1 - x0) * (uint64_t)dimy;
  h.nsections = nsections;
  h.offsets_at = SM_SNAP_HEADER;
  h.records_at = (h.offsets_at + 8 * (h.ncells + 1) + 31) / 32 * 32;
  h.freq_at = h.records_at + 32 * nsections;
  h.total_bytes = h.freq_at + 12 * h.ncells;
}

// The header checks of a restore (everything except the offsets and the records, which k_snap_validate reads):
// nullptr when the header is well-formed, matches the map and fits in `bytes`; otherwise what is wrong.
SM_HD const char* snap_check_header(const SnapHeader& h, int64_t bytes, int dimx, int dimy, int nsoils) {
  const char m[8] = {'S', 'M', 'S', 'N', 'A', 'P', 0, 0};
  if (bytes < (int64_t)SM_SNAP_HEADER) return "snapshot: shorter than its header";
  for (int i = 0; i < 8; i++) if (h.magic[i] != m[i]) return "snapshot: bad magic";
  if (h.version != SM_SNAP_VERSION || h.header_bytes != SM_SNAP_HEADER) return "snapshot: unsupported version";
  if (h.dimx != dimx || h.dimy != dimy) return "snapshot: map dimensions differ from the context's";
  if (nsoils < 1) return "snapshot: soil table not set";
  if (h.nsoils != nsoils) return "snapshot: number of soils differs from the context's soil table";
  if (h.x0 < 0 || h.x1 > dimx || h.x0 >= h.x1) return "snapshot: bad x-range";
  SnapHeader want;
  snap_layout(want, dimx, dimy, h.x0, h.x1, nsoils, h.nsections);
  if (h.nsections > (uint64_t)1 << 40 || h.ncells != want.ncells || h.offsets_at != want.offsets_at ||
      h.records_at != want.records_at || h.freq_at != want.freq_at || h.total_bytes != want.total_bytes)
    return "snapshot: inconsistent layout";
  if ((uint64_t)bytes < h.total_bytes) return "snapshot: truncated";
  return nullptr;
}

// The offsets a restore reads on the host before the slice [lo, hi] of cells it takes is validated on the device:
// off[0], off[ncells], off[lo], off[hi].  false unless the offsets run from 0 to nsections and the slice lies inside.
SM_HD bool snap_check_ends(uint64_t first, uint64_t last, uint64_t lo, uint64_t hi, uint64_t nsections) {
  return first == 0 && last == nsections && lo <= hi && hi <= nsections;
}

// ---- per cell --------------------------------------------------------------------------------------------------
// sections of one column, following `below` through the pool
SM_HD uint64_t snap_count_cell(const Sec32& top, const Sec32* pool) {
  if (top.type == SM_EMPTY) return 0;
  uint64_t n = 1;
  for (uint32_t b = top.below; b != SM_NIL; b = pool[b].below) n++;
  return n;
}
SM_HD void snap_rec_of(SnapRec& o, const Sec32& r) {
  o.size = r.size; o.floor = r.floor; o.saturation = r.saturation; o.type = r.type; o.reserved = 0;
}
// the column's n sections, bottom -> top, into out[0, n)
SM_HD void snap_pack_cell(const Sec32& top, const Sec32* pool, uint64_t n, SnapRec* out) {
  if (!n) return;
  Sec32 r = top;
  for (uint64_t i = n; i-- > 0;) {
    snap_rec_of(out[i], r);
    if (r.below == SM_NIL) break;
    r = pool[r.below];
  }
}
// Cell c of the slice off[0, cells] of a snapshot's offsets, whose records start at rec (the record of index off[0]).
// false: the cell's offsets run backwards or leave the slice, or one of its records names a soil the table lacks.
// Reads the slice only, never a record outside [off[0], off[cells]).
SM_HD bool snap_valid_cell(const uint64_t* off, const SnapRec* rec, uint64_t cells, uint64_t c, int nsoils) {
  const uint64_t rec0 = off[0], end = off[cells];
  if (off[c + 1] < off[c] || off[c] < rec0 || off[c + 1] > end) return false;
  for (uint64_t k = off[c]; k < off[c + 1]; k++)
    if (rec[k - rec0].type >= (uint32_t)nsoils) return false;
  return true;
}
// the column's buried sections, which need pool slots
SM_HD uint64_t snap_buried(const uint64_t* off, uint64_t c) {
  const uint64_t n = off[c + 1] - off[c];
  return n ? n - 1 : 0;
}
// One column of a validated slice (as snap_valid_cell): the top record into `top`, the buried ones into the consecutive
// pool slots [base, base + n - 1), bottom first, each linked to the one underneath.
SM_HD void snap_unpack_cell(const uint64_t* off, const SnapRec* rec, uint64_t c, uint32_t base, Sec32& top,
                            Sec32* pool) {
  const uint64_t lo = off[c] - off[0], n = off[c + 1] - off[c];
  if (!n) { rec_set_empty(top); return; }
  for (uint64_t i = 0; i < n; i++) {
    const SnapRec& s = rec[lo + i];
    Sec32 r;
    r.size = s.size; r.floor = s.floor; r.saturation = s.saturation; r.type = s.type;
    r.below = i ? base + (uint32_t)(i - 1) : SM_NIL;
    if (i + 1 < n) pool[base + i] = r;
    else top = r;
  }
}
