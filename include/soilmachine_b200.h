/* soilmachine_b200 -- C ABI of the H100-native particle/terrain hot path.
 *
 * The reference (weigert/SoilMachine) has no plugin or FFI layer: its frame loop
 * (SoilMachine.cpp:283-329) calls WaterParticle/WindParticle::move/interact
 * (source/particle/water.h:43-121, wind.h:54-136), Particle::cascade (particle.h:24-101) and the
 * Layermap column operations (source/layermap.h:230-439) directly.  This header is the boundary a
 * binding of that loop would call instead; include/soilmachine/ holds the C++ facade that exposes
 * the reference's own class names on top of it.  Every entry point cites what it replaces.
 *
 * Conventions: plain pointers and sizes, caller-owned host buffers, context-owned device memory,
 * int status (0 = ok), sm_last_error() for the message, never throws, one caller thread per
 * context.  Cell order of every per-cell array is x*dimy + y (layermap.h:151) unless stated;
 * frequency/track arrays use y*dimx + x (water.h:53,349).
 */
#ifndef SOILMACHINE_B200_H
#define SOILMACHINE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SM_OK 0
#define SM_ERR_INVALID 1      /* bad argument */
#define SM_ERR_CUDA 2         /* CUDA runtime error (message in sm_last_error) */
#define SM_ERR_POOL 3         /* section pool exhausted: the reference prints and drops mass
                                 (layermap.h:92-95,232-234); here the drop is counted and reported */
#define SM_ERR_REACH 4        /* a particle step left its conflict box (internal invariant) */
#define SM_ERR_NOGPU 5        /* no CUDA device: there is no CPU fallback */

#define SM_MAX_SOILS 64

typedef struct sm_context sm_context;

/* Numeric mirror of SurfParam (surface.h:11-39).  Index in the table = SurfType; 0 is "Air"
 * (surface.h:41-57). */
typedef struct sm_soil {
  int32_t transports, erodes, cascades, abrades;
  float density, porosity, solubility, equrate, friction, erosionrate, maxdiff, settling,
      suspension, abrasion;
} sm_soil;

/* Numeric mirror of SurfLayer (surface.h:65-101): value = max(min, bias + scale*fbm). */
typedef struct sm_layer {
  int32_t type;
  float min, bias, scale, octaves, lacunarity, gain, frequency;
} sm_layer;

typedef struct sm_config {
  int32_t dimx, dimy;       /* SIZEX, SIZEY (SoilMachine.cpp:9-10) */
  int32_t scale;            /* SCALE (SoilMachine.cpp:11) */
  int32_t device;           /* CUDA device ordinal */
  int64_t pool_capacity;    /* buried-section pool slots (POOLSIZE, SoilMachine.cpp:16); 0 = auto: one GPU - grows
                               with sm_initialize / sm_upload_columns; sharded - 2 x strip cells + 4 Mi, FIXED at
                               creation (the peers map it), so give strip cells x (layers - 1) + headroom for
                               presets with four or more layers (SM_ERR_POOL says so otherwise) */
  int32_t max_particles;    /* largest batch a *_run call will be given; 0 = 262144 */
  int32_t flags;            /* SM_FLAG_* */
} sm_config;
#define SM_FLAG_BUDGET 1      /* keep the per-particle mass budget (sm_last_budget) and the hydrology's
                                 (sm_last_hydro_budget); a few % slower */
#define SM_FLAG_CELL_BUDGET 2 /* with SM_FLAG_BUDGET: also keep the per-cell maps of the last batch
                                 (sm_last_cell_budget); 24 B per cell */
#define SM_FLAG_HYDRO_CELL_BUDGET 4 /* with SM_FLAG_BUDGET: also keep the per-cell maps of the last sm_water_flood /
                                       sm_seep call (sm_last_hydro_cell_budget); 32 B per cell; unsharded only */

/* Per-call counters (all accumulated over the call). */
typedef struct sm_stats {
  int64_t steps;       /* particle-steps: move() true and interact() ran */
  int64_t sweeps;      /* lockstep sweeps executed */
  int64_t exit_oob;    /* water: left the map (water.h:65-69) | wind: move() false (wind.h:56,83-88) */
  int64_t exit_evap;   /* water: volume <= minvol (water.h:119) */
  int64_t exit_stall;  /* water: no motion (water.h:56-57), the reference's flood candidates */
  int64_t pool_drops;  /* sections dropped because the pool was exhausted */
  int64_t alive;       /* particles still alive when the call returned (max_sweeps reached) */
  double device_ms;    /* CUDA-event time of the sweep kernel(s) of this call */
} sm_stats;

/* ---- lifetime ------------------------------------------------------------------------------ */
int sm_create(const sm_config* cfg, sm_context** out);
void sm_destroy(sm_context* ctx);
const char* sm_last_error(const sm_context* ctx);   /* ctx may be NULL: last create error */
int sm_sync(sm_context* ctx);

/* ---- sharded maps (one context per rank; ranks = GPUs, or contexts sharing one GPU) ------------------- */
/* The map is cut into nranks x-strips; rank q owns columns [x0, x1) (sm_shard_range) and executes the
 * particles whose cell lies there.  Contexts reach each other's arrays through peer pointers: every rank
 * exports a blob (sm_peer_export), the blobs are gathered (torch.distributed / MPI / same process) and
 * every rank attaches all of them (sm_peer_attach; use_ipc = 1 opens CUDA-IPC mappings of another
 * process's GPU memory, 0 takes the raw pointers of contexts living in the same process).  After that
 * sm_initialize / sm_upload_columns / downloads work on the rank's own strip (cell order
 * (x - x0)*dimy + y) and sm_*_run_device must be called on EVERY rank (the kernels meet in a cross-rank
 * barrier every sweep); results are bit-identical to the unsharded run.  share = number of contexts
 * that run their kernels concurrently on this device.
 * Read-only views of the whole map also work on a sharded context: sm_mesh_update / sm_mesh_device_ptr /
 * sm_export_* cover the rank's own strip (cell order (x - x0)*dimy + y, i.e. the slice [x0*dimy, x1*dimy) of the
 * unsharded arrays); sm_cell_query / sm_height_bilinear / sm_cell_column take global coordinates of any cell, on any
 * rank; sm_lbm_set_boundary(ctx, NULL) builds the boundary of the whole lattice from the whole map.  All of these
 * read other ranks' strips, so before calling any of them every rank's earlier work on the map (a batch,
 * sm_initialize, sm_upload_columns) must have completed: sm_sync on every rank, then a host barrier; and no rank may
 * change its strip again until the other ranks' calls have returned (a batch is safe: its ranks meet in a barrier
 * before any of them writes).  The pooling hydrology (sm_water_flood, sm_seep) runs on a sharded context from ONE rank,
 * any rank, that has been named the issuer with sm_hydro_issuer(ctx, 1) and has its peers attached: the call reads and
 * writes every strip through the peer pointers and the other ranks do not call it; same precondition, and no rank may
 * touch the map until it returns.  On a rank that is not the issuer these calls return SM_ERR_INVALID, so that a call
 * made on every rank in lockstep, as the batches are, cannot run several times over the same map.  The single-cell
 * calls that change the map return SM_ERR_INVALID on a sharded context; a group (sm_create_group) offers them.
 * sm_apply_layer works on a rank's own strip (same precondition).  sm_relax returns SM_ERR_INVALID on a sharded context:
 * each of its phases needs every rank's previous phase, a barrier across processes per phase; a group offers it.
 * sm_composition and sm_voxelize read a rank's own strip (same precondition; a voxel window must lie inside the strip):
 * each rank reads its own part and the caller joins the parts.
 * sm_drainage on a rank computes the whole map on the rank's device through the peer pointers (same precondition) and
 * writes the rank's strip; every rank that calls it repeats the whole-map work.
 * sm_peer_attach with use_ipc = 0 enables peer access to a blob's device when it differs from the context's. */
#define SM_PEER_ARRAYS 23
#define SM_PEER_SLOTS 24
typedef struct sm_peer_blob {
  uint64_t ptr[SM_PEER_SLOTS];
  unsigned char ipc[SM_PEER_SLOTS][64];
  uint64_t pool_cap;
  int32_t rank, device;
} sm_peer_blob;
int sm_create_sharded(const sm_config* cfg, int32_t nranks, int32_t rank, int32_t share, sm_context** out);
int sm_shard_range(sm_context* ctx, int32_t* x0, int32_t* x1);
int sm_peer_export(sm_context* ctx, sm_peer_blob* out);
int sm_peer_attach(sm_context* ctx, const sm_peer_blob* blobs, int32_t nblobs, int32_t use_ipc);
/* on = 1: this rank issues the pooling hydrology of the whole sharded map (sm_water_flood, sm_seep); 0: it does not
 * (the default).  At most one rank should be the issuer at a time.  No effect on an unsharded context, which always
 * issues its own. */
int sm_hydro_issuer(sm_context* ctx, int32_t on);

/* ---- groups: a sharded map behind ONE context (every rank in this process) ----------------------------- */
/* One handle over a map cut into nranks x-strips, all ranks living in THIS process.  devices[r] = CUDA ordinal of
 * rank r; devices == NULL: every rank on cfg->device.  Ranks with equal entries share that device (each is created
 * with share = ranks on that device).  nranks == 1 behaves exactly as sm_create (on devices[0] if given).
 * The group creates one sm_create_sharded context per rank, attaches them to each other without IPC (enabling peer
 * access between different devices; SM_ERR_CUDA "no peer access between devices a and b" where the hardware has none)
 * and issues the pooling hydrology from rank 0.  Every sm_* call that takes a context takes the group and acts on the
 * WHOLE map in the unsharded cell order (x*dimy + y; frequency arrays y*dimx + x): callers never see strips, and the
 * results are bit-identical to one context.  What the calls do on a group:
 *   tables, sm_initialize, sm_frequency_update, sm_lbm_create/_set_boundary/_init/_step, sm_wind_use_lbm, sm_sync:
 *     every rank (sm_lbm_step reports the slowest rank's time);
 *   sm_upload_columns, sm_set_frequency: the whole-map input is cut at the strips;
 *   downloads, sm_mesh_update (host vertices), sm_export_*, sm_last_cell_budget: each rank writes its slice of the
 *     caller's whole-map buffer; sm_checksum adds the ranks' checksums; sm_height_sum runs the one-context reduction
 *     tree over the whole map from rank 0;
 *   batches (sm_*_run, *_run_device, *_begin, *_sweeps): the spawn list goes to every rank and every rank's kernel is
 *     launched before anything waits for one (they meet in a cross-rank barrier each sweep).  For *_run_device the list
 *     lives on rank 0's device (sm_device_* act on rank 0) and is copied to the other ranks asynchronously.  Stats:
 *     steps, exits and pool_drops are summed; sweeps, alive and device_ms are the largest rank's.  sm_last_budget sums
 *     the ranks per particle, then in particle order; sm_*_state takes each particle from the rank that holds it;
 *   sm_water_flood, sm_seep, sm_last_hydro_budget, sm_cell_query, sm_height_bilinear, sm_cell_column, sm_lbm_get,
 *     sm_lbm_advect, sm_timer_*, sm_device_*: rank 0 (the first six after every rank's work has completed);
 *   sm_cell_add / _remove / _cascade / _seep / _water_cascade: one warp on rank 0 that sends every record access, pool
 *     allocation and free to the column's owner;
 *   sm_launch_count: the ranks' launches summed; sm_last_error: the failing rank's message, prefixed "rank r: ";
 *   sm_mesh_device_ptr: SM_ERR_INVALID (there is no single device array: sm_group_rank + the rank's pointer);
 *   sm_peer_export, sm_peer_attach, sm_hydro_issuer: SM_ERR_INVALID (the group manages its ranks).
 *   sm_composition, sm_voxelize: every rank computes its slice of the whole-map planes after every rank's work has
 *     completed; device output lands in rank 0's buffer; the counts are summed, device_ms is the slowest rank's.
 *   sm_drainage: rank 0 computes the whole map after every rank's work has completed, into the caller's buffers.
 * The group waits for every rank (sm_sync on each) before a call that reads or writes other ranks' strips, and only
 * when something was enqueued since the last wait.  SM_FLAG_BUDGET and SM_FLAG_CELL_BUDGET pass through to the ranks;
 * SM_FLAG_HYDRO_CELL_BUDGET with nranks > 1 is refused as by sm_create_sharded.  pool_capacity == 0 keeps the sharded
 * auto rule; a non-zero value is the WHOLE map's capacity, divided among the ranks by strip cells, rounded up.
 * sm_destroy waits for every rank, batches still in flight included, before it frees anything. */
int sm_create_group(const sm_config* cfg, int32_t nranks, const int32_t* devices, sm_context** out);
/* the rank contexts, for tests and tools (owned by the group; do not destroy) */
int sm_group_size(sm_context* ctx, int32_t* nranks);           /* 1 for a plain context */
int sm_group_rank(sm_context* ctx, int32_t rank, sm_context** rank_ctx);
/* Host only, no device needed: the strip [x0, x1) sm_create_group / sm_create_sharded give rank `rank` of nranks, and
 * the pool_capacity a group hands that rank (0 = auto).  SM_ERR_INVALID, with sm_create_sharded's message in
 * sm_last_error(NULL), when the map is too narrow for that many ranks.  Any out pointer may be NULL. */
int sm_group_layout(const sm_config* cfg, int32_t nranks, int32_t rank, int32_t* x0, int32_t* x1, int64_t* pool_capacity);

/* ---- tables: soils[] / layers (surface.h:41-57,104; io.h:7-230 fills them) -------------------- */
int sm_set_soils(sm_context* ctx, const sm_soil* soils, int32_t n);

/* loadsoil() (source/io.h:7-230): parse a `.soil` text file into the tables (host only, no device work).
 * Buffers: soils[max_soils], names[max_soils][32], colors[max_soils][4], layers[max_layers],
 * world5 = {SIZEX, SIZEY, SCALE, NWATER, NWIND}.  ctx may be NULL.  Returns SM_ERR_INVALID on a missing
 * file or a syntax error (message in sm_last_error(NULL)). */
int sm_parse_soil_file(const char* path, sm_soil* soils, char* names, float* colors, int32_t max_soils,
                       int32_t* nsoils, sm_layer* layers, int32_t max_layers, int32_t* nlayers, int32_t* world5);

/* ---- terrain -------------------------------------------------------------------------------- */
/* Layermap::initialize (layermap.h:163-216): for each layer, for each cell, add(noise section).
 * Bit-identical to the reference's FastNoiseLite OpenSimplex2/FBm path (FastNoiseLite.h:321-340,
 * 686-727,865-885,1053-1150; noise seed fixed at 1337, SEED only shifts z). */
int sm_initialize(sm_context* ctx, int32_t seed, const sm_layer* layers, int32_t nlayers);

/* Columns as bottom->top CSR; floor is recomputed as the running sum exactly as add() does
 * (layermap.h:304).  saturation may be NULL (zeros). */
int sm_upload_columns(sm_context* ctx, const int64_t* offsets, const int32_t* type,
                      const double* size, const double* saturation);
int sm_section_count(sm_context* ctx, int64_t* n);
int sm_download_columns(sm_context* ctx, int64_t capacity, int64_t* offsets, int32_t* type,
                        double* size, double* floor, double* saturation);
int sm_download_height(sm_context* ctx, double* height);     /* Layermap::height(ivec2), layermap.h:422 */
int sm_download_surface(sm_context* ctx, int32_t* surface);  /* Layermap::surface, layermap.h:417 */
int sm_height_sum(sm_context* ctx, double* sum);             /* deterministic tree sum on device */
/* Position-sensitive 64-bit checksum of every section (size, floor, saturation, type, cell, depth) of this
 * context's columns; the checksums of the strips of a sharded map add up (mod 2^64) to the checksum of the
 * whole map.  soilmachine_b200/checksum.py computes the same number from downloaded / reference columns. */
int sm_checksum(sm_context* ctx, uint64_t* checksum);

/* ---- snapshots: one canonical byte image of the columns and the frequency arrays ------------------------------------
 * The reference can only read a map from files (io.h:232: "Should be able to also WRITE to file!!").  A snapshot
 * (format version 1, little-endian, DESIGN.md section 10) covers the x-range [x0, x1) of the map:
 *   header, 128 B: magic "SMSNAP\0\0"; u32 version = 1, header_bytes = 128; i32 dimx, dimy, x0, x1, nsoils,
 *                  reserved = 0; u64 ncells = (x1 - x0)*dimy, nsections, offsets_at, records_at, freq_at, total_bytes,
 *                  checksum (sm_checksum of the covered columns, global cell indices); zeros up to 128 B
 *   offsets:       u64[ncells + 1] at offsets_at = 128, cell order (x - x0)*dimy + y: the CSR of sm_download_columns
 *   records:       at records_at (32-B aligned): nsections x {f64 size, floor, saturation; u32 type, reserved = 0},
 *                  bottom -> top within each column; floor is stored as it is, not recomputed on restore
 *   frequency:     f32 water_frequency, water_track, wind_frequency, each [dimy][x1 - x0]
 * It is canonical: contexts whose columns and frequency arrays are equal byte for byte write identical snapshots,
 * whatever their pool history and sharding.  NOT in a snapshot: the soil table and colours (the application sets
 * them; nsoils must match), the volume factor, the lattice and sm_wind_use_lbm, particle state and any open batch,
 * budgets and per-cell maps.
 * Who saves and restores what:
 *   a plain context: whole-map snapshots;
 *   a rank of a sharded map (sm_create_sharded): saves the snapshot of its own strip; restores a whole-map snapshot
 *     (its own slice of columns and frequency columns) or a strip snapshot of exactly its range.  Every rank's
 *     earlier work must have completed before any rank restores, every rank restores before the next batch, and each
 *     rank writes only its own strip.  The strips of a cut concatenate into the whole-map snapshot
 *     (soilmachine_b200/snapshot.py: join / cut);
 *   a group (sm_create_group): whole-map snapshots, every rank saving or restoring its slice.
 * So a snapshot taken on one GPU restores on any number of them, and the reverse.
 * sm_snapshot_bytes: the size sm_snapshot_save would write now (runs the count pass on the device).
 * sm_snapshot_save: dst is host memory (pageable or pinned) or, dst_on_device != 0, device memory on the context's
 *   device (rank 0's for a group), e.g. from sm_device_alloc.  SM_ERR_INVALID when capacity is too small.  A save to
 *   host memory needs the offsets array and a 32 MB staging buffer of extra device memory, never a copy of the map.
 * sm_snapshot_restore: the context's columns and frequency arrays (over the snapshot's range) become the snapshot's.
 *   Everything is validated before anything is written - the header (magic, version, dimensions, nsoils against the
 *   soil table, which must be set, the x-range, bytes), the offsets (from 0, monotone, ending at nsections) and every
 *   record (type < nsoils) - so a refused restore leaves the context as it was.  SM_ERR_POOL when a fixed
 *   pool_capacity (or a sharded rank's pool) is too small; pool_capacity == 0 on one context grows the pool as
 *   sm_upload_columns does.  A host source is copied to the device whole (offsets and records of the restored
 *   range) before it is validated.  Afterwards the pool is compact (bump = buried sections, free rings empty), the
 *   mesh is stale and no batch is open: sm_*_sweeps and sm_water_flood are refused until the next batch.
 *   Last, the restored columns' checksum is compared with the header's where the context holds all the snapshot
 *   covers (a plain context, a group, a rank restoring a strip snapshot of its range): SM_ERR_INVALID when they
 *   differ, and the map then HOLDS WHAT THE DAMAGED SNAPSHOT DESCRIBES.  A rank restoring its slice of a whole-map
 *   snapshot cannot check alone; the sum of the ranks' checksums must equal the header's (sharded.py does this). */
int sm_snapshot_bytes(sm_context* ctx, int64_t* bytes);
int sm_snapshot_save(sm_context* ctx, void* dst, int64_t capacity, int32_t dst_on_device);
int sm_snapshot_restore(sm_context* ctx, const void* src, int64_t bytes, int32_t src_on_device);

/* ---- layer rasters: deposit or strip one soil type on every cell in one call (DESIGN.md section 11) ------------------
 * delta: one f64 per cell, cell order (x - x0)*dimy + y - the whole map on a plain context and on a group, the rank's
 * strip [x0, x1) on a rank of a sharded map.  type: one soil index, 0 <= type < nsoils.  For every cell:
 *   delta > 0   exactly sm_cell_add(x, y, delta, type), i.e. Layermap::add(pos, new sec(delta, type)) (layermap.h:230-307),
 *               the Air case included: the new section goes under the standing water, the water back on top;
 *   delta < 0   strips h = -delta with the reference's own Layermap::remove (layermap.h:310-339):
 *                 left = h; while (left > 0 && dat[pos] != NULL) { empty_top = dat[pos]->size <= 0;
 *                                                                  r = remove(pos, left); if (!empty_top) left = r; }
 *               a zero-size top is popped without using up height; leftover[cell] = left, non-zero only where the
 *               column ran empty (one remove() call would stop at the first section boundary);
 *   +-0.0       the cell is untouched.
 * Each cell changes its own column only and pool slots never influence values, so the result does not depend on the
 * order the cells run in: it is the result of those calls made cell by cell.  Frequency arrays, budgets, per-cell maps
 * and hydrology maps are not touched; the mesh is left as sm_cell_add leaves it (sm_mesh_update recomputes it); an open
 * batch is treated as by sm_cell_add.
 * All or nothing: nothing is written unless every entry is finite, type is in range (SM_ERR_INVALID otherwise) and the
 * pool can serve every section the raster pushes - counted exactly first: 0 on an empty column or an equal-type top, 1
 * for an ordinary push, 0 to 2 on an Air top - from the slots it can hand out now (SM_ERR_POOL otherwise; the pool is
 * not grown).  A refused call leaves the map as it was.
 * on_device != 0: delta and leftover are device pointers on the context's device (rank 0's for a group); otherwise host
 * memory, and the raster is staged through 8 B per cell of device memory (16 B with leftover).  leftover may be NULL.
 * check_only != 0: run the check alone and fill stats (the all-or-nothing decision of a map sharded over processes:
 * every rank checks, the ranks agree, then every rank applies).  stats may be NULL; on SM_ERR_POOL it still holds the
 * counts.
 * Rank of a sharded map: allowed (its columns and their buried sections live in its own pool; no peer access), with the
 * precondition of the read-only views: every rank's earlier work has completed (sm_sync on every rank, then a host
 * barrier).  The single-cell calls stay refused there.  Group: every rank checks its slice of the raster (a device
 * raster is copied to the other ranks' devices), any refusal refuses the whole call, then every rank applies
 * concurrently; the stats are summed, device_ms is the slowest rank's. */
typedef struct sm_layer_stats {
  int64_t cells;       /* cells with delta != 0 */
  int64_t pushed;      /* sections the raster pushes (what the pool had to serve) */
  int64_t free_slots;  /* slots the pool could hand out when the call began */
  int64_t emptied;     /* columns stripped to empty (leftover > 0) */
  double device_ms;    /* CUDA-event time of the check and apply kernels */
} sm_layer_stats;
int sm_apply_layer(sm_context* ctx, const double* delta, int32_t type, double* leftover, int32_t on_device,
                   int32_t check_only, sm_layer_stats* stats);

/* ---- slope relaxation: Particle::cascade at every cell until the slopes are stable (DESIGN.md section 12) -----------
 * Runs up to max_passes passes of the reference's Particle::cascade(vec2(x, y), map, vp, transferloop)
 * (particle.h:24-101) over every cell, in this order:
 *   R = 1 + transferloop                  // footprint radius of one cascade call, re-cascades included
 *   P = 2R + 1                            // phase period: 3, 5, 7, 9 for transferloop 0..3
 *   for pass in 1..max_passes:
 *     for p in 0 .. P*P-1:                // phase p = (px, py) = (p / P, p % P)
 *       for x = px; x < dimx; x += P:     // x-major inside a phase
 *         for y = py; y < dimy; y += P:
 *           Particle::cascade(vec2(x, y), map, vp, transferloop)
 * A cascade at c reads and writes only the columns within Chebyshev distance R of c, two cells of one phase are at
 * least P = 2R + 1 apart and pool slot numbers never influence values, so the cells of a phase commute exactly: the
 * device runs each phase at once, and the result is the result of the calls above, cell by cell.
 * transferloop: 0..3 (the reference's water particles use 0, its wind particles 1); max_passes >= 1; SM_ERR_INVALID
 * otherwise, with the map unchanged.
 * A visit that cannot change anything is skipped: a cascade call is a function of the columns within R, the soil table
 * and SCALE, so a cell is visited only when a column within R of it changed since its previous visit in this call, or
 * that visit changed something (every cell is visited in the first pass).  A column changed when its top record's
 * bytes differ before and after; settling == 0 and transfers col_add ignores change nothing.  The skipped visits are
 * exact no-ops: the result is the same as visiting every cell.
 * A pass that changes no column leaves nothing to visit, so the call stops there: the map then equals the result of
 * exactly max_passes passes.  stats->passes = passes run, stats->stable = 1 when the last pass changed nothing.  The
 * passes need not converge (with SCALE > 80 and settling near 1 a transfer can overshoot and oscillate), hence the cap.
 * Frequency arrays, budgets, per-cell budget maps and hydrology maps are not touched; the mesh is left as
 * sm_cell_cascade leaves it (sm_mesh_update recomputes it); an open batch is treated as by sm_cell_add.
 * Pool: a section the pool cannot serve is dropped, as the reference does (layermap.h:92-95); the call finishes the
 * phase in which that happened, stops and returns SM_ERR_POOL with the partial stats (which cells lose the race for
 * the last slots is not pinned).  Slots freed by one phase are reused by the next.
 * Group: every rank runs each phase on the phase cells of its strip (global coordinates, the one-context order) and
 * reaches its neighbours' columns, pools and stale bits through the peer pointers; the counts are summed, device_ms
 * is the slowest rank's.  Rank of a sharded map: SM_ERR_INVALID (see sm_peer_attach above).  stats may be NULL. */
typedef struct sm_relax_stats {
  int64_t passes;      /* passes run */
  int64_t stable;      /* 1: the last pass changed no column */
  int64_t visits;      /* cascade calls made (visits that were not skipped) */
  int64_t transfers;   /* transfers that changed a column */
  int64_t pool_drops;  /* sections the pool could not serve */
  double device_ms;    /* CUDA-event time around the call's kernels */
} sm_relax_stats;
int sm_relax(sm_context* ctx, int32_t max_passes, int32_t transferloop, sm_relax_stats* stats);

/* ---- strata views: what lies under the surface, per cell, in one call (DESIGN.md section 13) ------------------------
 * Column terms are those of Sec32: the top record is top[cell], buried records are chained through `below`; "top ->
 * bottom" is chain order.  H is the value sm_download_height returns for the cell: top.floor + top.size, or 0.0 for an
 * empty column.  Both calls walk every section of the chain: a restored snapshot keeps `floor` verbatim (section 10), so
 * floors need not be running sums and no walk stops early.  The accumulation order is fixed, so the results are
 * deterministic and bit-identical on every sharding.
 *
 * sm_composition: types[0..ntypes) are distinct soil indices, 0 <= t < nsoils, 1 <= ntypes <= nsoils (type 0, Air, is
 * the standing water).  The window lo <= hi: neither may be NaN, +-inf is allowed.  flags: SM_COMP_BELOW_SURFACE
 * measures the window down from the surface; SM_COMP_PORE_WATER weights each overlap by the section's pore water.
 * Per cell c:
 *   [a, b] = BELOW_SURFACE ? [H - hi, H - lo] : [lo, hi]
 *   out[i][c] = +0.0 for every slot i
 *   for each section s of the column, top -> bottom:
 *     ov = min(s.floor + s.size, b) - max(s.floor, a)
 *     if ov > 0 and s.type == types[i]:
 *       out[i][c] += PORE_WATER ? ov * s.saturation * (double)soils[s.type].porosity    // left to right
 *                               : ov
 * The output is planar: out[i * ncells + cell], cell order x*dimy + y, or (x - x0)*dimy + y on a rank's strip, so each
 * slot is one raster and a rank's slice of a plane is contiguous.
 *
 * sm_voxelize: a window [x0, x1) x [y0, y1) in global coordinates, non-empty and inside the map (on a rank of a sharded
 * map also inside the rank's strip); sample heights z_k = z0 + (double)k * dz for k < nz, z0 finite, dz > 0 finite,
 * 1 <= nz <= SM_VOXEL_MAX_NZ (the library builds with -fmad=false: the expression means the same on host and device).
 * With W the window's cells, out[k * W + (x - x0)*(y1 - y0) + (y - y0)] is the type of the FIRST section met walking
 * top -> bottom with s.floor <= z_k < s.floor + s.size, or SM_VOXEL_NONE when no section contains z_k (above the column,
 * under its bottom, an empty column).  Plane k is a horizontal slice at z_k; a window one cell wide is a vertical strata
 * section.  "First met" decides only where sections overlap, which a restored snapshot can hold.
 *
 * Both calls are read-only: columns, pool, frequency arrays, budgets, per-cell maps, the mesh and an open batch are left
 * exactly as they were.  on_device != 0: out is a device pointer on the context's device (rank 0's for a group);
 * otherwise host memory, staged through at most 32 MB of device memory in cell-range chunks and copied into the planes
 * with 2-D copies, so the extra device memory is bounded whatever the output size.  Every argument is checked before
 * any launch; a refused call returns SM_ERR_INVALID with out untouched: a NaN bound, lo > hi, a type out of range or
 * repeated, ntypes outside 1..nsoils, unknown flag bits, no soil table (sm_composition); an empty window or one outside
 * the map or the rank's strip, z0 or dz not finite, dz <= 0, nz outside 1..SM_VOXEL_MAX_NZ (sm_voxelize); a null out.
 * Rank of a sharded map: allowed on its own strip (its columns and buried sections live in its own pool, no peer
 * access), with the precondition of the views above: every rank's earlier work has completed.  Group: the ranks are
 * settled, each computes its slice; host output goes straight into the caller's whole-map planes, device output into
 * rank 0's buffer (the kernel writes it where the rank shares rank 0's device, else through a rank-local staging buffer
 * and a peer copy).  cells, sections and bytes_out are summed, device_ms is the slowest rank's; the result equals one
 * context byte for byte.  stats may be NULL. */
#define SM_COMP_BELOW_SURFACE 1
#define SM_COMP_PORE_WATER 2
#define SM_VOXEL_NONE 255
#define SM_VOXEL_MAX_NZ 65536
typedef struct sm_view_stats {
  int64_t cells;       /* cells covered */
  int64_t sections;    /* sections read */
  int64_t bytes_out;   /* bytes written to out */
  double device_ms;    /* CUDA-event time of the kernels */
} sm_view_stats;
int sm_composition(sm_context* ctx, const int32_t* types, int32_t ntypes, double lo, double hi, int32_t flags,
                   double* out, int32_t on_device, sm_view_stats* stats);
int sm_voxelize(sm_context* ctx, int32_t x0, int32_t x1, int32_t y0, int32_t y1, double z0, double dz, int32_t nz,
                uint8_t* out, int32_t on_device, sm_view_stats* stats);

/* ---- drainage: how the map drains, in one call (DESIGN.md section 14) -----------------------------------------------
 * Definitions (cell order x*dimy + y, like every other raster):
 *   H(c), the height of cell c: without flags, what sm_download_height returns: top.floor + top.size, or 0.0 for an
 *     empty column.  With SM_DRAIN_GROUND, the ground under standing water: floor + size of the first section met
 *     walking top -> bottom whose type is not Air (type 0), or 0.0 if there is none (the chain walk of the strata views).
 *   Border cells are those with x in {0, dimx - 1} or y in {0, dimy - 1}.  They are the outlets: water leaves the map
 *     there.
 *   spill W(c): the minimum, over all 8-connected paths from c to a border cell, of the largest H on the path, c
 *     included.  Equivalently, W is the unique solution of W = H on border cells and W(c) = max(H(c), min over the 8
 *     neighbours W(n)) inside.  The cell's depression depth is W - H: one subtraction, bit-exact against the same H.
 *     W uses only min and max, so it is exact in f64 in any evaluation order.
 *   dir(c): an index k into the neighbour order n[] = (-1,-1), (-1,0), (-1,1), (0,-1), (0,1), (1,-1), (1,0), (1,1)
 *     of (dx, dy).  Rules, in order:
 *     -1 on a border cell.
 *     A drained cell has a neighbour with W(n) < W(c).  Its dir is the k of largest (W(c) - W(n)) / d, with d = 1.0 or
 *     sqrt(2.0) (f64, correctly rounded).  Ties go to the lower k.
 *     Any other interior cell lies on a flat.  dist(c) is the number of 8-connected steps through cells of equal W to
 *     the nearest drained or border cell of that W.  The flat cell's dir is the lowest k with W(n) == W(c) and
 *     dist(n) == dist(c) - 1.
 *     After filling, such an n always exists.  The receivers form a forest rooted at the border cells: each hop lowers
 *     W, or keeps W and lowers dist.
 *   area(c) = 1 + the sum of area(d) over every d whose receiver is c: the cells that drain through c, itself
 *     included.  An exact int64.
 *   basin(c) = the global index x*dimy + y of the border cell at which c's receiver chain ends.
 * Any of spill, dir, area, basin may be NULL: that output is then not written, but it is still computed when a later
 * output needs it.  flags: SM_DRAIN_GROUND, no other bit.  on_device != 0: the outputs are device pointers on the
 * context's device (rank 0's for a group); otherwise host memory.  stats may be NULL.
 * The call is read-only: columns, pool, frequency arrays, budgets and per-cell maps, the mesh and an open batch are left
 * exactly as they were.  A refusal (an unknown flag bit, all four outputs NULL, no map: a rank of a sharded map
 * without its peers attached) returns SM_ERR_INVALID before any launch, with nothing written.
 * The view is global: a cell's spill height can depend on the far side of the map, so every computation runs over the
 * whole map on one device, which first gathers H of every strip into a whole-map raster.  It needs about 50 B per cell
 * of device memory there (about 3.4 GB at 8192^2), freed when the call returns.  Group: rank 0 computes after every
 * rank's work has completed, and the results go into the caller's whole-map buffers.  Rank of a sharded map (in
 * process or across processes over CUDA IPC): it needs sm_peer_attach and the precondition of the views above (every
 * rank's earlier work has completed); the rank computes the whole map and writes its own strip, in cell order
 * (x - x0)*dimy + y, with basin still holding global indices.  Each rank that calls it repeats the whole-map work.
 * Every output is byte for byte that of one context.
 * Stats: fill_passes and dist_passes are the tile passes of the two relaxations, up to the one that changed nothing;
 * with tiles racing in one pass they can differ from run to run, the results cannot.  jump_passes: the pointer-jumping
 * passes of the basins.  longest_walk: the most receivers one walker of the area phase visited.  phase_ms: CUDA-event
 * time of heights, fill, dist, receivers, area, basin; device_ms is their sum. */
#define SM_DRAIN_GROUND 1
typedef struct sm_drain_stats {
  int64_t fill_passes;      /* tile passes of the fill */
  int64_t flat_cells;       /* interior cells that are not drained */
  int64_t depressed_cells;  /* cells with W > H */
  int64_t outlets;          /* border cells with area > 1 */
  double device_ms;         /* CUDA-event time of the kernels */
  int64_t dist_passes;      /* tile passes of the flat distances */
  int64_t jump_passes;      /* pointer-jumping passes of the basins */
  int64_t longest_walk;     /* receivers visited by the longest area walker */
  double phase_ms[6];       /* heights, fill, dist, receivers, area, basin */
} sm_drain_stats;
int sm_drainage(sm_context* ctx, int32_t flags, double* spill, int8_t* dir, int64_t* area, int64_t* basin,
                int32_t on_device, sm_drain_stats* stats);

/* WaterParticle::frequency/track, WindParticle::frequency (water.h:345-346, wind.h:48).
 * Any pointer may be NULL. */
int sm_get_frequency(sm_context* ctx, float* water_frequency, float* water_track, float* wind_frequency);
int sm_set_frequency(sm_context* ctx, const float* water_frequency, const float* water_track,
                     const float* wind_frequency);
/* mapfrequency + resetfrequency (water.h:353-365; SoilMachine.cpp:313-320) */
int sm_frequency_update(sm_context* ctx);

/* ---- meshing / export (renderer side of the boundary) ---------------------------------------------- */
/* SurfParam::color per soil (surface.h:17; io.h:158-159), rgba, n = number of soils. */
int sm_set_soil_colors(sm_context* ctx, const float* rgba, int32_t n);
/* Layermap::update(Vertexpool&) (layermap.h:551-555 = update(ivec2,...) :475-549 for every cell): one
 * 44-byte Vertex {position[3], normal[3], color[4], index} per cell in cell order, sliced at the plane
 * SLICE (SoilMachine.cpp:12).  The vertices stay in device memory (sm_mesh_device_ptr, e.g. for GL
 * interop); host_vertices may be NULL or a buffer of cells*11 floats (cells of this rank's strip on a sharded map). */
int sm_mesh_update(sm_context* ctx, int32_t slice, float* host_vertices);
int sm_mesh_device_ptr(sm_context* ctx, void** dptr);   /* SM_ERR_INVALID on a group of several ranks */
/* exportheight / exportcolor (io.h:234-252): the values the reference writes to the PNGs, as floats:
 * height[cell] = position.y / SCALE / sqrt(2); color[cell*4..] = (b, g, r, 1) of the vertex colour.
 * Both read the mesh of the last sm_mesh_update. */
int sm_export_height(sm_context* ctx, float* height);
int sm_export_color(sm_context* ctx, float* bgra);

/* ---- single-cell operations (what the facade's legacy Layermap calls forward to) -------------- */
int sm_cell_add(sm_context* ctx, int32_t x, int32_t y, double size, int32_t type); /* layermap.h:230 */
int sm_cell_remove(sm_context* ctx, int32_t x, int32_t y, double h, double* leftover); /* :310 */
int sm_cell_cascade(sm_context* ctx, float x, float y, int32_t transferloop);  /* particle.h:24 */
int sm_cell_query(sm_context* ctx, int32_t x, int32_t y, double* height, int32_t* surface,
                  float* normal3);  /* layermap.h:422,417,341 */
int sm_height_bilinear(sm_context* ctx, float x, float y, double* height); /* layermap.h:427 */
/* one whole column bottom -> top (Layermap::top(ivec2) and its prev chain, layermap.h:150-152); *n = number of
 * sections in the column, at most `capacity` of them are written */
int sm_cell_column(sm_context* ctx, int32_t x, int32_t y, int32_t capacity, int32_t* n, int32_t* type, double* size,
                   double* floor, double* saturation);
/* static WaterParticle::seep(vec2, ...) (water.h:285-333) and WaterParticle::cascade(vec2, ..., spill)
 * (water.h:151-283, nested particles included) for one cell */
int sm_cell_seep(sm_context* ctx, int32_t x, int32_t y);
int sm_cell_water_cascade(sm_context* ctx, int32_t x, int32_t y, int32_t spill);
/* WaterParticle::volumeFactor (water.h:33,368: a mutable static upstream, default 0.015) for later floods */
int sm_set_volume_factor(sm_context* ctx, double volume_factor);

/* ---- the hot path --------------------------------------------------------------------------- */
/* One batch of n particles run to completion in lockstep sweeps: in every sweep each live particle,
 * in ascending index order, executes move() && interact().  Replaces the loop
 * SoilMachine.cpp:288-298 (water; the flood tail is sm_water_flood) / 304-307 (wind).  spawn_xy = n (x,y) pairs,
 * the positions the ctor draws (water.h:13, wind.h:15).  max_sweeps <= 0: until all are dead. */
int sm_water_run(sm_context* ctx, int32_t n, const float* spawn_xy, int32_t max_sweeps, sm_stats* stats);
int sm_wind_run(sm_context* ctx, int32_t n, const float* spawn_xy, int32_t max_sweeps, sm_stats* stats);

/* Same, spawn list already in device memory (no host<->device copy, no sync; stats fetched by
 * sm_last_stats after sm_sync). */
int sm_water_run_device(sm_context* ctx, int32_t n, const float* d_spawn_xy, int32_t max_sweeps);
int sm_wind_run_device(sm_context* ctx, int32_t n, const float* d_spawn_xy, int32_t max_sweeps);
int sm_last_stats(sm_context* ctx, sm_stats* stats);

/* Mass budget of the last batch (contexts created with SM_FLAG_BUDGET).  The reference is not conservative -
 * sediment is discarded when a particle dies, clamped at 1 (water.h:117), cascade transfers are narrowed to f32
 * (particle.h:87-91), negative wind forces lower sediment without touching the map (wind.h:107-110) - so "mass
 * conservation" is a budget: every term is accumulated per particle in step order and summed in particle order,
 * bit-identical to the oracle port's accumulators (oracle/sm_oracle.cpp) on any number of GPUs.
 * Identity: change of (sum of all column heights) = deposited - eroded + cascade_net, to rounding. */
typedef struct sm_budget {
  double eroded;         /* height taken off the map by erosion           (water.h:98-100, wind.h:109) */
  double deposited;      /* height put on the map by deposition           (water.h:109, wind.h:123-124) */
  double cascade_net;    /* net height change of the cascade transfers    (particle.h:87-92) */
  double discarded;      /* water: sediment x volume lost at evaporation / map exit (water.h:65-69,118-119);
                            wind: sediment lost when the particle dies (wind.h:83-88) */
  double clamped;        /* water.h:117: (sediment - 1) x volume cut off */
  double wind_negative;  /* wind.h:107-110: sum of the negative suspension*force terms */
  int64_t particles;     /* particles of the batch */
} sm_budget;
int sm_last_budget(sm_context* ctx, sm_budget* budget);
/* the raw accumulators, 6 per particle (order as in sm_budget), for reductions over the ranks of a sharded map:
 * exactly one rank holds a particle's sums, the others hold zeros */
int sm_budget_particles(sm_context* ctx, int32_t n, double* out6n);
/* Per-cell maps of the mass budget of the last batch (contexts created with SM_FLAG_BUDGET | SM_FLAG_CELL_BUDGET):
 * where the batch eroded, deposited and moved height by cascades.  Three f64 per cell of this context's strip, cell
 * order x*dimy + y ((x - x0)*dimy + y on a sharded map, as sm_download_height); any pointer may be NULL.
 *   eroded       at the particle's ipos, around the erosion remove (water.h:98-100; wind.h:109, signed)
 *   deposited    water: at ipos (water.h:109); wind: at npos, then at ipos, each add measured at its own cell
 *                (wind.h:123-124)
 *   cascade_net  at both cells of every transfer of Particle::cascade (particle.h:87-92), nested re-cascades
 *                included: the higher cell gets its own change of height and the lower cell its own
 * Each delta is a column height (floor + top size) read right before and right after the column operation, at the
 * measurement points of sm_budget, credited to the cell whose height was read.  A cell's total starts at +0.0 when
 * the batch begins and every delta is added in execution order; two particle-steps that touch a cell are ordered by
 * the lockstep schedule, so the maps are deterministic and bit-identical to a sequential restatement on any schedule
 * and any number of ranks (the particle budget adds a transfer's two cells as one sum, the maps add each cell on its
 * own).  Per cell: height after - height before = deposited - eroded + cascade_net, to rounding; cells no step
 * touched hold exactly 0.0.
 * Scope: the last batch.  sm_water_run / sm_wind_run / *_run_device / *_begin reset the maps, *_sweeps adds onto them;
 * sm_water_flood, sm_seep and the single-cell calls never touch them, so the particles the pooling hydrology spawns
 * are not in the maps (sm_last_hydro_cell_budget has the floods' and the seep pass's own).  On a sharded map a step also writes into the neighbouring ranks' maps: every rank's batch must
 * have completed (sm_sync on every rank, then a host barrier) before the maps are read.
 * Memory: 24 B per cell (403 MB at 4096^2, 1.6 GB at 8192^2).  Only the warp sweep kernel keeps the maps.
 * SM_ERR_INVALID without SM_FLAG_CELL_BUDGET, before the first batch, or when the last batch ran on a kernel without
 * the maps (SM_KERNEL=thread).  sm_create refuses SM_FLAG_CELL_BUDGET without SM_FLAG_BUDGET, sm_peer_attach ranks
 * that disagree on it. */
int sm_last_cell_budget(sm_context* ctx, double* eroded, double* deposited, double* cascade_net);

/* Stepping interface for parity tests: begin a batch, advance k sweeps, read particle state. */
int sm_water_begin(sm_context* ctx, int32_t n, const float* spawn_xy);
int sm_water_sweeps(sm_context* ctx, int32_t k, sm_stats* stats);
int sm_water_state(sm_context* ctx, float* pos2, float* speed2, double* volume, double* sediment,
                   int32_t* contains, int32_t* alive);
int sm_wind_begin(sm_context* ctx, int32_t n, const float* spawn_xy);
int sm_wind_sweeps(sm_context* ctx, int32_t k, sm_stats* stats);
int sm_wind_state(sm_context* ctx, float* pos2, float* speed3, double* height, double* sediment,
                  int32_t* contains, int32_t* alive);

/* ---- pooling hydrology (the rest of the water part of the frame, SoilMachine.cpp:292-301) --------- */
typedef struct sm_hydro_stats {
  int64_t floods;        /* flood() calls that passed the volume/spill guard (water.h:125), nested ones included */
  int64_t nested;        /* particles spawned by the water-table cascade (water.h:243-256) */
  int64_t nested_steps;  /* their particle-steps */
  int64_t transfers;     /* partial water-table transfers (water.h:260-272) */
  int64_t cells;         /* sm_seep: cells visited (the cells where a visit can change anything) */
  double device_ms;      /* CUDA-event time of the call's kernels */
  double classify_ms;    /* sm_seep: the full-grid classification kernel alone (32 B per cell read) */
} sm_hydro_stats;
/* WaterParticle::flood (water.h:123-145) for every finished particle of the last water batch, in
 * ascending particle index; each flood is atomic, i.e. the water-table cascade (water.h:151-283) and the
 * particles it spawns run to completion inside it exactly as upstream.  Call after sm_water_run.
 * Sharded map: issued from the one rank named by sm_hydro_issuer once every rank's batch has completed (sm_sync on every rank, then a host
 * barrier); it floods every rank's finished particles over the whole map, bit-identical to one context, on the warp
 * executor whatever SM_HYDRO says.  Stats, budget and errors belong to the issuing context. */
int sm_water_flood(sm_context* ctx, sm_hydro_stats* stats);
/* WaterParticle::seep(map, vertexpool) (water.h:335-343): the per-frame pass over all cells in x-major
 * order, seep(cell) then the water-table cascade with spill 3.  Sharded map: as sm_water_flood (the issuing rank, the
 * whole map, warp executor). */
int sm_seep(sm_context* ctx, sm_hydro_stats* stats);
/* A water batch with sweep floods: the order of sm_water_run, except that after every sweep s the particles that
 * stopped in it call flood() (water.h:123-145), in ascending index, before sweep s+1 starts; the live particles of
 * sweep s+1 meet those ponds (Air tops, changed surfaces and heights).  Upstream floods each particle right after its
 * own loop (SoilMachine.cpp:290-297); sm_water_run + sm_water_flood floods only once the whole batch has ended.  Each
 * flood is atomic as in sm_water_flood and follows flood()'s own guard (volume >= minvol, spill left), so particles
 * that left the map or evaporated do not flood; a particle floods at most once.  For n = 1 this equals sm_water_run +
 * sm_water_flood.  max_sweeps > 0 stops after that many sweeps (and their floods); the survivors stay live, and
 * sm_water_sweeps can resume them without floods.
 * stats: the batch's counters (sweeps counts the sweeps that ran a particle; pool_drops covers the floods too).
 * hstats: the floods' counters summed over the call (cells = 0).  device_ms of both = the whole call's device time.
 * SM_FLAG_BUDGET: sm_last_budget covers the batch's particles, sm_last_hydro_budget every flood of the call, summed in
 * execution order; SM_FLAG_CELL_BUDGET / SM_FLAG_HYDRO_CELL_BUDGET: the batch maps and the hydrology maps cover the
 * same call.  The identity of the two budgets closes over the call: change of the whole map's height = the batch terms
 * + the flood terms.  A group floods from rank 0 over the whole map, bit-identical to one context.  A rank of a map
 * sharded over processes returns SM_ERR_INVALID (every sweep would need a flood issued across the processes). */
int sm_water_run_flooding(sm_context* ctx, int32_t n, const float* spawn_xy, int32_t max_sweeps, sm_stats* stats,
                          sm_hydro_stats* hstats);
/* Mass budget of the last successful sm_water_flood or sm_seep call (contexts created with SM_FLAG_BUDGET; such a
 * context runs both on the warp executor whatever SM_HYDRO says).  Same rules as sm_budget: each term is a change
 * of column height (floor + top size) read right before and right after the column operation, accumulated in
 * execution order, bit-identical to the oracle port's accumulators.  The terms are heights, not materials: a
 * remove on an Air-topped column takes water first, so nested_eroded can include water.  The single-cell calls
 * (sm_cell_seep, sm_cell_water_cascade) are not covered.
 * Identity: change of (sum of all column heights) = flood_sediment + flood_cascade_net + flood_water - seeped
 *           - to_particles + transfer_net + nested_deposited - nested_eroded + nested_cascade_net, to rounding.
 * SM_ERR_INVALID without SM_FLAG_BUDGET or before the first hydrology call.  On a sharded map it reports the last call
 * THIS context issued (the whole map's budget for that call). */
typedef struct sm_hydro_budget {
  double flood_sediment;      /* height added by the floods' sediment add                        (water.h:133) */
  double flood_cascade_net;   /* net height change of the floods' terrain cascade, as cascade_net (water.h:134) */
  double flood_water;         /* height added by the floods' Air add                             (water.h:138) */
  double seeped;              /* height of standing water removed by seep(cell), positive: inside the floods and
                                 in the seep pass (water.h:318-319) */
  double to_particles;        /* height removed when a whole water section leaves as a nested particle (water.h:248) */
  double transfer_net;        /* partial water-table transfers: height lost + height gained (water.h:268-271) */
  double nested_eroded;       /* sm_budget's eroded, deposited, cascade_net, discarded and clamped, summed over */
  double nested_deposited;    /*   every step of every particle the water-table cascade spawned (water.h:252-253) */
  double nested_cascade_net;
  double nested_discarded;
  double nested_clamped;
} sm_hydro_budget;
int sm_last_hydro_budget(sm_context* ctx, sm_hydro_budget* budget);
/* Per-cell maps of the hydrology's mass budget (contexts created with SM_FLAG_BUDGET | SM_FLAG_HYDRO_CELL_BUDGET):
 * where the last successful sm_water_flood or sm_seep call - the scope of sm_last_hydro_budget - changed the map.  Four
 * f64 per cell, cell order x*dimy + y (as sm_download_height); any pointer may be NULL.
 *   eroded       a nested particle's erosion, at its ipos                            (refines nested_eroded)
 *   deposited    the flood's sediment add at the truncated ipos (water.h:133); a nested particle's deposit
 *                                                                                    (flood_sediment + nested_deposited)
 *   cascade_net  both cells of every terrain-cascade transfer, each its own change of height: the flood's cascade
 *                (water.h:134) and the nested particles' cascades           (flood_cascade_net + nested_cascade_net)
 *   water_net    the flood's Air add (water.h:138, +); every seep(cell), in a flood and in the seep pass (-, the
 *                height removed); a whole water section leaving as a nested particle, at tpos (water.h:248, -); a
 *                partial transfer, tpos and bpos each their own change (water.h:268-271)
 *                                                         (flood_water - seeped - to_particles + transfer_net)
 * Each delta is measured where the sm_hydro_budget sums are and credited to the cell whose height was read; the
 * terms are heights, not materials (eroded can include water).  nested_discarded and nested_clamped have no cell.
 * Every cell starts each call at +0.0 and its deltas are added in execution order, so the maps are deterministic.
 * Per cell: height after - height before = deposited - eroded + cascade_net + water_net, to rounding; cells nothing
 * touched hold exactly 0.0; summed over the cells each map equals its group of sm_hydro_budget terms, to rounding.
 * The batch maps (sm_last_cell_budget) are not touched; the single-cell calls (sm_cell_seep, sm_cell_water_cascade)
 * are not covered.  Memory: 32 B per cell of device memory (537 MB at 4096^2, 2.1 GB at 8192^2), zeroed by every
 * sm_water_flood / sm_seep call inside its device_ms; this call stages the interleaved map through a 32 MB host buffer.
 * SM_ERR_INVALID without SM_FLAG_HYDRO_CELL_BUDGET, before the first sm_water_flood / sm_seep call (a water batch alone
 * does not count), or when the last of these calls failed (its maps were reset and are partial).  sm_create refuses
 * the flag without SM_FLAG_BUDGET, and sm_create_sharded refuses it with nranks > 1 (the pooling hydrology runs on a
 * sharded context without these maps). */
int sm_last_hydro_cell_budget(sm_context* ctx, double* eroded, double* deposited, double* cascade_net,
                              double* water_net);

/* ---- wind field: D3Q19 lattice Boltzmann, TRT collision (source/include/lbmwind/) ------------------------------
 * The reference runs this as OpenGL compute shaders and only draws it (WindParticle keeps a constant prevailing
 * wind, wind.h:29).  sm_lbm_create = lbmw::initialize (lbmwind.h:75-118: buffers + init.cs with an all-zero
 * boundary); sm_lbm_set_boundary = SoilMachine.cpp:234-239 (NULL: from this context's terrain, else nx*ny*nz
 * floats, > 0 = obstacle); sm_lbm_step = n x (collide.cs + stream.cs) fused into one kernel per step
 * (lbmwind.h:170-187); sm_lbm_get: populations in upstream's layout F[cell*19 + q] with cell = (x*ny + y)*nz + z,
 * density, velocity (x, y, z, w); sm_lbm_advect = move.cs (tracer particles, n x (x, y, z, w), in place).
 * Arithmetic is defined by oracle/lbm_oracle.c (parity with the GLSL unpinned: no GL here, no reference vectors).
 * Sharded map: the lattice is not sharded; every rank keeps a full, identical copy.  Every rank calls sm_lbm_create
 * with the same dimensions, builds the same boundary (NULL: from the whole map, with the precondition of the
 * sharded-map paragraph above) and steps the lattice the same number of times; sm_lbm_get returns the rank's full
 * lattice, and sm_wind_use_lbm couples each rank's wind particles to its own copy. */
int sm_lbm_create(sm_context* ctx, int32_t nx, int32_t ny, int32_t nz);
int sm_lbm_set_boundary(sm_context* ctx, const float* boundary);
int sm_lbm_init(sm_context* ctx);                        /* init.cs again, with the current boundary */
int sm_lbm_step(sm_context* ctx, int32_t nsteps, double* device_ms);
int sm_lbm_get(sm_context* ctx, float* f, float* rho, float* v4);
int sm_lbm_advect(sm_context* ctx, int32_t n, float* pos4);
/* EXTENSION, off by default (upstream never couples the two: wind.h:29 is a constant): on != 0 makes the prevailing
 * wind `pspeed` of later wind batches the lattice velocity at the particle (nearest lattice cell, / 0.05, components
 * clamped to [-2, 2]) instead of (-2, 0, 1).  The oracle port implements the same rule (smo_set_wind_field). */
int sm_wind_use_lbm(sm_context* ctx, int32_t on);

/* CUDA-event stopwatch on the context's stream (the stream every kernel of this context is
 * launched on): start records an event, stop records another, synchronises and returns the elapsed
 * device time between them. */
int sm_timer_start(sm_context* ctx);
int sm_timer_stop(sm_context* ctx, double* elapsed_ms);

/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
int sm_launch_count(sm_context* ctx, int64_t* n);
/* Device pointer helpers so a caller can keep spawn lists resident. */
int sm_device_alloc(sm_context* ctx, int64_t bytes, void** dptr);
int sm_device_free(sm_context* ctx, void* dptr);
int sm_device_upload(sm_context* ctx, void* dptr, const void* host, int64_t bytes);

#ifdef __cplusplus
}
#endif
#endif
