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
#define SM_FLAG_BUDGET 1      /* keep the per-particle mass budget (sm_last_budget); a few % slower */

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
 * that run their kernels concurrently on this device. */
#define SM_PEER_ARRAYS 20
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
 * interop); host_vertices may be NULL or a buffer of cells*11 floats. */
int sm_mesh_update(sm_context* ctx, int32_t slice, float* host_vertices);
int sm_mesh_device_ptr(sm_context* ctx, void** dptr);
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
 * particles it spawns run to completion inside it exactly as upstream.  Call after sm_water_run. */
int sm_water_flood(sm_context* ctx, sm_hydro_stats* stats);
/* WaterParticle::seep(map, vertexpool) (water.h:335-343): the per-frame pass over all cells in x-major
 * order, seep(cell) then the water-table cascade with spill 3. */
int sm_seep(sm_context* ctx, sm_hydro_stats* stats);

/* ---- wind field: D3Q19 lattice Boltzmann, TRT collision (source/include/lbmwind/) ------------------------------
 * The reference runs this as OpenGL compute shaders and only draws it (WindParticle keeps a constant prevailing
 * wind, wind.h:29).  sm_lbm_create = lbmw::initialize (lbmwind.h:75-118: buffers + init.cs with an all-zero
 * boundary); sm_lbm_set_boundary = SoilMachine.cpp:234-239 (NULL: from this context's terrain, else nx*ny*nz
 * floats, > 0 = obstacle); sm_lbm_step = n x (collide.cs + stream.cs) fused into one kernel per step
 * (lbmwind.h:170-187); sm_lbm_get: populations in upstream's layout F[cell*19 + q] with cell = (x*ny + y)*nz + z,
 * density, velocity (x, y, z, w); sm_lbm_advect = move.cs (tracer particles, n x (x, y, z, w), in place).
 * Arithmetic is defined by oracle/lbm_oracle.c (parity with the GLSL unpinned: no GL here, no reference vectors). */
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
