// sm_group.cuh -- a context group: one sm_context over a map cut into x-strips, every rank living in this process
// (sm_create_group).  Included by sm_engine.cu, which sends every entry point here when ctx->group is set.
//
// The group owns one sharded context per rank, attaches them to each other without IPC and names rank 0 the issuer of
// the pooling hydrology.  Callers see the whole map in the unsharded cell order: inputs are cut at the ranks' strips,
// outputs are written by each rank into its slice of the caller's buffer.  Calls that read or write other ranks'
// strips need every rank's earlier work to have completed; inside one process that is sm_sync on every rank
// (grp_settle), and `dirty` remembers whether anything was enqueued since the last one.
//
// Also here: k_cell_op_w, the warp form of the single-cell calls that change the map (sm_cell_coop.cuh), which the
// group launches on rank 0 - the one-thread k_cell_op knows one strip only.
#pragma once
#include "sm_cell_coop.cuh"

// The single-cell mutators on the back-end of the sharded hydrology: each record access, pool allocation and free goes
// to the column's owner.  Pool phase 0 as k_cell_op and k_hydro_flood_w (frees to ring 0, allocations from ring 1 or
// the bump counter), so a slot freed by one call is never popped by the next while it may still be linked.
template <bool MULTI>
__global__ void __launch_bounds__(32) k_cell_op_w(DevCtx c, CellOp o, CellRes* res, const __grid_constant__ FreqPeers fp) {
  __shared__ SoilDev s_soils[SM_MAX_SOILS];
  __shared__ CoopScratch sc;
  __shared__ CellCascadeScratch deep;
  __shared__ HydroScratch hx;
  const int lane = threadIdx.x;
  for (int i = lane; i < c.nsoils; i += 32) s_soils[i] = c.soils[i];
  __syncwarp();
  WarpDev w{lane};
  ActiveMap none{};
  HydroBack<MULTI, false> back(c, s_soils, none, false, nullptr, &fp);
  HydroCount hc{};
  const double d = cell_op_coop(w, back, &sc, &deep, &hx, o.op, o.x, o.y, o.fx, o.fy, o.v, o.t, hc);
  if (lane == 0) *res = CellRes{d, 0, {0.f, 0.f, 0.f}};
}
// one context: sm_cell_* keep k_cell_op; this instantiation is what the host emulation's arithmetic corresponds to
template __global__ void k_cell_op_w<false>(DevCtx c, CellOp o, CellRes* res, const __grid_constant__ FreqPeers fp);

struct sm_group {
  int n = 0;
  sm_context* rank[SM_MAX_RANKS] = {};
  bool dirty = true;             // something may be in flight on some rank
  cudaEvent_t ev = nullptr;      // on rank 0's device: orders the peers' copies of a device spawn list
};

// x-strips of equal width (a multiple of the largest bin edge, 16 cells); false: the rank would own no column
static const char kStripTooNarrow[] =
    "sm_create_sharded: the map is too narrow for this many ranks (needs >= 16 columns per rank)";
static bool shard_strip(int dimx, int nranks, int rank, int* strip_w, int* x0, int* x1) {
  *strip_w = (nranks == 1) ? dimx : ((((dimx + nranks - 1) / nranks) + 15) / 16) * 16;
  *x0 = rank * *strip_w;
  *x1 = std::min(dimx, *x0 + *strip_w);
  return *x1 > *x0;
}
// a non-zero pool_capacity is the whole map's: each rank gets its share by strip cells, rounded up
static int64_t shard_pool_capacity(int64_t whole, int dimx, int x0, int x1) {
  return whole <= 0 ? 0 : (whole * (int64_t)(x1 - x0) + dimx - 1) / dimx;
}

extern "C" {
static int create_impl(const sm_config* cfg, int nranks, int rank, int share, sm_context** out);
static int launch_run(sm_context* ctx, int kind, int n, const float* d_spawn, int max_sweeps);
static int zero_counters(sm_context* ctx);
static int height_sum(sm_context* ctx, bool whole_map, double* sum);
static int cell_op(sm_context* ctx, const CellOp& o, CellRes* out);
}

static int grp_err(sm_context* ctx, int r, int rc) {
  ctx->err = "rank " + std::to_string(r) + ": " + ctx->group->rank[r]->err;
  return rc;
}
// f(rank context, rank) on every rank; the calls may leave work in flight
template <class F> static int grp_each(sm_context* ctx, F f) {
  sm_group& G = *ctx->group;
  G.dirty = true;
  for (int r = 0; r < G.n; r++) {
    const int rc = f(G.rank[r], r);
    if (rc != SM_OK) return grp_err(ctx, r, rc);
  }
  return SM_OK;
}
static int grp_settle(sm_context* ctx) {
  sm_group& G = *ctx->group;
  if (!G.dirty) return SM_OK;
  const int rc = grp_each(ctx, [](sm_context* c, int) { return sm_sync(c); });
  if (rc == SM_OK) G.dirty = false;
  return rc;
}
// f(rank 0's context), without settling: calls that touch nothing but rank 0's own state
template <class F> static int grp_rank0(sm_context* ctx, F f) {
  const int rc = f(ctx->group->rank[0]);
  return rc != SM_OK ? grp_err(ctx, 0, rc) : SM_OK;
}
// settle, then f(rank context, rank) on every rank: each rank reads (its slice of) the settled map
template <class F> static int grp_settled_each(sm_context* ctx, F f) {
  const int rc = grp_settle(ctx);
  return rc != SM_OK ? rc : grp_each(ctx, f);
}
// settle, then f(rank 0's context): calls that take global coordinates or work on the whole map from one rank
template <class F> static int grp_settled_rank0(sm_context* ctx, F f) {
  const int rc = grp_settle(ctx);
  return rc != SM_OK ? rc : grp_rank0(ctx, f);
}

static void grp_destroy(sm_context* ctx) {
  sm_group& G = *ctx->group;
  // a rank's kernel may still be reading its peers' arrays: every rank is idle before any rank's memory goes
  for (int r = 0; r < G.n; r++)
    if (G.rank[r]) { cudaSetDevice(G.rank[r]->cfg.device); cudaStreamSynchronize(G.rank[r]->stream); }
  if (G.ev) { cudaSetDevice(G.rank[0]->cfg.device); cudaEventDestroy(G.ev); }
  for (int r = 0; r < G.n; r++) sm_destroy(G.rank[r]);
  delete ctx->group;
  delete ctx;
}

static int grp_create(const sm_config* cfg, int nranks, const int32_t* devices, sm_context** out) {
  if (!cfg || !out || nranks < 1 || nranks > SM_MAX_RANKS) {
    g_create_err = "sm_create_group: invalid arguments (1 <= nranks <= 8)";
    return SM_ERR_INVALID;
  }
  if (nranks == 1) {
    sm_config one = *cfg;
    if (devices) one.device = devices[0];
    return sm_create(&one, out);
  }
  for (int r = 0; r < nranks; r++) {
    int w, x0, x1;
    if (cfg->dimx >= 2 && !shard_strip(cfg->dimx, nranks, r, &w, &x0, &x1)) {
      g_create_err = kStripTooNarrow;
      return SM_ERR_INVALID;
    }
  }
  sm_context* ctx = new sm_context();
  ctx->group = new sm_group();
  sm_group& G = *ctx->group;
  G.n = nranks;
  ctx->cfg = *cfg;
  memset(&ctx->d, 0, sizeof(DevCtx));
  ctx->d.dimx = cfg->dimx; ctx->d.dimy = cfg->dimy; ctx->d.scale = cfg->scale;
  ctx->x1 = cfg->dimx;
  int rc = SM_OK;
  for (int r = 0; r < nranks && rc == SM_OK; r++) {
    sm_config rcfg = *cfg;
    if (devices) rcfg.device = devices[r];
    int share = 0, w, x0, x1;
    for (int q = 0; q < nranks; q++) share += (devices ? devices[q] : cfg->device) == rcfg.device;
    shard_strip(cfg->dimx, nranks, r, &w, &x0, &x1);
    rcfg.pool_capacity = shard_pool_capacity(cfg->pool_capacity, cfg->dimx, x0, x1);
    rc = create_impl(&rcfg, nranks, r, share, &G.rank[r]);      // g_create_err holds the rank's message
  }
  if (rc == SM_OK) {
    std::vector<sm_peer_blob> blobs((size_t)nranks);
    int bad = 0;
    for (int r = 0; r < nranks && rc == SM_OK; r++) { rc = sm_peer_export(G.rank[r], &blobs[(size_t)r]); bad = r; }
    for (int r = 0; r < nranks && rc == SM_OK; r++) { rc = sm_peer_attach(G.rank[r], blobs.data(), nranks, 0); bad = r; }
    if (rc == SM_OK) { rc = sm_hydro_issuer(G.rank[0], 1); bad = 0; }
    if (rc == SM_OK) {
      bad = 0;
      if (cudaSetDevice(G.rank[0]->cfg.device) != cudaSuccess ||
          cudaEventCreateWithFlags(&G.ev, cudaEventDisableTiming) != cudaSuccess) {
        G.rank[0]->err = "cudaEventCreate failed";
        rc = SM_ERR_CUDA;
      }
    }
    if (rc != SM_OK) g_create_err = "rank " + std::to_string(bad) + ": " + G.rank[bad]->err;
  }
  if (rc != SM_OK) {
    grp_destroy(ctx);
    return rc;
  }
  ctx->cells = ctx->lcells = (size_t)cfg->dimx * cfg->dimy;
  ctx->max_particles = G.rank[0]->max_particles;
  *out = ctx;
  return SM_OK;
}

// ---- whole-map inputs, cut at the strips ----------------------------------------------------------------------
static int grp_upload_columns(sm_context* ctx, const int64_t* offsets, const int32_t* type, const double* size,
                              const double* saturation) {
  if (!offsets || !type || !size) return fail(ctx, SM_ERR_INVALID, "sm_upload_columns: null argument");
  std::vector<int64_t> off;     // the strip's offsets, rebased; the sections themselves are passed in place
  return grp_each(ctx, [&](sm_context* c, int) {
    const size_t lo = (size_t)c->x0 * ctx->d.dimy;
    const int64_t base = offsets[lo];
    off.resize(c->lcells + 1);
    for (size_t i = 0; i <= c->lcells; i++) off[i] = offsets[lo + i] - base;
    return sm_upload_columns(c, off.data(), type + base, size + base, saturation ? saturation + base : nullptr);
  });
}
static int grp_download_columns(sm_context* ctx, int64_t capacity, int64_t* offsets, int32_t* type, double* size,
                                double* floor_, double* saturation) {
  int64_t base = 0;
  return grp_settled_each(ctx, [&](sm_context* c, int) {
    int64_t* const off = offsets + (size_t)c->x0 * ctx->d.dimy;
    const int rc = sm_download_columns(c, capacity - base, off, type ? type + base : nullptr, size ? size + base : nullptr,
                                       floor_ ? floor_ + base : nullptr, saturation ? saturation + base : nullptr);
    if (rc != SM_OK) return rc;
    const int64_t n = off[c->lcells];
    for (size_t i = 0; i <= c->lcells; i++) off[i] += base;
    base += n;
    return SM_OK;
  });
}
// frequency arrays are y*dimx + x: a rank's columns are a 2-D block; its copy is authoritative for those only
static int grp_frequency(sm_context* ctx, bool set, float* const host[3]) {
  const int rc = grp_settle(ctx);
  if (rc != SM_OK) return rc;
  sm_group& G = *ctx->group;
  const size_t pitch = (size_t)ctx->d.dimx * 4;
  for (int r = 0; r < G.n; r++) {
    sm_context* const c = G.rank[r];
    float* const dev[3] = {c->d.wfreq, c->d.wtrack, c->d.windfreq};
    CK(cudaSetDevice(c->cfg.device));
    for (int k = 0; k < 3; k++) {
      if (!host[k]) continue;
      const size_t width = (size_t)(c->x1 - c->x0) * 4;
      if (set) CK(cudaMemcpy2D(dev[k] + c->x0, pitch, host[k] + c->x0, pitch, width, (size_t)ctx->d.dimy, cudaMemcpyHostToDevice));
      else CK(cudaMemcpy2D(host[k] + c->x0, pitch, dev[k] + c->x0, pitch, width, (size_t)ctx->d.dimy, cudaMemcpyDeviceToHost));
    }
  }
  return SM_OK;
}

// ---- batches ---------------------------------------------------------------------------------------------------
// steps, exits and drops add up over the ranks; sweeps, device time and the live count are the same global quantity
// seen by every rank (as sharded.sum_stats)
static int grp_last_stats(sm_context* ctx, sm_stats* st) {
  sm_group& G = *ctx->group;
  sm_stats tot;
  memset(&tot, 0, sizeof(tot));
  int bad = -1, bad_rc = SM_OK;
  for (int r = 0; r < G.n; r++) {
    sm_stats s;
    memset(&s, 0, sizeof(s));
    const int rc = sm_last_stats(G.rank[r], &s);
    if (rc != SM_OK && bad < 0) { bad = r; bad_rc = rc; }
    tot.steps += s.steps; tot.exit_oob += s.exit_oob; tot.exit_evap += s.exit_evap; tot.exit_stall += s.exit_stall;
    tot.pool_drops += s.pool_drops;
    tot.sweeps = std::max(tot.sweeps, s.sweeps); tot.alive = std::max(tot.alive, s.alive);
    tot.device_ms = std::max(tot.device_ms, s.device_ms);
  }
  if (st) *st = tot;
  if (bad >= 0) return grp_err(ctx, bad, bad_rc);
  G.dirty = false;            // sm_last_stats synchronised every rank's stream
  return SM_OK;
}
// A batch's kernels meet in a cross-rank barrier every sweep, so every rank's kernel must be launched before anything
// waits for one of them.  Everything that can block (the spawn list's copies) is enqueued for all ranks first; the
// launch path itself (launch_run) only queries occupancy and enqueues.  h_xy: host list, copied to every rank.  d_xy:
// list on rank 0's device; the other ranks get asynchronous peer copies on their own streams, ordered after rank 0's
// stream.  Neither: resume the batch in flight for max_sweeps sweeps.
static int grp_run(sm_context* ctx, int kind, int n, const float* h_xy, const float* d_xy, int max_sweeps, bool spawn) {
  sm_group& G = *ctx->group;
  sm_context* const c0 = G.rank[0];
  if (c0->nsoils < 1) return fail(ctx, SM_ERR_INVALID, "soil table not set");
  if (n < 0 || n > ctx->max_particles) return fail(ctx, SM_ERR_INVALID, "batch larger than max_particles");
  if (spawn && n > 0 && !h_xy && !d_xy) return fail(ctx, SM_ERR_INVALID, "null spawn list");
  G.dirty = true;
  const size_t bytes = (size_t)n * 8;
  if (spawn && h_xy && n) {
    for (int r = 0; r < G.n; r++) {
      CK(cudaSetDevice(G.rank[r]->cfg.device));
      CK(cudaMemcpyAsync(G.rank[r]->d_spawn, h_xy, bytes, cudaMemcpyHostToDevice, G.rank[r]->stream));
    }
  } else if (spawn && n) {
    CK(cudaSetDevice(c0->cfg.device));
    CK(cudaEventRecord(G.ev, c0->stream));
    for (int r = 1; r < G.n; r++) {
      sm_context* const c = G.rank[r];
      CK(cudaSetDevice(c->cfg.device));
      CK(cudaStreamWaitEvent(c->stream, G.ev, 0));
      CK(cudaMemcpyPeerAsync(c->d_spawn, c->cfg.device, d_xy, c0->cfg.device, bytes, c->stream));
    }
  }
  if (spawn) { ctx->cur_kind = kind; ctx->cur_n = n; }
  return grp_each(ctx, [&](sm_context* c, int r) {
    if (!spawn) {
      const int rc = zero_counters(c);
      return rc != SM_OK ? rc : launch_run(c, kind, c->cur_n, nullptr, max_sweeps);
    }
    const float* const list = (d_xy && !h_xy && r == 0) ? d_xy : c->d_spawn;
    return kind == KIND_WATER ? sm_water_run_device(c, n, list, max_sweeps) : sm_wind_run_device(c, n, list, max_sweeps);
  });
}
static int grp_sweeps(sm_context* ctx, int kind, int k, sm_stats* st) {
  if (ctx->cur_kind != kind) return fail(ctx, SM_ERR_INVALID, "no batch of this kind in flight");
  if (k <= 0) return fail(ctx, SM_ERR_INVALID, "k must be positive");
  const int rc = grp_run(ctx, kind, ctx->cur_n, nullptr, nullptr, k, false);
  return rc != SM_OK ? rc : grp_last_stats(ctx, st);
}
// exactly one rank holds a particle's six sums, the others hold +0.0: adding the ranks per particle keeps the bits
static int grp_budget_particles(sm_context* ctx, int32_t n, double* out) {
  std::vector<double> part;
  return grp_settled_each(ctx, [&](sm_context* c, int r) {
    if (r == 0) return sm_budget_particles(c, n, out);
    part.resize((size_t)std::max(n, 0) * SM_BUDGET_SLOTS);
    const int rc = sm_budget_particles(c, n, part.data());
    if (rc == SM_OK) for (size_t i = 0; i < part.size(); i++) out[i] += part[i];
    return rc;
  });
}
// One record per particle, from the rank that holds it: a live particle is alive on exactly one rank; a dead one's
// final state lies where its `done` word carries the dead or flooded marker (every rank clears done[0, n) before a
// spawning launch and writes a particle's word only while it holds the particle; see k_hydro_flood_w<true>).
static int grp_fetch_state(sm_context* ctx, std::vector<float4>& a, std::vector<double2>& b, std::vector<uint2>& pc,
                           std::vector<unsigned char>& al) {
  const int rc = grp_settle(ctx);
  if (rc != SM_OK) return rc;
  sm_group& G = *ctx->group;
  const size_t n = (size_t)ctx->cur_n;
  a.assign(n, float4{}); b.assign(n, double2{}); pc.assign(n, uint2{}); al.assign(n, 0);
  if (!n) return SM_OK;
  std::vector<float4> ra(n); std::vector<double2> rb(n); std::vector<uint2> rc3(n);
  std::vector<unsigned char> ral(n); std::vector<unsigned int> rdone(n);
  for (int r = 0; r < G.n; r++) {
    const DevCtx& d = G.rank[r]->d;
    CK(cudaSetDevice(G.rank[r]->cfg.device));
    CK(cudaMemcpy(ra.data(), d.pa, n * sizeof(float4), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(rb.data(), d.pb, n * sizeof(double2), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(rc3.data(), d.pc, n * sizeof(uint2), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(ral.data(), d.alive, n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(rdone.data(), d.done, n * sizeof(unsigned int), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; i++)
      if (ral[i] || rdone[i] == 0xFFFFFFFFu || rdone[i] == SM_DONE_FLOODED) {
        a[i] = ra[i]; b[i] = rb[i]; pc[i] = rc3[i]; al[i] = ral[i];
      }
  }
  return SM_OK;
}

// ---- the single-cell calls -------------------------------------------------------------------------------------
static int cell_op_warp(sm_context* ctx, const CellOp& o, CellRes* out) {   // ctx: rank 0 of a settled group
  CK(cudaSetDevice(ctx->cfg.device));
  k_cell_op_w<true><<<1, 32, 0, ctx->stream>>>(ctx->d, o, ctx->d_cellres, ctx->freq_of);
  ctx->launches++;
  CK(cudaGetLastError());
  CellRes r;
  CK(cudaMemcpyAsync(&r, ctx->d_cellres, sizeof(CellRes), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (out) *out = r;
  return SM_OK;
}
static int grp_cell_op(sm_context* ctx, const CellOp& o, CellRes* out) {
  const bool read = o.op == 3 || o.op == 4;
  if (!read && ctx->group->rank[0]->nsoils < 1) return fail(ctx, SM_ERR_INVALID, "soil table not set");
  const int rc = grp_settled_rank0(ctx, [&](sm_context* c) { return read ? cell_op(c, o, out) : cell_op_warp(c, o, out); });
  if (rc == SM_OK) ctx->group->dirty = false;     // rank 0's call was synchronous, the other ranks were idle
  if (o.op == 5 || o.op == 6) for (int r = 0; r < ctx->group->n; r++) ctx->group->rank[r]->mesh_valid = false;
  return rc;
}
// the pooling hydrology: issued from rank 0 over the settled map; the call itself waits for its kernels
template <class F> static int grp_hydro(sm_context* ctx, F f) {
  const int rc = grp_settled_rank0(ctx, f);
  if (rc == SM_OK) ctx->group->dirty = false;
  for (int r = 0; r < ctx->group->n; r++) ctx->group->rank[r]->mesh_valid = false;
  return rc;
}
