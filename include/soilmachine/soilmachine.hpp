// include/soilmachine/soilmachine.hpp -- C++ facade: the reference's own class names and call shapes
// for the particle/terrain hot path, forwarding to the C ABI (include/soilmachine_b200.h).
//
// The reference has no plugin boundary; its frame loop (SoilMachine.cpp:283-329) is written against
// these types, which upstream defines in source/layermap.h, source/surface.h and
// source/particle/{particle,water,wind}.h.  A maintainer swaps those four #includes for this header
// (INTEGRATION.md shows the diff) and the loop runs on the GPU:
//
//   Layermap map(SEED, ivec2(SIZEX, SIZEY), vertexpool);      // SoilMachine.cpp:83   -> sm_initialize
//   WaterParticle::run(map, vertexpool, NWATER);              // replaces :288-298    -> sm_water_run
//   WindParticle::run(map, vertexpool, NWIND);                // replaces :304-307    -> sm_wind_run
//   WaterParticle::mapfrequency(map); ...resetfrequency(map); // :313-320             -> sm_frequency_update
//
// Legacy per-cell calls (map.height(p), map.add(p, map.pool.get(h, type)), map.remove, map.surface,
// map.normal, Particle::cascade) keep working: each forwards to one sm_cell_* call (one tiny kernel,
// fine for the GUI / initialisation code that uses them, not meant for inner loops).
//
// Everything is header-only and written from scratch; vector types are minimal stand-ins that
// convert implicitly from/to any type with .x/.y(/.z) members (so glm::ivec2 etc. can be passed).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <deque>
#include <map>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>
#include "../soilmachine_b200.h"
#include "soilfile.hpp"

namespace soilmachine {

struct ivec2 {
  int x = 0, y = 0;
  ivec2() {}
  ivec2(int a, int b) : x(a), y(b) {}
  template <class V, class = decltype(std::declval<V>().x + std::declval<V>().y)>
  ivec2(const V& v) : x((int)v.x), y((int)v.y) {}
};
struct vec2 {
  float x = 0, y = 0;
  vec2() {}
  vec2(float a, float b) : x(a), y(b) {}
  template <class V, class = decltype(std::declval<V>().x + std::declval<V>().y)>
  vec2(const V& v) : x((float)v.x), y((float)v.y) {}
};
struct vec3 { float x = 0, y = 0, z = 0; };
struct vec4 { float x = 0, y = 0, z = 0, w = 0; };

using SurfType = size_t;

// surface.h:11-39
struct SurfParam {
  std::string name;
  float density = 0.0f, porosity = 0.0f;
  vec4 color{0.5f, 0.5f, 0.5f, 1.0f}, phong{0.5f, 0.8f, 0.2f, 32.0f};
  SurfType transports = 0; float solubility = 1.0f, equrate = 1.0f, friction = 1.0f;
  SurfType erodes = 0; float erosionrate = 0.0f;
  SurfType cascades = 0; float maxdiff = 1.0f, settling = 0.0f;
  SurfType abrades = 0; float suspension = 0.0f, abrasion = 0.0f;
};
// surface.h:65-101 (parameters only; the noise itself runs on the device, sm_initialize)
struct SurfLayer {
  SurfType type = 0;
  float min = 0.0f, bias = 0.0f, scale = 1.0f, octaves = 1.0f, lacunarity = 1.0f, gain = 0.0f, frequency = 1.0f;
  explicit SurfLayer(SurfType t) : type(t) {}
};

// the reference's global tables (surface.h:41-57,104)
inline std::vector<SurfParam>& soils_table() {
  static std::vector<SurfParam> t = [] { SurfParam air; air.name = "Air"; air.porosity = 1.0f;
    air.color = vec4{0.0f, 0.2f, 0.4f, 1.0f}; air.solubility = 0.0f; air.equrate = 0.0f; air.friction = 0.0f;
    air.maxdiff = 0.0f; return std::vector<SurfParam>{air}; }();
  return t;
}
inline std::map<std::string, int>& soilmap_table() { static std::map<std::string, int> m{{"Air", 0}}; return m; }
inline std::vector<SurfLayer>& layers_table() { static std::vector<SurfLayer> l; return l; }
// loadsoil(), io.h:7-230: fills the soils / soilmap / layers tables from a `.soil` file (same quirks as
// upstream, see soilfile.hpp) and returns the WORLD block; an application that keeps the reference's global
// ints assigns them from the result (SIZEX = w.sizex; ...).
inline WorldEntry loadsoil(const std::string& file = "soil/default.soil") {
  SoilFile f;
  parse_soil_file(file, f);
  soils_table().clear(); soilmap_table().clear(); layers_table().clear();
  for (const SoilEntry& e : f.soils) {
    SurfParam p;
    p.name = e.name; p.density = e.density; p.porosity = e.porosity;
    p.color = vec4{e.color[0], e.color[1], e.color[2], e.color[3]};
    p.phong = vec4{e.phong[0], e.phong[1], e.phong[2], e.phong[3]};
    p.transports = (SurfType)e.transports; p.solubility = e.solubility; p.equrate = e.equrate; p.friction = e.friction;
    p.erodes = (SurfType)e.erodes; p.erosionrate = e.erosionrate;
    p.cascades = (SurfType)e.cascades; p.maxdiff = e.maxdiff; p.settling = e.settling;
    p.abrades = (SurfType)e.abrades; p.suspension = e.suspension; p.abrasion = e.abrasion;
    soils_table().push_back(p);
  }
  for (const auto& kv : f.soilmap) soilmap_table()[kv.first] = kv.second;
  for (const LayerEntry& l : f.layers) {
    SurfLayer L((SurfType)l.type);
    L.min = l.min; L.bias = l.bias; L.scale = l.scale; L.octaves = l.octaves; L.lacunarity = l.lacunarity;
    L.gain = l.gain; L.frequency = l.frequency;
    layers_table().push_back(L);
  }
  return f.world;
}

#define soils (::soilmachine::soils_table())
#define soilmap (::soilmachine::soilmap_table())
#define layers (::soilmachine::layers_table())

struct Error : std::runtime_error { int code; Error(int c, const std::string& m) : std::runtime_error(m), code(c) {} };

// layermap.h:37-62 -- a value carrier on the host (the device owns the real columns)
struct sec {
  sec* next = nullptr; sec* prev = nullptr;
  SurfType type = 0; double size = 0.0, floor = 0.0, saturation = 0.0;
  sec() {}
  sec(double s, SurfType t) : type(t), size(s) {}
  void reset() { next = prev = nullptr; type = 0; size = floor = saturation = 0.0; }
};
// layermap.h:64-119
class secpool {
 public:
  int size = 0; sec* start = nullptr; std::deque<sec*> free;
  secpool() {}
  ~secpool() { delete[] start; }
  void reserve(int N) { delete[] start; start = new sec[N]; free.clear(); for (int i = 0; i < N; i++) free.push_front(start + i); size = N; }
  template <class... A> sec* get(A&&... a) {
    if (free.empty()) return nullptr;                       // layermap.h:92-95
    sec* E = free.back(); *E = sec(std::forward<A>(a)...); free.pop_back(); return E;
  }
  void unget(sec* E) { if (!E) return; E->reset(); free.push_front(E); }
  void reset() { free.clear(); for (int i = 0; i < size; i++) free.push_front(start + i); }
};

// layermap.h:127-228
class Layermap {
 public:
  ivec2 dim; secpool pool; unsigned* section = nullptr;
  sm_context* ctx = nullptr;

  // Several GPUs: ngpus > 1 cuts the map into that many x-strips, rank r on devices[r] (default device + r); every
  // call below then acts on the whole map exactly as on one GPU (sm_create_group).  ngpus = 0 reads the environment:
  // SM_GPUS=N, and SM_GPU_DEVICES=0,0 for a device list (equal entries: ranks sharing a GPU).  0 or 1: one context.
  Layermap(int SEED, ivec2 _dim, int SCALE = 80, int device = 0, int ngpus = 0, const int* devices = nullptr) {
    pool.reserve(256); open(_dim, SCALE, device, ngpus, devices); initialize(SEED, _dim);
  }
  template <class VP> Layermap(int SEED, ivec2 _dim, VP&, int SCALE = 80, int device = 0, int ngpus = 0,
                               const int* devices = nullptr) : Layermap(SEED, _dim, SCALE, device, ngpus, devices) {}
  ~Layermap() { if (ctx) sm_destroy(ctx); }
  Layermap(const Layermap&) = delete;

  void initialize(int SEED, ivec2 _dim) {                   // layermap.h:163-216
    if (_dim.x != dim.x || _dim.y != dim.y) throw Error(SM_ERR_INVALID, "Layermap::initialize: size is fixed at construction");
    push_tables();
    std::vector<sm_layer> L;
    for (auto& l : layers) L.push_back(sm_layer{(int32_t)l.type, l.min, l.bias, l.scale, l.octaves, l.lacunarity, l.gain, l.frequency});
    touch();
    ck(sm_initialize(ctx, SEED, L.data(), (int32_t)L.size()));
  }
  // ---- per-cell reads (legacy call sites: GUI picking, custom initialisation) -------------------------------
  // A handful of reads between two mutations go to the device one cell at a time (one tiny kernel each).  Code
  // that reads many cells - a loop over the map - gets a HOST MIRROR instead: after kMirrorAfter single reads the
  // height and surface fields are downloaded once and served from host memory until the next call that
  // changes the map marks them dirty.
  static constexpr int kMirrorAfter = 64;
  double height(ivec2 p) {                                   // :422
    if (mirror_ready()) return h_height[(size_t)p.x * dim.y + p.y];
    double h; ck(sm_cell_query(ctx, p.x, p.y, &h, nullptr, nullptr)); return h;
  }
  double height(vec2 p) { double h; ck(sm_height_bilinear(ctx, p.x, p.y, &h)); return h; }                  // :427
  vec3 normal(ivec2 p) { float n[3]; ck(sm_cell_query(ctx, p.x, p.y, nullptr, nullptr, n)); return vec3{n[0], n[1], n[2]}; }  // :341
  template <class VP> vec3 normal(ivec2 p, VP&) { return normal(p); }
  vec3 normal(vec2 pos) {                                    // :379-390 (weights cross-wired exactly as upstream)
    const float fx = std::floor(pos.x), fy = std::floor(pos.y);
    const ivec2 p((int)fx, (int)fy);
    const float wx = pos.x - fx, wy = pos.y - fy;
    vec3 n{0.f, 0.f, 0.f};
    auto acc = [&](float w, ivec2 q) { const vec3 m = normal(q); n.x += w * m.x; n.y += w * m.y; n.z += w * m.z; };
    acc((1.0f - wx) * (1.0f - wy), p);
    acc((1.0f - wx) * wy, ivec2(p.x + 1, p.y));
    acc(wx * (1.0f - wy), ivec2(p.x, p.y + 1));
    acc(wx * wy, ivec2(p.x + 1, p.y + 1));
    return n;
  }
  SurfType surface(ivec2 p) {                                // :417
    if (mirror_ready()) return (SurfType)h_surface[(size_t)p.x * dim.y + p.y];
    int32_t s; ck(sm_cell_query(ctx, p.x, p.y, nullptr, &s, nullptr)); return (SurfType)s;
  }
  // Layermap::top(ivec2), layermap.h:150-152: the top section of a column; ->prev walks down.  The sections
  // are host COPIES (valid until the next top() call); the columns themselves live on the device.
  sec* top(ivec2 p) {
    int32_t n = 0;
    std::vector<int32_t> t(64); std::vector<double> sz(64), fl(64), sa(64);
    ck(sm_cell_column(ctx, p.x, p.y, 64, &n, t.data(), sz.data(), fl.data(), sa.data()));
    if (n > 64) {
      t.resize(n); sz.resize(n); fl.resize(n); sa.resize(n);
      ck(sm_cell_column(ctx, p.x, p.y, n, &n, t.data(), sz.data(), fl.data(), sa.data()));
    }
    column_copy.assign((size_t)n, sec());
    for (int i = 0; i < n; i++) {                            // bottom -> top
      sec& e = column_copy[(size_t)i];
      e.type = (SurfType)t[i]; e.size = sz[i]; e.floor = fl[i]; e.saturation = sa[i];
      e.prev = i > 0 ? &column_copy[(size_t)i - 1] : nullptr;
      e.next = i + 1 < n ? &column_copy[(size_t)i + 1] : nullptr;
    }
    return n ? &column_copy[(size_t)n - 1] : nullptr;
  }
  void add(ivec2 p, sec* E) {                               // :230 (E is consumed, as upstream)
    if (!E) return;
    touch();
    ck(sm_cell_add(ctx, p.x, p.y, E->size, (int32_t)E->type));
    pool.unget(E);
  }
  double remove(ivec2 p, double h) { double d; touch(); ck(sm_cell_remove(ctx, p.x, p.y, h, &d)); return d; }   // :310
  // add() / a full strip over remove() on every cell in one call (sm_apply_layer): delta[x*dim.y + y] > 0 deposits that
  // much of `type`, < 0 strips that much height, +-0.0 leaves the cell alone; leftover (may be null) gets the height each
  // strip could not take.  All or nothing: a refused raster throws with the map unchanged.
  void apply(const double* delta, SurfType type, double* leftover = nullptr) {
    touch();
    ck(sm_apply_layer(ctx, delta, (int32_t)type, leftover, 0, 0, nullptr));
  }
  // Particle::cascade (particle.h:24-101) at every cell, pass after pass in sm_relax's phase order, until a pass
  // changes nothing or max_passes passes have run.  A refused call (transferloop outside 0..3, max_passes < 1) throws
  // with the map unchanged.
  sm_relax_stats relax(int max_passes, int transferloop = 0) {
    sm_relax_stats st = {};
    touch();
    ck(sm_relax(ctx, max_passes, transferloop, &st));
    return st;
  }
  // What lies under the surface, per cell, in one read-only call (sm_composition): for every type of `types`, the
  // thickness of that soil inside the height window [lo, hi] (flags SM_COMP_BELOW_SURFACE: measured down from the
  // surface; SM_COMP_PORE_WATER: the pore water it holds there).  Planar: out[i*dim.x*dim.y + x*dim.y + y].
  std::vector<double> composition(const std::vector<SurfType>& types, double lo, double hi, int flags = 0) {
    std::vector<int32_t> t(types.begin(), types.end());
    std::vector<double> out(t.size() * (size_t)dim.x * (size_t)dim.y);
    ck(sm_composition(ctx, t.data(), (int32_t)t.size(), lo, hi, flags, out.data(), 0, nullptr));
    return out;
  }
  // The soil type at the heights z0 + k*dz, k < nz, of every cell of [lo.x, hi.x) x [lo.y, hi.y) (sm_voxelize): the
  // first section met top -> bottom that contains the height, SM_VOXEL_NONE where none does.  Planar:
  // out[k*W + (x - lo.x)*(hi.y - lo.y) + (y - lo.y)], W the window's cells.
  std::vector<uint8_t> voxels(ivec2 lo, ivec2 hi, double z0, double dz, int nz) {
    std::vector<uint8_t> out((size_t)std::max(nz, 0) * (size_t)std::max(hi.x - lo.x, 0) * (size_t)std::max(hi.y - lo.y, 0));
    ck(sm_voxelize(ctx, lo.x, hi.x, lo.y, hi.y, z0, dz, nz, out.data(), 0, nullptr));
    return out;
  }

  // ---- meshing (layermap.h:443-555) --------------------------------------------------------------------------
  // The renderer's vertex pool is outside the boundary; what crosses it is the vertex data.  update(vp) meshes
  // the whole map on the device (one 44-byte Vertex {position[3], normal[3], color[4], index} per cell, cell order
  // x*dim.y + y, cut at the slice plane) into `vertices`, and hands it to the pool if the pool type offers
  // upload(const float*, size_t nvertices).  update(ivec2, vp) - upstream's per-cell refresh after every column
  // change - only has to mark the mesh stale: the next update(vp)/meshpool(vp)/slice(vp, s) rebuilds all of it
  // in one bandwidth-bound pass.
  std::vector<float> vertices;
  int slice_plane = 160;                                     // SLICE = 2*SCALE (SoilMachine.cpp:12)
  bool mesh_stale = true;
  template <class VP> void meshpool(VP& vp) { update(vp); }                                                  // :443-473
  template <class VP> void update(ivec2, VP&) { mesh_stale = true; }                                         // :475-549
  template <class VP> void update(VP& vp) {                                                                  // :551-555
    vertices.resize((size_t)dim.x * dim.y * 11);
    ck(sm_mesh_update(ctx, slice_plane, vertices.data()));
    mesh_stale = false;
    upload_if_possible(vp, 0);
  }
  template <class VP> void slice(VP& vp, double s) { slice_plane = (int)s; update(vp); }                     // :557-
  template <class VP> void slice(VP& vp) { update(vp); }

  // ---- snapshots (what io.h:232 asks for: "Should be able to also WRITE to file!!") -------------------------------
  // save() writes the snapshot of the whole map - columns and frequency arrays, format in soilmachine_b200.h - to a
  // file; load() restores it, on one GPU or several, whichever wrote it.  The soil table must be the one of the saving
  // run (loadsoil of the same file).  The application keeps its own rand() stream, as upstream does.
  void save(const std::string& path) {
    int64_t n = 0;
    ck(sm_snapshot_bytes(ctx, &n));
    std::vector<unsigned char> buf((size_t)n);
    ck(sm_snapshot_save(ctx, buf.data(), n, 0));
    std::FILE* f = std::fopen(path.c_str(), "wb");
    if (!f) throw Error(SM_ERR_INVALID, "Layermap::save: cannot open " + path);
    const size_t w = std::fwrite(buf.data(), 1, buf.size(), f);
    if (std::fclose(f) != 0 || w != buf.size()) throw Error(SM_ERR_INVALID, "Layermap::save: cannot write " + path);
  }
  void load(const std::string& path) {
    std::FILE* f = std::fopen(path.c_str(), "rb");
    if (!f) throw Error(SM_ERR_INVALID, "Layermap::load: cannot open " + path);
    std::vector<unsigned char> buf;
    unsigned char chunk[1 << 16];
    for (size_t r; (r = std::fread(chunk, 1, sizeof(chunk), f)) > 0;) buf.insert(buf.end(), chunk, chunk + r);
    std::fclose(f);
    push_tables();
    touch();
    const int rc = sm_snapshot_restore(ctx, buf.data(), (int64_t)buf.size(), 0);
    if (rc != SM_OK) throw Error(rc, sm_last_error(ctx));
  }

  // every call that may change columns goes through here
  void touch() { mirror_valid = false; mirror_reads = 0; mesh_stale = true; }

  // A full section pool is not fatal upstream: secpool::get prints and returns NULL, add() drops the section
  // (layermap.h:92-95,232-234) and the program keeps running.  Same here: the drop is reported, the call
  // counts it in stats.pool_drops, and the status is per call.
  void ck(int rc) const {
    if (rc == SM_ERR_POOL) { std::fprintf(stderr, "Memory Pool Out-Of-Elements (%s)\n", sm_last_error(ctx)); return; }
    if (rc != SM_OK) throw Error(rc, sm_last_error(ctx));
  }
  void push_tables() {
    std::vector<sm_soil> t;
    for (auto& s : soils) t.push_back(sm_soil{(int32_t)s.transports, (int32_t)s.erodes, (int32_t)s.cascades, (int32_t)s.abrades,
                                              s.density, s.porosity, s.solubility, s.equrate, s.friction, s.erosionrate,
                                              s.maxdiff, s.settling, s.suspension, s.abrasion});
    ck(sm_set_soils(ctx, t.data(), (int32_t)t.size()));
    std::vector<float> col;
    for (auto& sp : soils) { col.push_back(sp.color.x); col.push_back(sp.color.y); col.push_back(sp.color.z); col.push_back(sp.color.w); }
    ck(sm_set_soil_colors(ctx, col.data(), (int32_t)soils.size()));
  }
 private:
  std::vector<double> h_height; std::vector<int32_t> h_surface; std::vector<sec> column_copy;
  bool mirror_valid = false; int mirror_reads = 0;
  bool mirror_ready() {
    if (mirror_valid) return true;
    if (++mirror_reads <= kMirrorAfter) return false;
    h_height.resize((size_t)dim.x * dim.y); h_surface.resize((size_t)dim.x * dim.y);
    ck(sm_download_height(ctx, h_height.data()));
    ck(sm_download_surface(ctx, h_surface.data()));
    return mirror_valid = true;
  }
  template <class VP> auto upload_if_possible(VP& vp, int) -> decltype(vp.upload((const float*)nullptr, (size_t)0), void()) {
    vp.upload(vertices.data(), (size_t)dim.x * dim.y);
  }
  template <class VP> void upload_if_possible(VP&, long) {}
  void open(ivec2 _dim, int SCALE, int device, int ngpus = 0, const int* devices = nullptr) {
    dim = _dim;
    sm_config cfg{dim.x, dim.y, SCALE, device, 0, 0, 0};
    std::vector<int32_t> devs;
    if (ngpus <= 0) {
      const char* e = std::getenv("SM_GPUS");
      ngpus = e ? std::atoi(e) : 1;
      if (const char* l = std::getenv("SM_GPU_DEVICES"))
        for (const char* q = l; *q;) {
          char* end = nullptr;
          const long v = std::strtol(q, &end, 10);
          if (end == q) break;
          devs.push_back((int32_t)v);
          q = (*end == ',') ? end + 1 : end;
        }
    } else if (devices) {
      devs.assign(devices, devices + ngpus);
    }
    int rc;
    if (ngpus <= 1) {
      rc = sm_create(&cfg, &ctx);
    } else {
      if (devs.empty()) for (int r = 0; r < ngpus; r++) devs.push_back(device + r);
      if ((int)devs.size() != ngpus) throw Error(SM_ERR_INVALID, "Layermap: one device per GPU rank (SM_GPU_DEVICES)");
      rc = sm_create_group(&cfg, ngpus, devs.data(), &ctx);
    }
    if (rc != SM_OK) throw Error(rc, sm_last_error(nullptr));
  }
};

// particle.h:11-103
struct Particle {
  vec2 pos; vec2 speed; bool isalive = true;
  template <class VP> static void cascade(vec2 p, Layermap& map, VP&, int transferloop = 0) {               // particle.h:24
    map.touch();
    map.ck(sm_cell_cascade(map.ctx, p.x, p.y, transferloop));
  }
};

namespace detail {
// spawn positions exactly as the particle constructors draw them (water.h:13, wind.h:15: GCC evaluates
// the two rand() arguments right to left, so y takes the first draw)
inline std::vector<float> spawn(const Layermap& map, int n) {
  std::vector<float> xy((size_t)n * 2);
  for (int i = 0; i < n; i++) { int y = rand() % map.dim.y; int x = rand() % map.dim.x; xy[2 * i] = (float)x; xy[2 * i + 1] = (float)y; }
  return xy;
}
// Upstream's water-table cascade constructs every nested particle with `WaterParticle particle(map)`
// (water.h:243), which draws two rand() values for a position that is overwritten right away.  The device never
// needs them, but an application that seeds rand() expects the same stream afterwards: consume them here.
inline void nested_ctor_draws(int64_t nested) { for (int64_t i = 0; i < 2 * nested; i++) (void)rand(); }
}  // namespace detail

// water.h:9-373 -- the batch entry point replaces the loop SoilMachine.cpp:288-298
struct WaterParticle : Particle {
  // Host mirrors of the device maps, indexed [y*dim.x + x] as upstream (water.h:345-346).  They exist only
  // after init(dimx, dimy) (upstream: init() allocates them, water.h:21-24) and are refreshed by
  // mapfrequency() / resetfrequency(), i.e. exactly where the reference frame loop reads them
  // (SoilMachine.cpp:314-319).  A headless loop that never calls init(...) pays no download.
  inline static float* frequency = nullptr;
  inline static float* track = nullptr;
  inline static double volumeFactor = 0.015;                  // water.h:33,368: a mutable static, passed to the device
  static void init() {}                                       // maps live on the device; no host mirror
  static void init(int dimx, int dimy) {
    delete[] frequency; delete[] track;
    frequency = new float[(size_t)dimx * dimy]();
    track = new float[(size_t)dimx * dimy]();
  }

  // ---- the reference's per-particle interface (water.h:11-19,43,75,123): the loop SoilMachine.cpp:288-298 compiles
  // unchanged against it.  Each particle is a batch of ONE on the device - a kernel launch and a read-back per
  // step - so this is the slow, source-compatible path; run() below is the same loop as one batch.
  double volume = 1.0, sediment = 0.0;
  int spill = 3;
  ivec2 ipos;
  SurfType contains = 0;
  explicit WaterParticle(Layermap& map) {                     // water.h:11-19
    map.push_tables();
    const std::vector<float> xy = detail::spawn(map, 1);
    map.touch();
    map.ck(sm_water_begin(map.ctx, 1, xy.data()));
    refresh(map);
  }
  // move() runs the whole particle-step (move && interact are one fused step on the device) and remembers
  // how it ended; interact() reports it.  `while (p.move(..) && p.interact(..));` therefore behaves as upstream:
  // move() is false when the particle stalled or left the map (water.h:56-57,65-69), interact() is false when
  // it evaporated (water.h:119).
  template <class VP> bool move(Layermap& map, VP&) {
    sm_stats st{};
    map.touch();
    map.ck(sm_water_sweeps(map.ctx, 1, &st));
    refresh(map);
    survived = st.alive > 0;
    return st.steps > 0;
  }
  template <class VP> bool interact(Layermap&, VP&) { return survived; }
  template <class VP> bool flood(Layermap& map, VP&) {        // water.h:123-145 (always returns false)
    map.touch();
    map.ck(sm_set_volume_factor(map.ctx, volumeFactor));
    sm_hydro_stats st{};
    map.ck(sm_water_flood(map.ctx, &st));
    detail::nested_ctor_draws(st.nested);
    return false;
  }
  // static WaterParticle::cascade(vec2, ..., spill) / seep(vec2, ...) for one cell (water.h:151,285)
  template <class VP> static void cascade(vec2 p, Layermap& map, VP&, int spill_ = 0) {
    map.touch();
    map.ck(sm_set_volume_factor(map.ctx, volumeFactor));
    map.ck(sm_cell_water_cascade(map.ctx, (int)p.x, (int)p.y, spill_));      // ivec2 ipos = pos truncates (:153)
  }
  template <class VP> static void seep(vec2 p, Layermap& map, VP&) {
    map.touch();
    map.ck(sm_cell_seep(map.ctx, (int)p.x, (int)p.y));
  }

  // ---- the batch entry points ------------------------------------------------------------------------------------
  WaterParticle() {}
  template <class VP> static sm_stats run(Layermap& map, VP&, int NWATER) {
    map.push_tables();                                        // upstream reads soils[] live (GUI sliders, :165-200)
    std::vector<float> xy = detail::spawn(map, NWATER);
    sm_stats st{};
    map.touch();
    map.ck(sm_water_run(map.ctx, NWATER, xy.data(), 0, &st));
    return st;
  }
  // The flood tail of the per-particle loop (SoilMachine.cpp:292-296, water.h:123-145) for the whole batch:
  // every finished particle of the last run() floods, in ascending particle index.
  template <class VP> static sm_hydro_stats flood_batch(Layermap& map, VP&) {
    sm_hydro_stats st{};
    map.touch();
    map.ck(sm_set_volume_factor(map.ctx, volumeFactor));
    map.ck(sm_water_flood(map.ctx, &st));
    detail::nested_ctor_draws(st.nested);
    return st;
  }
  // A batch whose particles flood at the end of the sweep they stop in (sm_water_run_flooding): later sweeps meet the
  // batch's own ponds, closer to upstream's per-particle flood (SoilMachine.cpp:290-297) than run() + flood_batch().
  template <class VP> static std::pair<sm_stats, sm_hydro_stats> run_flooding(Layermap& map, VP&, int NWATER) {
    map.push_tables();
    std::vector<float> xy = detail::spawn(map, NWATER);
    sm_stats st{};
    sm_hydro_stats hs{};
    map.touch();
    map.ck(sm_set_volume_factor(map.ctx, volumeFactor));
    map.ck(sm_water_run_flooding(map.ctx, NWATER, xy.data(), 0, &st, &hs));
    detail::nested_ctor_draws(hs.nested);
    return {st, hs};
  }
  // WaterParticle::seep(map, vertexpool), water.h:335-343 / SoilMachine.cpp:300-301
  template <class VP> static sm_hydro_stats seep(Layermap& map, VP&) {
    sm_hydro_stats st{};
    map.touch();
    map.ck(sm_set_volume_factor(map.ctx, volumeFactor));
    map.ck(sm_seep(map.ctx, &st));
    detail::nested_ctor_draws(st.nested);
    return st;
  }
  // water.h:358-365 + 353-356 fused on the device: frequency <- blend(track), track <- 0
  static void mapfrequency(Layermap& map) {
    map.ck(sm_frequency_update(map.ctx));
    if (frequency) map.ck(sm_get_frequency(map.ctx, frequency, track, nullptr));
  }
  static void resetfrequency(Layermap&) {}                                            // water.h:353-356 (done above)
  static std::vector<float> download_frequency(Layermap& map) {                       // water.h:345
    std::vector<float> f((size_t)map.dim.x * map.dim.y);
    map.ck(sm_get_frequency(map.ctx, f.data(), nullptr, nullptr));
    return f;
  }
 private:
  bool survived = true;
  void refresh(Layermap& map) {
    float p2[2], s2[2]; double v, sed; int32_t c, al;
    map.ck(sm_water_state(map.ctx, p2, s2, &v, &sed, &c, &al));
    pos = vec2(p2[0], p2[1]); speed = vec2(s2[0], s2[1]); volume = v; sediment = sed; contains = (SurfType)c;
    isalive = al != 0;
    ipos = ivec2((int)std::round(pos.x), (int)std::round(pos.y));
  }
};
// wind.h:11-140 -- the batch entry point replaces the loop SoilMachine.cpp:304-307
struct WindParticle : Particle {
  inline static float* frequency = nullptr;                   // wind.h:48; refreshed at the end of run()
  static void init() {}
  static void init(int dimx, int dimy) { delete[] frequency; frequency = new float[(size_t)dimx * dimy](); }

  // per-particle interface (wind.h:13-22,54,94), see WaterParticle
  vec3 speed{-2.f, 0.f, 1.f};                                 // shadows Particle::speed, as upstream (wind.h:29)
  double sediment = 0.0, height = 0.0;
  ivec2 ipos;
  SurfType contains = 0;
  explicit WindParticle(Layermap& map) {
    map.push_tables();
    const std::vector<float> xy = detail::spawn(map, 1);
    map.touch();
    map.ck(sm_wind_begin(map.ctx, 1, xy.data()));
    refresh(map);
  }
  template <class VP> bool move(Layermap& map, VP&) {         // false: the particle died in move() (wind.h:56,83-88)
    sm_stats st{};
    map.touch();
    map.ck(sm_wind_sweeps(map.ctx, 1, &st));
    refresh(map);
    return st.steps > 0;
  }
  template <class VP> bool interact(Layermap&, VP&) { return true; }   // wind.h:94-136 always returns true

  WindParticle() {}
  template <class VP> static sm_stats run(Layermap& map, VP&, int NWIND) {
    map.push_tables();
    std::vector<float> xy = detail::spawn(map, NWIND);
    sm_stats st{};
    map.touch();
    map.ck(sm_wind_run(map.ctx, NWIND, xy.data(), 0, &st));
    if (frequency) map.ck(sm_get_frequency(map.ctx, nullptr, nullptr, frequency));
    return st;
  }
  static std::vector<float> download_frequency(Layermap& map) {                       // wind.h:48
    std::vector<float> f((size_t)map.dim.x * map.dim.y);
    map.ck(sm_get_frequency(map.ctx, nullptr, nullptr, f.data()));
    return f;
  }
 private:
  void refresh(Layermap& map) {
    float p2[2], s3[3]; double h, sed; int32_t c, al;
    map.ck(sm_wind_state(map.ctx, p2, s3, &h, &sed, &c, &al));
    pos = vec2(p2[0], p2[1]); speed = vec3{s3[0], s3[1], s3[2]}; height = h; sediment = sed; contains = (SurfType)c;
    isalive = al != 0;
    ipos = ivec2((int)std::round(pos.x), (int)std::round(pos.y));
  }
};

}  // namespace soilmachine
