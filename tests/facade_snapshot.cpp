// tests/facade_snapshot.cpp -- Layermap::save / Layermap::load of the C++ facade.  Frames are the reference's: water
// batch, its floods, the seep pass, wind batch, frequency update.  Run with SM_GPUS / SM_GPU_DEVICES to use a group.
//   facade_snapshot <file.soil> save <snap> <final>   frames 1-2, save <snap>, frames 3-4, save <final>; then load
//                                                     <snap>, frames 3-4 again: prints "resume identical" when the
//                                                     checksum and the final snapshot are the same both times
//   facade_snapshot <file.soil> load <snap> <final>   load <snap> (written by any run), frames 3-4, save <final>
// Frames 3-4 draw their spawn lists after srand(SEED + 1), so every run draws the same ones.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "../include/soilmachine/soilmachine.hpp"
using namespace soilmachine;

int SIZEX = 96, SIZEY = 72, SCALE = 80, SEED = 23;
struct DummyVertexpool {} vertexpool;

static void frame(Layermap& map) {
  WaterParticle::run(map, vertexpool, 700);
  WaterParticle::flood_batch(map, vertexpool);
  WaterParticle::seep(map, vertexpool);
  WindParticle::run(map, vertexpool, 200);
  WaterParticle::mapfrequency(map);
}
static uint64_t checksum(Layermap& map) {
  uint64_t c = 0;
  map.ck(sm_checksum(map.ctx, &c));
  return c;
}
static std::string slurp(const std::string& p) {
  std::string s;
  if (FILE* f = fopen(p.c_str(), "rb")) {
    char b[1 << 16];
    for (size_t r; (r = fread(b, 1, sizeof(b), f)) > 0;) s.append(b, r);
    fclose(f);
  }
  return s;
}

int main(int argc, char** argv) {
  if (argc < 5) { printf("usage: facade_snapshot file.soil save|load snap final\n"); return 2; }
  try {
    WorldEntry w = loadsoil(argv[1]);
    SCALE = w.scale;
    const std::string mode = argv[2], snap = argv[3], fin = argv[4];
    srand(SEED);
    Layermap map(SEED, ivec2(SIZEX, SIZEY), vertexpool, SCALE);
    if (mode == "save") {
      frame(map); frame(map);
      map.save(snap);
      srand(SEED + 1);
      frame(map); frame(map);
      const uint64_t a = checksum(map);
      map.save(fin);
      const std::string first = slurp(fin);
      map.load(snap);
      srand(SEED + 1);
      frame(map); frame(map);
      const uint64_t b = checksum(map);
      map.save(fin);
      const bool same = a == b && first == slurp(fin) && !first.empty();
      printf("%s: checksum %016llx / %016llx\n", same ? "resume identical" : "resume DIFFERS", (unsigned long long)a,
             (unsigned long long)b);
      return same ? 0 : 1;
    }
    map.load(snap);
    srand(SEED + 1);
    frame(map); frame(map);
    map.save(fin);
    printf("loaded %s: checksum %016llx\n", snap.c_str(), (unsigned long long)checksum(map));
  } catch (const Error& e) {
    printf("soilmachine error %d: %s\n", e.code, e.what());
    return e.code == SM_ERR_NOGPU ? 77 : 1;
  } catch (const SoilFileError& e) { printf("%s\n", e.what()); return 2; }
  return 0;
}
