// tests/facade_drainage.cpp -- Layermap::drainage of the C++ facade after two of the reference's frames (water batch,
// its floods, the seep pass, wind batch, frequency update).  Run with SM_GPUS / SM_GPU_DEVICES to use a group.
//   facade_drainage <file.soil> <snapshot> <out>
// Saves the map's snapshot, then writes to <out>, one after the other: spill (f64), dir (i8), area (i64) and basin
// (i64) of the top of the columns, then the same four of the ground under standing water.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include "../include/soilmachine/soilmachine.hpp"
using namespace soilmachine;

int SIZEX = 96, SIZEY = 72, SCALE = 80, SEED = 29;
struct DummyVertexpool {} vertexpool;

int main(int argc, char** argv) {
  if (argc < 4) { printf("usage: facade_drainage file.soil snapshot out\n"); return 2; }
  try {
    WorldEntry w = loadsoil(argv[1]);
    SCALE = w.scale;
    srand(SEED);
    Layermap map(SEED, ivec2(SIZEX, SIZEY), vertexpool, SCALE);
    for (int i = 0; i < 2; i++) {
      WaterParticle::run(map, vertexpool, 700);
      WaterParticle::flood_batch(map, vertexpool);
      WaterParticle::seep(map, vertexpool);
      WindParticle::run(map, vertexpool, 200);
      WaterParticle::mapfrequency(map);
    }
    map.save(argv[2]);
    FILE* f = fopen(argv[3], "wb");
    if (!f) { printf("cannot write %s\n", argv[3]); return 2; }
    int64_t total = 0;
    for (int ground = 0; ground < 2; ground++) {
      const Layermap::Drainage d = map.drainage(ground != 0);
      fwrite(d.spill.data(), 8, d.spill.size(), f);
      fwrite(d.dir.data(), 1, d.dir.size(), f);
      fwrite(d.area.data(), 8, d.area.size(), f);
      fwrite(d.basin.data(), 8, d.basin.size(), f);
      for (size_t i = 0; i < d.area.size(); i++)
        if (d.dir[i] < 0) total += d.area[i];
    }
    fclose(f);
    printf("cells %d outlet area %lld\n", SIZEX * SIZEY, (long long)total);
    if (total != 2LL * SIZEX * SIZEY) { printf("the outlets' areas do not sum to the map\n"); return 1; }
  } catch (const Error& e) {
    printf("soilmachine error %d: %s\n", e.code, e.what());
    return e.code == SM_ERR_NOGPU ? 77 : 1;
  } catch (const SoilFileError& e) { printf("%s\n", e.what()); return 2; }
  return 0;
}
