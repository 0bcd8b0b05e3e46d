// tests/facade_apply.cpp -- Layermap::apply of the C++ facade: one layer raster over the whole map after two of the
// reference's frames (water batch, its floods, the seep pass, wind batch, frequency update).  Run with SM_GPUS /
// SM_GPU_DEVICES to use a group.
//   facade_apply <file.soil> <raster> <type> <before> <after>
// <raster>: SIZEX*SIZEY f64, cell order x*SIZEY + y.  Saves the snapshot of the map before and after the raster and
// prints the column checksum after it and the number of cells whose strip ran out of column.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include "../include/soilmachine/soilmachine.hpp"
using namespace soilmachine;

int SIZEX = 96, SIZEY = 72, SCALE = 80, SEED = 23;
struct DummyVertexpool {} vertexpool;

int main(int argc, char** argv) {
  if (argc < 6) { printf("usage: facade_apply file.soil raster type before after\n"); return 2; }
  try {
    WorldEntry w = loadsoil(argv[1]);
    SCALE = w.scale;
    std::vector<double> delta((size_t)SIZEX * SIZEY), left(delta.size());
    FILE* f = fopen(argv[2], "rb");
    if (!f || fread(delta.data(), 8, delta.size(), f) != delta.size()) { printf("cannot read %s\n", argv[2]); return 2; }
    fclose(f);
    srand(SEED);
    Layermap map(SEED, ivec2(SIZEX, SIZEY), vertexpool, SCALE);
    for (int i = 0; i < 2; i++) {
      WaterParticle::run(map, vertexpool, 700);
      WaterParticle::flood_batch(map, vertexpool);
      WaterParticle::seep(map, vertexpool);
      WindParticle::run(map, vertexpool, 200);
      WaterParticle::mapfrequency(map);
    }
    map.save(argv[4]);
    map.apply(delta.data(), (SurfType)atoi(argv[3]), left.data());
    map.save(argv[5]);
    uint64_t c = 0;
    map.ck(sm_checksum(map.ctx, &c));
    int emptied = 0;
    for (double l : left) emptied += l > 0;
    printf("checksum %016llx emptied %d\n", (unsigned long long)c, emptied);
  } catch (const Error& e) {
    printf("soilmachine error %d: %s\n", e.code, e.what());
    return e.code == SM_ERR_NOGPU ? 77 : 1;
  } catch (const SoilFileError& e) { printf("%s\n", e.what()); return 2; }
  return 0;
}
