// tests/facade_strata.cpp -- Layermap::composition and Layermap::voxels of the C++ facade after two of the reference's
// frames (water batch, its floods, the seep pass, wind batch, frequency update).  Run with SM_GPUS / SM_GPU_DEVICES to
// use a group.
//   facade_strata <file.soil> <snapshot> <out>
// Saves the map's snapshot, then writes to <out>, one after the other: the composition of every soil over the whole
// column (f64), the pore water of every soil in the top 1.0 below the surface (f64), the voxels of the whole map at
// z = -0.25 + k/8, k < 48 (u8), and the strata section of row y = 17 at z = k/64, k < 256 (u8).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include "../include/soilmachine/soilmachine.hpp"
using namespace soilmachine;

int SIZEX = 96, SIZEY = 72, SCALE = 80, SEED = 23;
struct DummyVertexpool {} vertexpool;

int main(int argc, char** argv) {
  if (argc < 4) { printf("usage: facade_strata file.soil snapshot out\n"); return 2; }
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
    std::vector<SurfType> all;
    for (size_t t = 0; t < soils.size(); t++) all.push_back(t);
    const std::vector<double> comp = map.composition(all, -INFINITY, INFINITY);
    const std::vector<double> pore = map.composition(all, 0.0, 1.0, SM_COMP_BELOW_SURFACE | SM_COMP_PORE_WATER);
    const std::vector<uint8_t> vox = map.voxels(ivec2(0, 0), ivec2(SIZEX, SIZEY), -0.25, 0.125, 48);
    const std::vector<uint8_t> row = map.voxels(ivec2(0, 17), ivec2(SIZEX, 18), 0.0, 1.0 / 64, 256);
    FILE* f = fopen(argv[3], "wb");
    if (!f) { printf("cannot write %s\n", argv[3]); return 2; }
    fwrite(comp.data(), 8, comp.size(), f);
    fwrite(pore.data(), 8, pore.size(), f);
    fwrite(vox.data(), 1, vox.size(), f);
    fwrite(row.data(), 1, row.size(), f);
    fclose(f);
    printf("soils %zu cells %d\n", all.size(), SIZEX * SIZEY);
  } catch (const Error& e) {
    printf("soilmachine error %d: %s\n", e.code, e.what());
    return e.code == SM_ERR_NOGPU ? 77 : 1;
  } catch (const SoilFileError& e) { printf("%s\n", e.what()); return 2; }
  return 0;
}
