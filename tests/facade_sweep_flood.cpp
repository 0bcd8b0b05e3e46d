// tests/facade_sweep_flood.cpp -- WaterParticle::run_flooding of the C++ facade: one frame whose water batch floods
// its particles at the end of the sweep they stop in, then the seep pass and a wind batch.
//   facade_sweep_flood <file.soil>
// Prints the column checksum and the batch's and the floods' counters.
#include <cstdio>
#include <cstdlib>
#include "../include/soilmachine/soilmachine.hpp"
using namespace soilmachine;

int SIZEX = 64, SIZEY = 48, SCALE = 80, SEED = 11;
struct DummyVertexpool {} vertexpool;

int main(int argc, char** argv) {
  if (argc < 2) { printf("usage: facade_sweep_flood file.soil\n"); return 2; }
  try {
    WorldEntry w = loadsoil(argv[1]);
    SCALE = w.scale;
    srand(SEED);
    Layermap map(SEED, ivec2(SIZEX, SIZEY), vertexpool, SCALE);
    const auto r = WaterParticle::run_flooding(map, vertexpool, 600);
    WaterParticle::seep(map, vertexpool);
    WindParticle::run(map, vertexpool, 100);
    WaterParticle::mapfrequency(map);
    uint64_t c = 0;
    map.ck(sm_checksum(map.ctx, &c));
    printf("checksum %016llx steps %lld sweeps %lld floods %lld nested %lld next %d\n", (unsigned long long)c,
           (long long)r.first.steps, (long long)r.first.sweeps, (long long)r.second.floods, (long long)r.second.nested,
           rand());
  } catch (const Error& e) {
    printf("soilmachine error %d: %s\n", e.code, e.what());
    return e.code == SM_ERR_NOGPU ? 77 : 1;
  } catch (const SoilFileError& e) { printf("%s\n", e.what()); return 2; }
  return 0;
}
