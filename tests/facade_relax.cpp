// tests/facade_relax.cpp -- Layermap::relax of the C++ facade: slope relaxation over the whole map after one of the
// reference's frames (water batch, its floods, the seep pass, wind batch, frequency update).  Run with SM_GPUS /
// SM_GPU_DEVICES to use a group.
//   facade_relax <file.soil> <transferloop> <before>
// Saves the snapshot of the map before the relaxation, runs up to 5 passes and prints the column checksum and stats.
#include <cstdio>
#include <cstdlib>
#include "../include/soilmachine/soilmachine.hpp"
using namespace soilmachine;

int SIZEX = 96, SIZEY = 72, SCALE = 80, SEED = 23;
struct DummyVertexpool {} vertexpool;

int main(int argc, char** argv) {
  if (argc < 4) { printf("usage: facade_relax file.soil transferloop before\n"); return 2; }
  try {
    WorldEntry w = loadsoil(argv[1]);
    SCALE = w.scale;
    srand(SEED);
    Layermap map(SEED, ivec2(SIZEX, SIZEY), vertexpool, SCALE);
    WaterParticle::run(map, vertexpool, 700);
    WaterParticle::flood_batch(map, vertexpool);
    WaterParticle::seep(map, vertexpool);
    WindParticle::run(map, vertexpool, 200);
    WaterParticle::mapfrequency(map);
    map.save(argv[3]);
    const sm_relax_stats st = map.relax(5, atoi(argv[2]));
    uint64_t c = 0;
    map.ck(sm_checksum(map.ctx, &c));
    printf("checksum %016llx passes %lld visits %lld transfers %lld\n", (unsigned long long)c, (long long)st.passes,
           (long long)st.visits, (long long)st.transfers);
    bool refused = false;
    try { map.relax(0); } catch (const Error& e) { refused = e.code == SM_ERR_INVALID; }
    if (!refused) { printf("relax(0) was not refused\n"); return 1; }
  } catch (const Error& e) {
    printf("soilmachine error %d: %s\n", e.code, e.what());
    return e.code == SM_ERR_NOGPU ? 77 : 1;
  } catch (const SoilFileError& e) { printf("%s\n", e.what()); return 2; }
  return 0;
}
