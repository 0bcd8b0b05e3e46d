// tests/facade_group.cpp -- the facade's legacy per-cell calls (map.add, map.remove, Particle::cascade,
// WaterParticle::seep(vec2), WaterParticle::cascade(vec2)) across a strip boundary of a Layermap created over several
// GPU ranks by its constructor argument.  Writes every column to a file; run with ngpus = 1 it writes what one context
// computes, and the two files must be equal (tests/test_group.py).
//   facade_group <file.soil> <ngpus> <out.bin>       (ranks share device 0)
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../include/soilmachine/soilmachine.hpp"
using namespace soilmachine;

int SIZEX = 96, SIZEY = 64, SCALE = 80, SEED = 42;
struct DummyVertexpool {} vertexpool;

int main(int argc, char** argv) {
  if (argc < 4) { printf("usage: facade_group file.soil ngpus out.bin\n"); return 2; }
  try {
    WorldEntry w = loadsoil(argv[1]);
    SCALE = w.scale;
    const int ngpus = atoi(argv[2]);
    const std::vector<int> devices((size_t)(ngpus > 0 ? ngpus : 1), 0);
    srand(SEED);
    WaterParticle::init(SIZEX, SIZEY); WindParticle::init(SIZEX, SIZEY);
    Layermap map(SEED, ivec2(SIZEX, SIZEY), vertexpool, SCALE, 0, ngpus, devices.data());
    WaterParticle::run(map, vertexpool, 400);                 // ponds for the water-table calls
    WaterParticle::flood_batch(map, vertexpool);
    const int edge = 48;                                      // two ranks: columns [0, 48) and [48, 96)
    double left = 0.0;
    for (int y = 2; y < SIZEY - 2; y += 3)
      for (int x = edge - 2; x <= edge + 1; x++) {
        map.add(ivec2(x, y), map.pool.get(0.02 + 0.001 * y, (SurfType)(1 + (x + y) % ((int)soils.size() - 1))));
        left += map.remove(ivec2(x, y), 0.004 * (1 + y % 5));
        Particle::cascade(vec2(x + 0.25f, y + 0.125f), map, vertexpool, y % 4);
        map.add(ivec2(x, y), map.pool.get(0.01, 0));          // standing water
        WaterParticle::seep(vec2((float)x, (float)y), map, vertexpool);
        WaterParticle::cascade(vec2((float)x, (float)y), map, vertexpool, y % 2 ? 3 : 0);
      }
    FILE* f = fopen(argv[3], "wb");
    if (!f) return 3;
    fwrite(&left, 8, 1, f);
    for (int x = 0; x < SIZEX; x++) for (int y = 0; y < SIZEY; y++) {
      int n = 0;
      for (sec* e = map.top(ivec2(x, y)); e != nullptr; e = e->prev) n++;
      fwrite(&n, sizeof(int), 1, f);
      for (sec* e = map.top(ivec2(x, y)); e != nullptr; e = e->prev) {
        const long long t = (long long)e->type;
        fwrite(&t, sizeof(t), 1, f); fwrite(&e->size, 8, 1, f); fwrite(&e->floor, 8, 1, f); fwrite(&e->saturation, 8, 1, f);
      }
    }
    fclose(f);
    printf("facade group ok: %d ranks, leftover sum %.17g\n", ngpus, left);
  } catch (const Error& e) {
    printf("soilmachine error %d: %s\n", e.code, e.what());
    return e.code == SM_ERR_NOGPU ? 77 : 1;
  } catch (const SoilFileError& e) { printf("%s\n", e.what()); return 2; }
  return 0;
}
