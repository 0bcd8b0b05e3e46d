// sm_cell_coop.cuh -- the single-cell calls that change the map (Layermap::add / remove, Particle::cascade,
// WaterParticle::seep(vec2) and WaterParticle::cascade(vec2, spill)), executed by ONE WARP.
//
// k_cell_op (sm_engine.cu) runs these on one thread against DevAccess, which knows one strip.  Here they are written
// against the two policies of sm_coop.cuh (warp W, backing B under CoopWin), i.e. on the back-end the warp hydrology
// uses: every record access, pool allocation and free goes to the owner of the column the last focus() named, so the
// same code serves a map cut into strips.  Same arithmetic, same order of column operations as the one-thread forms;
// tests/group_cells runs this very code on the host against the golden vectors.
#pragma once
#include "sm_hydro_coop.cuh"

// Particle::cascade called from outside a particle-step carries a transfer-loop budget of up to 3 (particle.h:96-97),
// i.e. up to four nested neighbour loops; CoopScratch holds the two a particle-step needs.  CascadeCoop reads its
// per-depth scratch through `a.s`, so the accessor below names a deeper one and leaves CoopScratch's layout alone.
struct CellCascadeScratch {
  double hs[4][8];
  unsigned char ord[4][8];
  uint32_t u;
  double acc[SM_BUDGET_SLOTS];
};
template <class B> struct CellCascadeWin : CoopWin<B> {
  CellCascadeScratch* s;     // hides CoopWin::s for CascadeCoop; CoopWin's own members keep using the window scratch
  SM_HD CellCascadeWin(B& b_, CoopScratch* win, CellCascadeScratch* deep) : CoopWin<B>(b_, win), s(deep) {}
};

// op 0 add (x, y, v, t = soil) | 1 remove (x, y, v), returns the leftover | 2 cascade (fx, fy, t = transfer-loop budget)
// | 5 seep (x, y) | 6 water cascade (x, y, t = spill): one frame pushed and drained, nested particles included.
// No active-cell marking, no budget.  Every lane returns the same value.
template <class W, class B, class S>
SM_HD double cell_op_coop(W& w, B& back, CoopScratch* sc, CellCascadeScratch* deep, S* hx, int op, int x, int y,
                          float fx, float fy, double v, int t, HydroCount& hc) {
  if (op == 2) {
    CellCascadeWin<B> a(back, sc, deep);
    a.detach();                                   // records in place
    CascadeCoop<3, W, CellCascadeWin<B> >::run(w, a, (int)roundf(fx), (int)roundf(fy), t);
    return 0.0;
  }
  CoopWin<B> a(back, sc);
  a.detach();
  if (op == 0 || op == 1) {
    Sec32* const r = a.rec(x, y);
    w.one([&]() {
      a.focus(x, y);
      sc->d = 0.0;
      if (op == 0) col_add(a, *r, v, (uint32_t)t);                  // layermap.h:230
      else sc->d = col_remove(a, *r, v);                            // layermap.h:310
    });
    return sc->d;
  }
  if (op == 5) {
    w.one([&]() { hydro_seep_cell(a, x, y); });                     // water.h:285-333
  } else if (op == 6) {                                             // water.h:151-283
    int sp = 0;
    hydro_push_coop(w, a, hx, sp, x, y, t, hc);
    hydro_drain_coop(w, a, hx, sp, hc);
  }
  return 0.0;
}
