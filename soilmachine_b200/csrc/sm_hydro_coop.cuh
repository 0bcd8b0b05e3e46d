// sm_hydro_coop.cuh -- pooling hydrology (flood, water-table cascade, seep) executed by ONE WARP.
//
// Same canonical order and the same arithmetic as sm_hydro.cuh (reference: water.h:123-343): floods in ascending
// particle index, the seep pass over the flagged cells in x-major order, every flood / visit atomic with its
// nested particles.  That order is sequential by definition, so what a warp can shorten is the work inside one
// flood or visit:
//   * a water-cascade frame evaluates its (up to) eight neighbours on eight lanes at once; the first neighbour in
//     visiting order that acts is executed, the ones before it had no effect (the early exits of water.h:211-234
//     are side-effect free), the ones after it are evaluated again on the new state - exactly the states the
//     reference loop sees (same argument as CascadeCoop in sm_coop.cuh);
//   * opening a frame (eight heights + stable rank sort) is lane-parallel;
//   * a nested particle runs the cooperative particle-step (water_step_coop), the flood's terrain cascade the
//     cooperative cascade.
// Column mutations are done by one lane.  Written against the same two policies as sm_coop.cuh (warp W, accessor
// A = CoopWin<B>), so tests/hostsim runs this very code on the host against the reference's golden vectors.
#pragma once
#include "sm_coop.cuh"
#include "sm_hydro.cuh"

// Mass budget of one hydrology call (scratch HydroScratchBudget, with B::kBudget for the particle-step's six slots of
// sm_coop.cuh): eleven f64 accumulators, summed in execution order by the lane that mutates columns, identical in the
// oracle port's budget extension (tests/hydro_budget/port_budget.cpp).  Heights are column heights (floor + size of
// the top section) read right before and right after the column operation, as the step's budget reads them.  They are heights, not materials: a remove on an
// Air-topped column takes the water first, so a nested particle's `eroded` can be water.
//   0 flood_sediment     height added by the flood's sediment add                  (water.h:133)
//   1 flood_cascade_net  net height change of the flood's terrain cascade          (water.h:134), as cascade_net
//   2 flood_water        height added by the flood's Air add                       (water.h:138)
//   3 seeped             height removed by seep(cell), positive: the flood's seep and the seep pass (water.h:318-319)
//   4 to_particles       height removed when a whole water section leaves as a nested particle (water.h:248)
//   5 transfer_net       partial water-table transfers: height lost at tpos + height gained at bpos (water.h:268-271)
//   6..10                the step budget's slots 0-4 (eroded, deposited, cascade_net, discarded, clamped), summed
//                        over every step of every nested particle
// Identity: d(sum of heights) = [0] + [1] + [2] - [3] - [4] + [5] + [7] - [6] + [8], to rounding.
//
// Per-cell maps of the same sums (SM_FLAG_HYDRO_CELL_BUDGET): a backing with kCellBudget gets cell_budget(term, x, y,
// d) at every measurement point above, each delta credited to the cell whose height was read.  Terms 0-2 are the
// step's (sm_coop.cuh; the nested particles' steps and the flood's terrain cascade call them), plus
//   1 deposited  the flood's sediment add at the truncated ipos                              (slot 0)
//   3 water_net  the flood's Air add (+) and every seep(cell) (-, the height removed); a whole water section leaving as
//                a nested particle at tpos (-); a partial transfer, tpos and bpos each their own change (slots 2-5)
// Per cell: d(height) = deposited - eroded + cascade_net + water_net, to rounding.
#define SM_HYDRO_BUDGET_SLOTS 11
#define SM_HYDRO_CELL_TERMS 4

struct HydroScratch {          // per warp; written by one lane, read by all
  static constexpr bool kBudget = false;
  WFrame st[SM_WSTACK];
};
// The scratch of an executor that keeps the hydrology's budget: a separate type, so that the one without keeps its
// layout (and its code).  The budget is kept where the scratch has it; the step's six slots it sums need B::kBudget.
struct HydroScratchBudget : HydroScratch {
  static constexpr bool kBudget = true;
  double bud[SM_HYDRO_BUDGET_SLOTS];   // mass budget of the current call (single lane)
};
template <bool BUDGET> struct HydroScratchOf { typedef HydroScratch type; };
template <> struct HydroScratchOf<true> { typedef HydroScratchBudget type; };

// gather the in-bounds neighbours and their visiting order (water.h:155-183): highest first, stable
template <class W, class A> SM_HD void hydro_open_coop(W& w, A& a, WFrame* f, int cx, int cy, int spill) {
  const int dimx = a.dimx(), dimy = a.dimy();
  double* const hs = a.s->hs[0];
  unsigned char* const ord = a.s->ord[0];
  const unsigned int inb = ((cx > 0 ? 0x07u : 0u) | 0x18u | (cx < dimx - 1 ? 0xE0u : 0u)) &
                           ((cy > 0 ? 0x29u : 0u) | 0x42u | (cy < dimy - 1 ? 0x94u : 0u));   // :171-172
  w.each(8, [&](int k) {
    const int kk = k + (k >= 4 ? 1 : 0);
    hs[k] = ((inb >> k) & 1u) ? a.height(cx + kk / 3 - 1, cy + kk % 3 - 1) : -1.0e300;
  });
  w.each(8, [&](int k) {
    const double hk = hs[k];
    int r = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const double hj = hs[j];
      r += (j > k) ? (hj > hk ? 1 : 0) : ((j < k) ? (hk > hj ? 0 : 1) : 0);
    }
    ord[r] = (unsigned char)k;
  });
  w.one([&]() {
    unsigned int order = 0;
    for (int r = 0; r < 8; r++) order |= (unsigned int)ord[r] << (4 * r);
    f->cx = cx; f->cy = cy; f->order = order; f->num = SM_POPC(inb); f->i = 0; f->spill = spill;
  });
}
template <class W, class A>
SM_HD void hydro_push_coop(W& w, A& a, HydroScratch* hsx, int& sp, int cx, int cy, int spill, HydroCount& hc) {
  if (sp >= SM_WSTACK) { hc.overflow++; return; }
  hydro_open_coop(w, a, &hsx->st[sp], cx, cy, spill);
  sp++;
}

// would the water cascade act on neighbour (nx, ny) of (cx, cy) right now?  (water.h:185-234; no side effects)
template <class A> SM_HD bool hydro_neighbour_acts(A& a, int cx, int cy, int nx, int ny, int SCALE) {
  const Sec32* pa = a.rec(cx, cy);
  const Sec32* pb = a.rec(nx, ny);
  double whA = 0, whB = 0, fA = 0.0, fB = 0.0;
  if (pa->type != SM_EMPTY) { whA = pa->size; fA = pa->floor; }
  if (pb->type != SM_EMPTY) { whB = pb->size; fB = pb->floor; }
  const double num = (fA + whA - fB - whB) * (double)SCALE;
  if (num == 0) return false;
  const Sec32* top = (num > 0) ? pa : pb;
  if (top->type != SM_AIR) return false;
  const double diff = num / 80.0;
  if (diff == 0) return false;
  double transfer = fabs(diff) / 2.0;
  const double wh = top->size;
  transfer = (wh < transfer) ? wh : transfer;
  return !(transfer <= 0);
}

template <class W, class A, class S>
SM_HD void hydro_flood_coop(W& w, A& a, const WaterP& p, int spill, S* hsx, int& sp, HydroCount& hc);

// run every open frame to its end (water.h:185-281 as a frame machine, see sm_hydro.cuh).  S: HydroScratch or
// HydroScratchBudget.
template <class W, class A, class S> SM_HD void hydro_drain_coop(W& w, A& a, S* hsx, int& sp, HydroCount& hc) {
  static_assert(!S::kBudget || A::kBudget, "the hydrology budget sums the step budget's slots");
  const int SCALE = a.scale();
  SM_UNROLL1
  while (sp > 0) {
    WFrame* const fp = &hsx->st[sp - 1];
    const int cx = fp->cx, cy = fp->cy, fnum = fp->num, fi = fp->i;
    const unsigned int order = fp->order;
    if (fi >= fnum) { sp--; continue; }
    const unsigned int act = w.ballot(fnum, [&](int r) {
      if (r < fi) return false;
      const int k = (int)((order >> (4 * r)) & 7u);
      const int kk = k + (k >= 4 ? 1 : 0);
      return hydro_neighbour_acts(a, cx, cy, cx + kk / 3 - 1, cy + kk % 3 - 1, SCALE);
    });
    if (act == 0) { sp--; continue; }            // the rest of the frame is a no-op
    const int i = SM_FFS(act) - 1;
    const int k = (int)((order >> (4 * i)) & 7u);
    const int kk = k + (k >= 4 ? 1 : 0);
    const int nx = cx + kk / 3 - 1, ny = cy + kk % 3 - 1;
    Sec32* const pa = a.rec(cx, cy);
    Sec32* const pb = a.rec(nx, ny);
    // the acting neighbour, evaluated again by every lane (uniform): same expressions as hydro_drain
    double whA = 0, whB = 0, fA = 0.0, fB = 0.0;
    if (pa->type != SM_EMPTY) { whA = pa->size; fA = pa->floor; }
    if (pb->type != SM_EMPTY) { whB = pb->size; fB = pb->floor; }
    const double num = (fA + whA - fB - whB) * (double)SCALE;
    Sec32* const top = (num > 0) ? pa : pb;
    Sec32* const bot = (num > 0) ? pb : pa;
    const int tx = (num > 0) ? cx : nx, ty = (num > 0) ? cy : ny;
    const int bx = (num > 0) ? nx : cx, by = (num > 0) ? ny : cy;
    const double diff = num / 80.0;
    double transfer = fabs(diff) / 2.0;                             // :227
    const double wh = top->size;                                    // :230
    transfer = (wh < transfer) ? wh : transfer;
    const int fspill = fp->spill;
    if (transfer == wh) {                                           // :240-258 all of it leaves as a particle
      w.one([&]() {
        fp->i = i + 1;
        double h0 = 0.0;
        if constexpr (S::kBudget) h0 = rec_height(*top);
        a.focus(tx, ty);
        col_remove(a, *top, transfer);
        if constexpr (S::kBudget) { const double d = h0 - rec_height(*top); hsx->bud[4] += d; a.cell_budget(3, tx, ty, -d); }
        a.dirty_rec(top, tx, ty);
      });
      WaterP q;
      q.px = (float)tx; q.py = (float)ty;
      {
        const float dx = (float)bx - (float)tx, dy = (float)by - (float)ty;   // :246
        const float inv = 1.0f / sqrtf(dx * dx + dy * dy);
        q.sx = SM_SQRT2F * (dx * inv);
        q.sy = SM_SQRT2F * (dy * inv);
      }
      q.volume = transfer / a.volume_factor();                      // :250
      q.sediment = 0.0;
      q.contains = a.soil(rec_surface(*top)).transports;            // see sm_hydro.cuh: the ctor's rand() cannot reach the map
      hc.nested++;
      SM_UNROLL1
      for (;;) {                                                    // :252-253
        const int rc = water_step_coop(w, a, q);
        // Air-topped records the step modified keep the seep pass's index up to date (one lane), then write back
        const uint32_t dm = a.dirtym;
        w.one([&]() {
          for (int l = 0; l < SM_CW_SLOTS; l++)
            if ((dm >> l) & 1u) {
              const int ox = l < 9 ? a.ax : a.bx, oy = l < 9 ? a.ay : a.by, kq = l < 9 ? l : l - 9;
              a.b.air_mark(&a.s->win[l], ox + kq / 3 - 1, oy + kq % 3 - 1);
            }
          if constexpr (S::kBudget)                                 // the step's slots 0-4 (sm_coop.cuh)
            for (int k = 0; k < 5; k++) hsx->bud[6 + k] += a.s->acc[k];
        });
        a.flush(w);
        if (rc == SM_ALIVE || rc == SM_EXIT_EVAP) hc.nested_steps++;
        if (rc != SM_ALIVE) break;
      }
      a.detach();
      hydro_flood_coop(w, a, q, fspill, hsx, sp, hc);               // :254
    } else {                                                        // :260-272
      w.one([&]() {
        fp->i = i + 1;
        double ht0 = 0.0, hb0 = 0.0;
        if constexpr (S::kBudget) { ht0 = rec_height(*top); hb0 = rec_height(*bot); }
        a.focus(tx, ty);
        col_remove(a, *top, transfer);
        a.dirty_rec(top, tx, ty);
        a.focus(bx, by);
        col_add(a, *bot, transfer, SM_AIR);
        if (bot->type != SM_EMPTY) bot->saturation = 1.0;           // map.top(bpos)->saturation = 1.0f
        if constexpr (S::kBudget) {
          const double dt = rec_height(*top) - ht0, db = rec_height(*bot) - hb0;
          hsx->bud[5] += dt + db;
          a.cell_budget(3, tx, ty, dt);
          a.cell_budget(3, bx, by, db);
        }
        a.wet_mark(bx, by);
        a.dirty_rec(bot, bx, by);
        if (fspill > 0) fp->spill = fspill - 1;                     // :277-278 cascade(npos, --spill)
      });
      hc.transfers++;
      if (fspill > 0) hydro_push_coop(w, a, hsx, sp, nx, ny, fspill - 1, hc);
    }
  }
}

// WaterParticle::flood, water.h:123-145; its trailing cascade call becomes a pushed frame
template <class W, class A, class S>
SM_HD void hydro_flood_coop(W& w, A& a, const WaterP& p, int spill, S* hsx, int& sp, HydroCount& hc) {
  if (p.volume < SM_MINVOL || spill-- <= 0) return;                 // :125-126
  hc.floods++;
  const int ix = (int)p.px, iy = (int)p.py;                         // :128 ipos = pos truncates
  Sec32* const r = a.rec(ix, iy);
  const double sed = p.sediment * a.soil(p.contains).equrate;
  const uint32_t what = p.contains;
  w.one([&]() {
    double h0 = 0.0;
    if constexpr (S::kBudget) h0 = rec_height(*r);
    a.focus(ix, iy);
    col_add(a, *r, sed, what);                                      // :133
    if constexpr (S::kBudget) {
      const double d = rec_height(*r) - h0;
      hsx->bud[0] += d;
      a.cell_budget(1, ix, iy, d);
      a.s->acc[2] = 0.0;                                            // the cascade sums into acc[2]
    }
    a.dirty_rec(r, ix, iy);
  });
  CascadeCoop<0, W, A>::run(w, a, (int)roundf(p.px), (int)roundf(p.py), 0);   // :134
  const double water = p.volume * a.volume_factor();
  w.one([&]() {
    double h0 = 0.0;
    if constexpr (S::kBudget) { hsx->bud[1] += a.s->acc[2]; h0 = rec_height(*r); }
    a.focus(ix, iy);
    col_add(a, *r, water, SM_AIR);                                  // :138
    a.dirty_rec(r, ix, iy);
    if constexpr (S::kBudget) {
      const double d = rec_height(*r) - h0;
      hsx->bud[2] += d;
      a.cell_budget(3, ix, iy, d);
      h0 = rec_height(*r);
    }
    hydro_seep_cell(a, ix, iy);                                     // :139
    if constexpr (S::kBudget) { const double d = h0 - rec_height(*r); hsx->bud[3] += d; a.cell_budget(3, ix, iy, -d); }
  });
  hydro_push_coop(w, a, hsx, sp, ix, iy, spill, hc);                // :140
}

// the frame loop's per-particle tail: flood of one finished batch particle (SoilMachine.cpp:292-296)
template <class W, class A, class S>
SM_HD void hydro_flood_particle_coop(W& w, A& a, S* hsx, const WaterP& p, HydroCount& hc) {
  int sp = 0;
  a.detach();
  hydro_flood_coop(w, a, p, 3, hsx, sp, hc);                        // spill = 3, water.h:33
  hydro_drain_coop(w, a, hsx, sp, hc);
}
// one cell of the full-grid pass WaterParticle::seep(map,...), water.h:335-343
template <class W, class A, class S>
SM_HD void hydro_seep_visit_coop(W& w, A& a, S* hsx, int x, int y, HydroCount& hc) {
  int sp = 0;
  a.detach();
  w.one([&]() {
    double h0 = 0.0;
    if constexpr (S::kBudget) h0 = a.height(x, y);
    hydro_seep_cell(a, x, y);
    if constexpr (S::kBudget) { const double d = h0 - a.height(x, y); hsx->bud[3] += d; a.cell_budget(3, x, y, -d); }
  });
  hydro_push_coop(w, a, hsx, sp, x, y, 3, hc);
  hydro_drain_coop(w, a, hsx, sp, hc);
  hc.cells++;
}
