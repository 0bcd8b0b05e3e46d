// tests/wind_handoff -- tests/hostsim with one more wind schedule, for tests/test_wind_handoff_host.py.  TEST TOOL ONLY.
// The host simulator is compiled as it is; its hs_wind_sweep becomes hs_wind_sweep_index_order, and the hs_wind_sweep
// below runs a sweep in the box-rule adversarial order when hs_box_mode(1, .) is set, in the simulator's own order
// otherwise.
#define hs_wind_sweep hs_wind_sweep_index_order
#include "../hostsim/hostsim.cpp"
#undef hs_wind_sweep
#include "../../soilmachine_b200/csrc/sm_handoff.cuh"

namespace {
// The conservative wind schedule on one rank (wind_wait, sm_sweep.cuh) lets a whole step run once every lower-index
// particle that handoff_waits (sm_handoff.cuh) names is finished - with no own-bin order.  Here a wind sweep runs in the
// legal order that departs most from index order: passes from the HIGHEST index down, each particle stepping as soon as
// the rule lets it.  G_box_shrink > 0 shrinks the range by that many cells.
int G_box = 0, G_box_shrink = 0;
void sweep_box_adversarial(std::vector<WindP>& parts, const std::vector<int>& live, std::vector<int>& res) {
  const size_t n = live.size();
  std::vector<Fly> fly(n);
  for (size_t k = 0; k < n; k++) {
    const WindP& p = parts[live[k]];
    fly[k] = Fly{live[k], 0, (int)roundf(p.px), (int)roundf(p.py), 0, 0, host_reach(p)};
  }
  res.assign(n, SM_ALIVE);
  WarpHost w;
  size_t left = n;
  for (int pass = 0; left > 0; pass++) {
    if (pass > 100000) { fprintf(stderr, "sweep_box_adversarial: no progress\n"); abort(); }
    for (size_t kk = n; kk-- > 0;) {
      Fly& A = fly[kk];
      if (A.phase == 2) continue;
      bool ok = true, lower_open = false;
      for (size_t j = 0; j < kk && ok; j++) {
        const Fly& B = fly[j];
        if (B.phase == 2) continue;
        lower_open = true;
        if (handoff_waits(A.id, A.ix, A.iy, A.R - G_box_shrink, B.id, B.ix, B.iy, B.R)) ok = false;
      }
      if (!ok) continue;
      if (lower_open) G_adv_ahead++;
      HostBack b; CoopScratch sc; CoopWin<HostBack> cw(b, &sc);
      res[kk] = wind_step_coop(w, cw, parts[A.id]);
      cw.flush(w);
      A.phase = 2; left--;
    }
  }
}

// sm_handoff.cuh exhaustively over every relative position (|B - A| up to 12) and reach pair in {3, 4, 5}, against the
// boxes as explicit cell sets.  out[0]: asymmetric pairs (A in range of B but not B of A); out[1]: pairs whose boxes
// meet and neither waits for the other; out[2]: wait pairs whose waited-for side need not release; out[3]: pairs
// checked.  shrink > 0 evaluates the predicates with the range shrunk by that many cells (negative control).
void handoff_exhaustive(int shrink, long long* out) {
  for (int ra = 3; ra <= 5; ra++) for (int rb = 3; rb <= 5; rb++)
  for (int dx = -12; dx <= 12; dx++) for (int dy = -12; dy <= 12; dy++) {
    const int sa = ra - shrink;
    if (handoff_in_range(dx, dy, sa, rb) != handoff_in_range(-dx, -dy, rb, sa)) out[0]++;
    CellSet A, B; A.rect(0, 0, ra); B.rect(dx, dy, rb);
    const bool meet = A.meets(B);
    for (int ab = 0; ab < 2; ab++) {          // A has index 1 and B index 0, then the other way round
      const int ia = ab, ib = 1 - ab;
      const bool a_waits = handoff_waits(ia, 0, 0, sa, ib, dx, dy, rb);
      const bool b_waits = handoff_waits(ib, dx, dy, rb, ia, 0, 0, sa);
      if (meet && !a_waits && !b_waits) out[1]++;
      if (a_waits && !handoff_releases_for(ib, dx, dy, rb, ia, 0, 0, sa)) out[2]++;
      out[3]++;
    }
  }
}
}  // namespace

extern "C" {
void hs_box_mode(int on, int shrink) { G_box = on; G_box_shrink = shrink; }
void hs_check_handoff(int shrink, long long* out4) {
  for (int i = 0; i < 4; i++) out4[i] = 0;
  handoff_exhaustive(shrink, out4);
}
int hs_wind_sweep(Stats* st) {
  if (!G_box) return hs_wind_sweep_index_order(st);
  std::vector<int> adv, next;
  sweep_box_adversarial(D, Dlive, adv);
  size_t kpos = 0;
  for (int i : Dlive) {          // the bookkeeping of hs_wind_sweep
    if (adv[kpos++] != SM_ALIVE) { st->exit_oob++; continue; }
    st->steps++;
    next.push_back(i);
  }
  Dlive.swap(next); st->sweeps++;
  return (int)Dlive.size();
}
}
