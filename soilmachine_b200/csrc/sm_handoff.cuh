// sm_handoff.cuh -- the wind sweep's hand-off rule as pure predicates, host + device.
// Two wind steps can only touch a common cell when their published boxes (ipos +- R, R = particle_reach in 3..5) meet,
// so a particle waits for exactly the lower-index particles whose box can meet its own, and its hand-off needs a release
// exactly when a higher-index particle waits for it by that same test.  Every wait is a direct one: a waiter never relies
// on a chain of hand-offs, so a step that nobody waits for publishes with a plain store and the sweep barrier's fence
// makes its writes visible to the next sweep.  tests/wind_handoff checks these exhaustively and replays the golden
// wind frames under them (tests/test_wind_handoff_host.py).  d* = B - A, R* = the published reaches.
#pragma once
#include "sm_core.cuh"

SM_HD bool handoff_in_range(int dx, int dy, int ra, int rb) {
  dx = dx < 0 ? -dx : dx;
  dy = dy < 0 ? -dy : dy;
  return dx <= ra + rb && dy <= ra + rb;
}
// A waits for B
SM_HD bool handoff_waits(int a, int ax, int ay, int ra, int b, int bx, int by, int rb) {
  return b < a && handoff_in_range(bx - ax, by - ay, ra, rb);
}
// B must publish its hand-off with a release because of A (B releases when this holds for some A)
SM_HD bool handoff_releases_for(int b, int bx, int by, int rb, int a, int ax, int ay, int ra) {
  return a > b && handoff_in_range(ax - bx, ay - by, rb, ra);
}
