"""CPU: the wind sweep's hand-off rule (soilmachine_b200/csrc/sm_handoff.cuh).  A wind particle waits for exactly the
lower-index particles whose published box can meet its own, and releases its hand-off exactly when a higher-index
particle waits for it; there is no own-bin order.  Checked exhaustively on the predicates, and by replaying the golden
frames with every wind sweep run in the most out-of-order order the rule allows (tests/wind_handoff: tests/hostsim
with that schedule added)."""
import ctypes as C
import os
import subprocess
import pytest
import _golden
import _hostsim
from test_host_build import Backend, stats5

SRC = os.path.join(_hostsim.HERE, "wind_handoff", "handoff_host.cpp")
LIB = os.path.join(_hostsim.HERE, "wind_handoff", "libhandoffhost.so")
DEPS = [SRC, _hostsim.SRC, _hostsim.CORE, _hostsim.NOISE, _hostsim.HYDRO, _hostsim.COOP, _hostsim.HCOOP,
        os.path.join(_hostsim.HERE, "..", "soilmachine_b200", "csrc", "sm_foot.cuh"),
        os.path.join(_hostsim.HERE, "..", "soilmachine_b200", "csrc", "sm_handoff.cuh")]


def _build():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(d) for d in DEPS):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", SRC, "-o", LIB])
    return LIB


class HandoffSim(_hostsim.HostSim):
    """the host simulator's interface over tests/wind_handoff"""

    def __init__(self):
        self.lib = C.CDLL(_build())
        self.lib.hs_nsections.restype = C.c_int64
        self.lib.hs_adversarial_ahead.restype = C.c_longlong


class BoxBackend(Backend):
    def __init__(self, g):
        self.hs = HandoffSim()
        self.hs.init(int(g["dimx"]), int(g["dimy"]), int(g["scale"]), g["soils"])


def _check(shrink):
    out = (C.c_longlong * 4)()
    HandoffSim().lib.hs_check_handoff(shrink, out)
    return list(out)


def test_handoff_predicates_cover_every_meeting_pair():
    """over every relative position up to 12 cells and every reach pair in {3, 4, 5}: the range test is symmetric,
    every pair whose boxes can meet is a wait pair (one way or the other), and the waited-for side always releases"""
    asym, missed, unreleased, pairs = _check(0)
    assert pairs == 9 * 25 * 25 * 2
    assert asym == 0
    assert missed == 0
    assert unreleased == 0


def test_handoff_predicates_with_a_range_one_short_are_caught():
    """negative control: with the range shrunk by one cell some meeting boxes are no longer a wait pair"""
    asym, missed, unreleased, _ = _check(1)
    assert missed > 0


def _replay(case, shrink):
    g = _golden.load(case)
    b = BoxBackend(g)
    b.hs.lib.hs_box_mode(1, shrink)
    try:
        b.hs.lib.hs_adversarial_ahead()
        b.hs.set_columns(_golden.cols(g, "init"))
        _golden.replay_frame(g, b, stats5)
        return b.hs.lib.hs_adversarial_ahead()
    finally:
        b.hs.lib.hs_box_mode(0, 0)


# the golden frames whose wind particles do work (in the others they die in their first move)
WIND_CASES = ["frame_rocksand_56", "frame_rgps_64"]


@pytest.mark.parametrize("case", WIND_CASES)
def test_wind_box_rule_is_sound_under_the_most_out_of_order_legal_execution(case):
    """every wind sweep of the golden frames run highest index first, each particle stepping as soon as no unfinished
    lower-index particle is in range - no own-bin order - reproduces the reference byte for byte"""
    ahead = _replay(case, 0)
    assert ahead > 1000        # the order really was far from index order


def test_wind_replay_with_no_waits_is_caught():
    """negative control of the replay: with the range shrunk until no pair waits, the same order must NOT reproduce the
    reference - the replay can see an unsound rule (a range one cell short is not enough to show here: the boxes bound
    what a step touches, so the golden frames have no conflict at the box's outer ring)"""
    with pytest.raises(AssertionError):
        _replay("frame_rocksand_56", 10)
