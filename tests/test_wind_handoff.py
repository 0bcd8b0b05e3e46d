"""GPU: wind batches under the hand-off rule of sm_handoff.cuh (wait for the lower-index particles in range only, release
only when a higher-index particle in range waits) bit for bit against the reference's lockstep loop, under the
conservative (SM_EXACT=0) and the exact-footprint (SM_EXACT=3) schedules; then the same batches, and a config-3 sized
batch, on an audit build (-DSM_AUDIT_HANDOFF) where every waiter checks that the hand-off it acquired was a release."""
import json
import os
import subprocess
import sys

import pytest

import _wind_handoff

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("exact", ["0", "3"])
@pytest.mark.parametrize("batch", sorted(_wind_handoff.BATCHES))
def test_wind_batch_matches_reference(ref, monkeypatch, batch, exact):
    monkeypatch.setenv("SM_EXACT", exact)
    _wind_handoff.run(batch, ref)


@pytest.fixture(scope="module")
def audit_lib(tmp_path_factory):
    """the library built with -DSM_AUDIT_HANDOFF -DSM_PROFILE (SM_AUDIT_LIB: one built already)"""
    lib = os.environ.get("SM_AUDIT_LIB")
    if lib:
        return lib
    lib = str(tmp_path_factory.mktemp("audit") / "libsoilmachine_b200_audit.so")
    subprocess.check_call(["bash", os.path.join(ROOT, "build.sh"), "-DSM_AUDIT_HANDOFF", "-DSM_PROFILE"],
                          env=dict(os.environ, SM_LIB_OUT=lib))
    return lib


def test_audit_build_sees_every_wait_released(ref, audit_lib):
    env = dict(os.environ, SM_LIB_PATH=audit_lib)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "_wind_handoff.py")], env=env, cwd=ROOT,
                         capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0, out.stderr[-4000:]
    rows = [json.loads(l) for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(rows) == 2 * (len(_wind_handoff.BATCHES) + 1), out.stdout
    for r in rows:
        assert r["audit_misses"] == 0, r
    # the crowded batch really has scans with more than 128 lower-index particles in range
    assert all(r["crowded_scans"] > 0 for r in rows if r["batch"] == "crowded"), rows
    assert all(r["sweeps"] == 300 for r in rows if r["batch"] == "config3"), rows
