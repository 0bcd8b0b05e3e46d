"""CPU: the snapshot format (soilmachine_b200/snapshot.py, the numpy statement of it) and the device's per-cell logic
(soilmachine_b200/csrc/sm_snap.cuh) compiled for the host by tests/snapshot/host_snap.cpp.

* On the four golden frames and the two golden hydrology cases: the twin round-trips, strips cut at 2 and 3 places
  join back into the whole-map snapshot, and the header's checksum is checksum.columns_checksum.
* The host build of the device functions, on a top / pool image of the same columns whose pool slots are shuffled and
  have holes: it packs the twin's bytes; unpacking the twin's bytes and packing again gives them back; unpacking a
  strip keeps every pool index inside that strip's pool; a pack that skips a column's deepest buried section fails.
* The restore's checks reject a wrong magic, a truncated buffer, offsets that run backwards and a type >= nsoils.
* host.spawn_list counts its rand() draws for Simulation.save / load."""
import ctypes as C
import os

import numpy as np
import pytest

import _golden
from _hydro_budget import _build
from soilmachine_b200 import checksum, snapshot

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "soilmachine_b200", "csrc")
NIL = 0xFFFFFFFF
SEC32 = np.dtype([("size", "<f8"), ("floor", "<f8"), ("saturation", "<f8"), ("type", "<u4"), ("below", "<u4")])
CASES = [(c, "after_frame") for c in _golden.FRAME_CASES] + [(c, "after_seep_2") for c in _golden.HYDRO_CASES]


def _lib():
    src = os.path.join(HERE, "snapshot", "host_snap.cpp")
    lib = C.CDLL(_build("host_snap", src, [os.path.join(CSRC, "sm_snap.cuh"), os.path.join(CSRC, "sm_core.cuh")]))
    lib.hsnap_pack.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    lib.hsnap_validate.argtypes = [C.c_char_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.hsnap_unpack.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]
    return lib


def _case(name, prefix):
    g = _golden.load(name)
    dimx, dimy = int(g["dimx"]), int(g["dimy"])
    freq = {k: g["freq_" + k] for k in snapshot.FREQ_KEYS}
    return g, _golden.cols(g, prefix), freq, dimx, dimy, int(len(g["soils"]))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def shuffled_image(cols, seed, holes=997):
    """top[ncells] / pool of the CSR's columns: buried sections in random pool slots, `holes` slots of garbage among
    them"""
    rng = np.random.default_rng(seed)
    off = np.asarray(cols["offsets"], np.int64)
    nc, n = len(off) - 1, int(off[-1])
    counts = np.diff(off)
    is_top = np.zeros(n, bool)
    is_top[off[1:][counts > 0] - 1] = True
    nb = n - int(is_top.sum())
    pool = np.zeros(nb + holes, SEC32)
    garbage = rng.integers(0, 2**63, size=(nb + holes, 4), dtype=np.int64).view(np.uint8).reshape(-1)
    pool.view(np.uint8)[:] = garbage
    slot = np.full(n, NIL, np.int64)
    slot[~is_top] = rng.permutation(nb + holes)[:nb]
    first = np.repeat(off[:-1], counts)                       # index of each section's column's bottom
    below = np.where(np.arange(n) > first, np.concatenate([[NIL], slot[:-1]]), NIL)
    rec = np.zeros(n, SEC32)
    for k in ("size", "floor", "saturation"):
        rec[k] = cols[k]
    rec["type"] = cols["type"]
    rec["below"] = below
    pool[slot[~is_top]] = rec[~is_top]
    top = np.zeros(nc, SEC32)
    top["type"] = NIL
    top["below"] = NIL
    top[counts > 0] = rec[is_top]
    return top, pool


def _pack(lib, top, pool, broken=0):
    off = np.zeros(len(top) + 1, np.uint64)
    lib.hsnap_pack(len(top), _p(top), _p(pool), _p(off), None, 0)
    rec = np.zeros(int(off[-1]), snapshot.RECORD_DTYPE)
    lib.hsnap_pack(len(top), _p(top), _p(pool), _p(off), _p(rec), broken)
    return off, rec


def _parts(buf):
    h = snapshot.header(buf)
    b = np.frombuffer(buf, np.uint8)
    off = b[h["offsets_at"]:h["offsets_at"] + 8 * (h["ncells"] + 1)].view("<u8")
    return off, b[h["records_at"]:h["freq_at"]].view(snapshot.RECORD_DTYPE)


@pytest.mark.parametrize("name,prefix", CASES)
def test_twin_round_trips_and_carries_the_checksum(name, prefix):
    g, cols, freq, dimx, dimy, ns = _case(name, prefix)
    buf = snapshot.build(cols, freq, dimx, dimy, nsoils=ns)
    h, c2, f2 = snapshot.parse(buf)
    _golden.same_cols(c2, cols, name + ": parse(build)")
    for k in snapshot.FREQ_KEYS:
        _golden.same(f2[k].reshape(-1), np.asarray(freq[k], np.float32), name + ": " + k)
    assert h["checksum"] == checksum.columns_checksum(cols)
    assert (h["dimx"], h["dimy"], h["x0"], h["x1"], h["nsoils"], h["nsections"]) == (dimx, dimy, 0, dimx, ns, len(cols["type"]))
    assert h["records_at"] % 32 == 0 and len(buf) == h["total_bytes"]


@pytest.mark.parametrize("name,prefix", CASES)
@pytest.mark.parametrize("cuts", [[0.5], [0.3, 0.71]], ids=["2strips", "3strips"])
def test_strips_join_into_the_whole_map_snapshot(name, prefix, cuts):
    g, cols, freq, dimx, dimy, ns = _case(name, prefix)
    whole = snapshot.build(cols, freq, dimx, dimy, nsoils=ns)
    xs = [0] + [int(round(c * dimx)) | 1 for c in cuts] + [dimx]      # odd edges: widths not multiples of 16
    strips = [snapshot.cut(whole, a, b) for a, b in zip(xs, xs[1:])]
    assert any((b - a) % 16 for a, b in zip(xs, xs[1:]))
    assert sum(snapshot.header(s)["checksum"] for s in strips) % (1 << 64) == snapshot.header(whole)["checksum"]
    assert snapshot.join(strips[::-1]) == whole


@pytest.mark.parametrize("name,prefix", CASES)
def test_host_build_of_the_device_code_packs_and_unpacks_the_twins_bytes(name, prefix):
    lib = _lib()
    g, cols, freq, dimx, dimy, ns = _case(name, prefix)
    buf = snapshot.build(cols, freq, dimx, dimy, nsoils=ns)
    want_off, want_rec = _parts(buf)
    top, pool = shuffled_image(cols, seed=len(name))
    off, rec = _pack(lib, top, pool)
    assert off.tobytes() == want_off.tobytes() and rec.tobytes() == want_rec.tobytes()
    # negative control: a pack that never writes a column's deepest buried section (where a column has one)
    off_b, rec_b = _pack(lib, top, pool, broken=1)
    assert (rec_b.tobytes() != want_rec.tobytes()) == bool((np.diff(off) >= 2).any())
    # unpack the whole map, pack again
    assert lib.hsnap_validate(buf, len(buf), dimx, dimy, ns, 0, dimx) == 0
    t2 = np.zeros(dimx * dimy, SEC32)
    p2 = np.zeros(len(want_rec) + 1, SEC32)
    need = C.c_int64()
    lib.hsnap_unpack(buf, 0, dimx, _p(t2), _p(p2), C.byref(need))
    off2, rec2 = _pack(lib, t2, p2)
    assert off2.tobytes() == want_off.tobytes() and rec2.tobytes() == want_rec.tobytes()
    assert need.value == len(want_rec) - int((np.diff(want_off.astype(np.int64)) > 0).sum())


@pytest.mark.parametrize("name,prefix", CASES[:2] + CASES[-1:])
def test_unpacking_a_strip_stays_in_its_own_pool(name, prefix):
    lib = _lib()
    g, cols, freq, dimx, dimy, ns = _case(name, prefix)
    whole = snapshot.build(cols, freq, dimx, dimy, nsoils=ns)
    xs = [0, 17, 2 * dimx // 3 + 1, dimx]
    for a, b in zip(xs, xs[1:]):
        assert lib.hsnap_validate(whole, len(whole), dimx, dimy, ns, a, b) == 0
        top = np.zeros((b - a) * dimy, SEC32)
        pool = np.zeros(len(cols["type"]) + 1, SEC32)
        need = C.c_int64()
        lib.hsnap_unpack(whole, a, b, _p(top), _p(pool), C.byref(need))
        links = np.concatenate([top["below"], pool["below"][:need.value]])
        assert ((links == NIL) | (links < need.value)).all(), "a pool link leaves the strip's pool"
        off, rec = _pack(lib, top, pool)
        assert snapshot.cut(whole, a, b) == snapshot.build(
            {"offsets": off.astype(np.int64), "type": rec["type"].astype(np.int32), "size": rec["size"],
             "floor": rec["floor"], "saturation": rec["saturation"]},
            {k: np.asarray(v).reshape(dimy, dimx)[:, a:b] for k, v in freq.items()}, dimx, dimy, a, b, ns)


def test_restore_checks_reject_malformed_snapshots():
    lib = _lib()
    g, cols, freq, dimx, dimy, ns = _case("frame_rocksand_56", "after_frame")
    buf = snapshot.build(cols, freq, dimx, dimy, nsoils=ns)
    h = snapshot.header(buf)
    assert lib.hsnap_validate(buf, len(buf), dimx, dimy, ns, 0, dimx) == 0

    def edited(at, value, dtype):
        b = bytearray(buf)
        b[at:at + np.dtype(dtype).itemsize] = np.array(value, dtype).tobytes()
        return bytes(b)

    assert lib.hsnap_validate(b"XM" + buf[2:], len(buf), dimx, dimy, ns, 0, dimx) == 1            # magic
    assert lib.hsnap_validate(buf, len(buf) - 1, dimx, dimy, ns, 0, dimx) == 1                   # truncated
    assert lib.hsnap_validate(buf, 100, dimx, dimy, ns, 0, dimx) == 1
    assert lib.hsnap_validate(buf, len(buf), dimx + 1, dimy, ns, 0, dimx) == 1                   # dimensions
    assert lib.hsnap_validate(buf, len(buf), dimx, dimy, ns + 1, 0, dimx) == 1                   # nsoils
    off = np.frombuffer(buf, np.uint8)[h["offsets_at"]:h["offsets_at"] + 8 * (h["ncells"] + 1)].view("<u8")
    c = int(np.nonzero(np.diff(off.astype(np.int64)) >= 2)[0][h["ncells"] // 3 % 50])
    bad = edited(h["offsets_at"] + 8 * (c + 1), off[c] - 1, "<u8")                               # runs backwards
    assert lib.hsnap_validate(bad, len(bad), dimx, dimy, ns, 0, dimx) == 3
    bad = edited(h["offsets_at"] + 8 * h["ncells"], h["nsections"] + 1, "<u8")                   # wrong end
    assert lib.hsnap_validate(bad, len(bad), dimx, dimy, ns, 0, dimx) == 2
    bad = edited(h["records_at"] + 32 * (h["nsections"] // 2) + 24, ns, "<u4")                   # type >= nsoils
    assert lib.hsnap_validate(bad, len(bad), dimx, dimy, ns, 0, dimx) == 3


def test_spawn_list_counts_its_rand_draws():
    from soilmachine_b200 import host
    host.srand(5)
    assert host.draws() == 0
    host.spawn_list(7, 32, 24)
    host.spawn_list(3, 32, 24)
    assert host.draws() == 20
    a = host.spawn_list(4, 32, 24)
    host.srand(5)
    assert host.draws() == 0
    host.spawn_list(10, 32, 24)
    assert np.array_equal(host.spawn_list(4, 32, 24), a)
