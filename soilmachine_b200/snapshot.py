"""The snapshot format of sm_snapshot_save / sm_snapshot_restore in numpy (format version 1, DESIGN.md section 10).

A snapshot is one little-endian byte image of the columns of the x-range [x0, x1) of a map and of its three frequency
arrays over the same columns:

    header     128 B  magic "SMSNAP\\0\\0", version, header_bytes, dimx, dimy, x0, x1, nsoils, reserved, ncells,
                      nsections, offsets_at, records_at, freq_at, total_bytes, checksum (checksum.columns_checksum of
                      the covered columns, global cell indices), zeros
    offsets           u64[ncells + 1], cell order (x - x0)*dimy + y
    records           at records_at (32-B aligned): {f64 size, floor, saturation; u32 type, reserved}, bottom -> top
    frequency         f32 water_frequency, water_track, wind_frequency, each [dimy][x1 - x0]

build() writes exactly the bytes the device writes, so this module is the statement the kernels are tested against;
cut() and join() move between a whole-map snapshot and the strips of a sharded map.
"""
import numpy as np

from . import checksum

MAGIC = b"SMSNAP\0\0"
VERSION = 1
HEADER_BYTES = 128
FREQ_KEYS = ("water_frequency", "water_track", "wind_frequency")
HEADER_DTYPE = np.dtype([
    ("magic", "S8"), ("version", "<u4"), ("header_bytes", "<u4"),
    ("dimx", "<i4"), ("dimy", "<i4"), ("x0", "<i4"), ("x1", "<i4"), ("nsoils", "<i4"), ("reserved", "<i4"),
    ("ncells", "<u8"), ("nsections", "<u8"), ("offsets_at", "<u8"), ("records_at", "<u8"), ("freq_at", "<u8"),
    ("total_bytes", "<u8"), ("checksum", "<u8"), ("pad", "V32"),
])
RECORD_DTYPE = np.dtype([("size", "<f8"), ("floor", "<f8"), ("saturation", "<f8"), ("type", "<u4"),
                         ("reserved", "<u4")])
assert HEADER_DTYPE.itemsize == HEADER_BYTES and RECORD_DTYPE.itemsize == 32


def layout(dimx, dimy, x0, x1, nsections):
    """(ncells, offsets_at, records_at, freq_at, total_bytes) of a snapshot"""
    ncells = (x1 - x0) * dimy
    offsets_at = HEADER_BYTES
    records_at = (offsets_at + 8 * (ncells + 1) + 31) // 32 * 32
    freq_at = records_at + 32 * nsections
    return ncells, offsets_at, records_at, freq_at, freq_at + 12 * ncells


def _strip_freq(a, dimx, dimy, x0, x1):
    a = np.ascontiguousarray(a, np.float32).reshape(-1)
    if a.size == dimy * (x1 - x0):
        return a.reshape(dimy, x1 - x0)
    assert a.size == dimy * dimx, "a frequency array is [dimy][dimx] or [dimy][x1 - x0]"
    return a.reshape(dimy, dimx)[:, x0:x1]


def build(cols, freq, dimx, dimy, x0=0, x1=None, nsoils=0):
    """The snapshot of the columns `cols` (bottom -> top CSR {"offsets", "type", "size", "floor", "saturation"} of the
    cells of [x0, x1), as sm_download_columns) and the frequency arrays `freq` (dict of FREQ_KEYS, each the whole map
    [dimy][dimx] as sm_get_frequency or the strip [dimy][x1 - x0]).  Returns bytes."""
    x1 = dimx if x1 is None else x1
    off = np.ascontiguousarray(cols["offsets"], np.int64)
    n = int(off[-1])
    ncells, offsets_at, records_at, freq_at, total = layout(dimx, dimy, x0, x1, n)
    assert len(off) == ncells + 1 and off[0] == 0
    h = np.zeros((), HEADER_DTYPE)
    h["magic"], h["version"], h["header_bytes"] = MAGIC, VERSION, HEADER_BYTES
    h["dimx"], h["dimy"], h["x0"], h["x1"], h["nsoils"] = dimx, dimy, x0, x1, nsoils
    h["ncells"], h["nsections"] = ncells, n
    h["offsets_at"], h["records_at"], h["freq_at"], h["total_bytes"] = offsets_at, records_at, freq_at, total
    h["checksum"] = checksum.columns_checksum(cols, first_cell=x0 * dimy)
    buf = np.zeros(total, np.uint8)
    buf[:HEADER_BYTES] = np.frombuffer(h.tobytes(), np.uint8)
    buf[offsets_at:offsets_at + 8 * (ncells + 1)] = off.astype("<u8").view(np.uint8)
    rec = np.zeros(n, RECORD_DTYPE)
    for k in ("size", "floor", "saturation"):
        rec[k] = np.asarray(cols[k], np.float64)
    rec["type"] = np.asarray(cols["type"]).astype(np.uint32)
    buf[records_at:freq_at] = rec.view(np.uint8)
    for i, k in enumerate(FREQ_KEYS):
        a = _strip_freq(freq[k], dimx, dimy, x0, x1)
        buf[freq_at + 4 * ncells * i:freq_at + 4 * ncells * (i + 1)] = np.ascontiguousarray(a, "<f4").view(np.uint8).reshape(-1)
    return buf.tobytes()


def header(buf):
    """the header of a snapshot as a dict (ValueError when it is not one)"""
    b = np.frombuffer(memoryview(buf), np.uint8)
    if b.size < HEADER_BYTES:
        raise ValueError("snapshot: shorter than its header")
    h = b[:HEADER_BYTES].view(HEADER_DTYPE)[0]
    if bytes(h["magic"]).ljust(8, b"\0") != MAGIC or int(h["version"]) != VERSION:
        raise ValueError("snapshot: bad magic or version")
    out = {k: int(h[k]) for k in HEADER_DTYPE.names if k not in ("magic", "pad")}
    if (out["ncells"], out["offsets_at"], out["records_at"], out["freq_at"], out["total_bytes"]) != \
            layout(out["dimx"], out["dimy"], out["x0"], out["x1"], out["nsections"]) or b.size < out["total_bytes"]:
        raise ValueError("snapshot: inconsistent layout or truncated")
    return out


def parse(buf):
    """-> (header dict, cols, freq): cols the CSR of the covered cells as sm_download_columns returns it, freq a dict
    of FREQ_KEYS, each float32 of shape (dimy, x1 - x0)"""
    h = header(buf)
    b = np.frombuffer(memoryview(buf), np.uint8)
    nc, n = h["ncells"], h["nsections"]
    off = b[h["offsets_at"]:h["offsets_at"] + 8 * (nc + 1)].view("<u8").astype(np.int64)
    rec = b[h["records_at"]:h["freq_at"]].view(RECORD_DTYPE)
    cols = {"offsets": off, "type": rec["type"].astype(np.int32), "size": rec["size"].copy(),
            "floor": rec["floor"].copy(), "saturation": rec["saturation"].copy()}
    assert len(rec) == n
    w = h["x1"] - h["x0"]
    freq = {k: b[h["freq_at"] + 4 * nc * i:h["freq_at"] + 4 * nc * (i + 1)].view("<f4").astype(np.float32).reshape(h["dimy"], w)
            for i, k in enumerate(FREQ_KEYS)}
    return h, cols, freq


def cut(buf, x0, x1):
    """the strip snapshot of [x0, x1) out of a snapshot that covers it"""
    h, cols, freq = parse(buf)
    assert h["x0"] <= x0 < x1 <= h["x1"]
    dimy = h["dimy"]
    off = cols["offsets"]
    a, b = (x0 - h["x0"]) * dimy, (x1 - h["x0"]) * dimy
    lo, hi = off[a], off[b]
    part = {"offsets": off[a:b + 1] - lo}
    for k in ("type", "size", "floor", "saturation"):
        part[k] = cols[k][lo:hi]
    f = {k: v[:, x0 - h["x0"]:x1 - h["x0"]] for k, v in freq.items()}
    return build(part, f, h["dimx"], dimy, x0, x1, h["nsoils"])


def join(strips):
    """the snapshot of the union of strip snapshots that follow each other along x (in any order): offsets rebased,
    records concatenated, frequency rows interleaved"""
    parts = sorted((parse(s) for s in strips), key=lambda p: p[0]["x0"])
    h0 = parts[0][0]
    for (ha, _, _), (hb, _, _) in zip(parts, parts[1:]):
        assert ha["x1"] == hb["x0"] and (ha["dimx"], ha["dimy"], ha["nsoils"]) == (hb["dimx"], hb["dimy"], hb["nsoils"])
    off, base = [np.zeros(1, np.int64)], 0
    for _, c, _ in parts:
        off.append(c["offsets"][1:] + base)
        base += int(c["offsets"][-1])
    cols = {"offsets": np.concatenate(off)}
    for k in ("type", "size", "floor", "saturation"):
        cols[k] = np.concatenate([c[k] for _, c, _ in parts])
    freq = {k: np.concatenate([f[k] for _, _, f in parts], axis=1) for k in FREQ_KEYS}
    return build(cols, freq, h0["dimx"], h0["dimy"], h0["x0"], parts[-1][0]["x1"], h0["nsoils"])


def write(path, buf):
    with open(path, "wb") as f:
        f.write(memoryview(buf))


def read(path):
    with open(path, "rb") as f:
        return f.read()
