#!/usr/bin/env python
"""What the reference importer's own packing code writes for the cases of tests/test_reference_cs.py and
tests/test_gpu_pack_reference.py, stored as tests/golden/ref_cs_pack_<case>.npz so that both compare with the reference
wherever they run.

The compiled reference is oracle/_ref/libref_cs.so, built from the reference's C# by oracle/refcs/build_ref_cs.py.
`reference(name)` returns its output for case `name`: computed on the spot when that library is present, otherwise read from
the fixture.  A fixture keeps, per format combination, every blob whole up to SMALL bytes, and of a larger blob its sha256
and a seeded sample of its bytes; the bounds; the conversions the reference left unspecified (see `convention_mask`); and
the sha256 of the input records, so that a changed scene cannot pass as the stored one.
Run from the repo root:  python tests/golden/make_ref_cs_golden.py [case ...]   (every case when none is named)
"""
import ctypes as C
import hashlib
import io
import os
import subprocess
import sys
import zipfile
from pathlib import Path

import numpy as np

GOLD = Path(__file__).resolve().parent
ROOT = GOLD.parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

LIB = ROOT / "oracle" / "_ref" / "libref_cs.so"
SMALL, SAMPLE = 1 << 13, 512
BLOBS = ("chunkData", "posData", "otherData", "colorData", "shData")

# ---- format combinations --------------------------------------------------------------------------------------------
PRESETS = {"VeryHigh": (0, 0, 0, 0), "High": (1, 1, 1, 2), "Medium": (2, 2, 2, 3), "Low": (2, 3, 2, 6), "VeryLow": (2, 3, 3, 8)}
# tests/test_gpu_pack.py::CUSTOM and every combination of tests/util.py FORMAT_CASES: BC7 colour and clustered SH included,
# their compressed / clustered bytes left out of the comparison
CUSTOM = ((0, 3, 2, 0), (1, 2, 0, 1), (3, 0, 1, 3), (2, 1, 3, 2), (0, 0, 0, 7),
          (3, 3, 0, 1), (0, 1, 3, 1), (1, 0, 3, 0), (2, 3, 3, 2), (3, 2, 3, 3), (0, 2, 0, 0), (2, 2, 1, 2), (1, 3, 2, 3),
          (0, 0, 1, 4), (1, 2, 0, 5), (1, 3, 1, 6), (2, 1, 2, 7), (3, 0, 1, 8), (3, 0, 3, 8))
ALL_FORMATS = tuple(dict.fromkeys(tuple(PRESETS.values()) + CUSTOM))
LOSSY = ((2, 2, 2, 3), (1, 1, 1, 2), (0, 3, 2, 0))     # Medium, High, Norm8x4 with chunked Float32 SH
VSIZE = (12, 6, 4, 2)


def label(f):
    return "f%d%d%d%d" % tuple(f)


_lib = []


def ref_cs():
    """The compiled reference (built first where the reference's sources exist), or None."""
    if _lib:
        return _lib[0]
    if os.path.isdir("/root/reference/package/Editor"):
        subprocess.run([sys.executable, str(ROOT / "oracle" / "refcs" / "build_ref_cs.py")], check=True, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT)
    if not LIB.exists():
        return None
    L = C.CDLL(str(LIB))
    L.ref_cs_sizes.restype, L.ref_cs_sizes.argtypes = None, [C.c_int] * 5 + [C.c_void_p]
    L.ref_cs_create_asset.restype = C.c_long
    L.ref_cs_create_asset.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p] * 8
    L.ref_cs_linearize.restype, L.ref_cs_linearize.argtypes = None, [C.c_void_p, C.c_int]
    L.ref_cs_f32tof16.restype, L.ref_cs_f32tof16.argtypes = C.c_uint32, [C.c_float]
    L.ref_cs_half3.restype, L.ref_cs_half3.argtypes = None, [C.c_void_p, C.c_void_p]
    for f in ("pow", "min", "max"):
        getattr(L, "ref_cs_" + f).restype, getattr(L, "ref_cs_" + f).argtypes = C.c_float, [C.c_float, C.c_float]
    L.ref_cs_saturate.restype, L.ref_cs_saturate.argtypes = C.c_float, [C.c_float]
    L.ref_cs_to_uint.restype, L.ref_cs_to_uint.argtypes = C.c_uint32, [C.c_float, C.POINTER(C.c_int)]
    L.ref_cs_to_ulong.restype, L.ref_cs_to_ulong.argtypes = C.c_uint64, [C.c_float, C.POINTER(C.c_int)]
    _lib.append(L)
    return L


def ref_pack(L, splats, f):
    """The reference's CreateAsset on a copy of `splats` with formats f: {blob: bytes or None}, bounds, conventions."""
    n = splats.shape[0]
    sz = np.zeros(7, np.int64)
    L.ref_cs_sizes(n, *f, sz.ctypes.data)
    blobs = {name: np.zeros(int(s), np.uint8) for name, s in zip(BLOBS, sz[:5])}
    rec, rows, bounds = np.zeros(n, np.uint8), np.zeros(int(sz[6]), np.uint8), np.zeros(6, np.float32)
    work = np.ascontiguousarray(splats, np.float32).copy()
    morton = L.ref_cs_create_asset(work.ctypes.data, n, *f, *(blobs[b].ctypes.data for b in ("posData", "otherData", "colorData", "shData",
                                                                                               "chunkData")), bounds.ctypes.data,
                                   rec.ctypes.data, rows.ctypes.data)
    assert morton >= 0
    if not sz[0]:
        blobs["chunkData"] = None
    if f[2] == 3:
        blobs["colorData"] = None      # BC7: Unity's compressor is not in the reference
    if f[3] > 3:
        blobs["shData"] = None         # clustered: the k-means palette is not compared
    return blobs, bounds, {"morton": np.int64(morton), "rec": rec, "rows": rows, "tex_w": np.int64(sz[5])}


def convention_mask(name, size, f, n, conv, tex_w):
    """Bytes of blob `name` whose value the reference leaves to a choice it does not make: a float -> integer conversion
    out of range (C# leaves the result unspecified), and -- where chunks apply -- every value derived from math.pow, which
    Burst compiles to its own pow, not the managed double-precision one the shim states.  An out-of-range Morton code makes
    the order, and so every per-splat byte, a convention."""
    m = np.zeros(size, bool)
    per_splat = name in ("posData", "otherData", "shData", "colorData")
    if int(conv["morton"]) and per_splat:
        m[:] = True
        return m
    ostride = 4 + VSIZE[f[1]] + (2 if f[3] > 3 else 0)
    rec = conv["rec"]
    if name == "posData":
        for i in np.flatnonzero(rec & 1):
            m[i * VSIZE[f[0]]:(i + 1) * VSIZE[f[0]]] = True
    elif name == "otherData":
        for i in np.flatnonzero(rec & 2):
            m[i * ostride:(i + 1) * ostride] = True
        if any(f):                                               # chunked: scale is pow(scale, 1/8)
            for k in range(4, 4 + VSIZE[f[1]]):
                m[k:n * ostride:ostride] = True
    elif name == "shData" and f[3] <= 3:
        stride = (192, 96, 60, 32)[f[3]]
        for i in np.flatnonzero(rec & 4):
            m[i * stride:(i + 1) * stride] = True
    elif name == "colorData":
        row = size // max(1, len(conv["rows"]))
        for y in np.flatnonzero(conv["rows"]):
            m[y * row:(y + 1) * row] = True
    elif name == "chunkData":
        for k in range(40, 52):                                  # sclX / sclY / sclZ: halves of pow(scale, 1/8)
            m[k::64] = True
    return m


# ---- cases ------------------------------------------------------------------------------------------------------------
def _g():
    import unitygaussiansplatting_b200 as g
    return g


def _recs(n, seed, kind=1):
    return _g().generate_input_splats(kind, n, seed)


def _f32(x):
    return np.float32(x)


def case_formats():
    return _recs(4133, 0x5EED0D00), ALL_FORMATS


def case_count(n):
    return lambda: (_recs(n, 0x5EED0D10 + n, 2), ((2, 2, 2, 3), (0, 0, 0, 0), (1, 1, 1, 2)))


def case_morton():
    """Splats on boundsMax of each axis, duplicated codes (exact copies), and +-0 coordinates."""
    s = _recs(3000, 0x5EED0D20)
    s[:, 0:3] = np.clip(s[:, 0:3], -10, 10)
    s[0, 0:3] = (10, 0.5, 0.5)
    s[1, 0:3] = (0.5, 10, 0.5)
    s[2, 0:3] = (0.5, 0.5, 10)
    s[3, 0:3] = (-10, -10, -10)
    s[4, 0:3] = (10, 10, 10)
    s[100:400] = s[400:700]                                       # duplicate codes: the tie goes to index order
    s[700:760, 0:3] = 0.0
    s[760:820, 0:3] = -0.0
    s[820:880, 0] = np.where(np.arange(60) % 2, _f32(-0.0), _f32(0.0))
    # pairs in one Morton cell but for x, where (pos - min) * inv * kScaler lands on an integer that
    # (pos - min) * (inv * kScaler) misses: the order of the pair depends on the product's association
    a, bq = morton_association_pairs(60)
    s[1000:1060, 0], s[1060:1120, 0] = a, bq
    s[1000:1060, 1:3] = s[1060:1120, 1:3] = np.float32([[1.25, -3.5]])
    return s, ((2, 2, 2, 3), (0, 0, 0, 0), (1, 1, 1, 2), (3, 3, 0, 1))


def morton_association_pairs(count, lo=-10.0, hi=10.0):
    """(x_a, x_b): x_a where ((x - lo) * inv) * kScaler truncates to m but (x - lo) * (inv * kScaler) to m - 1 (or the
    reverse), x_b in cell m - 1 under both.  inv = 1 / (hi - lo), all float32."""
    k, inv = np.float32(2097151.0), np.float32(1.0) / (np.float32(hi) - np.float32(lo))
    m = np.arange(1, 2097150, dtype=np.float64)
    x = (m / 2097151.0 * (hi - lo) + lo).astype(np.float32)
    x = np.concatenate([x, np.nextafter(x, np.float32(-np.inf)), np.nextafter(x, np.float32(np.inf))])
    d = x - np.float32(lo)
    c1, c2 = np.floor(d * inv * k), np.floor(d * (inv * k))
    xa = x[c1 != c2][:count]
    lowcell = np.minimum(c1, c2)[c1 != c2][:count]
    xb = np.nextafter(xa, np.float32(-np.inf))
    for _ in range(64):                                           # step down until both products truncate to the lower cell
        db = xb - np.float32(lo)
        ok = (np.floor(db * inv * k) == lowcell) & (np.floor(db * (inv * k)) == lowcell)
        if ok.all():
            break
        xb = np.where(ok, xb, np.nextafter(xb, np.float32(-np.inf)))
    assert xa.size == count and ok.all()
    return xa, xb


def case_zero_bounds():
    """Positions in [0, 1] with +0 and -0 on every axis, in both orders: which zero the bounds and chunk folds keep."""
    s = _recs(600, 0x5EED0D28)
    s[:, 0:3] = np.abs(np.clip(s[:, 0:3] / 30, -1, 1))
    z = np.where(np.arange(600) % 2, _f32(-0.0), _f32(0.0)).astype(np.float32)
    for k in range(3):
        s[k::7, k] = z[k::7]
    s[5::11, 0:3] = -0.0
    return s, ((2, 2, 2, 3), (0, 0, 0, 0), (1, 1, 1, 2), (0, 1, 0, 0))


def case_degree0():
    """A degree-0 capture: no f_rest, every SH zero, so every chunk's SH range is 0 and only the 1e-5 bound keeps it apart."""
    s = _recs(1000, 0x5EED0D70)
    s[:, 9:54] = 0.0
    return s, LOSSY


def case_thin_axis():
    """All splats within 1e-30 of each other on y: inv = 1 / 1e-30 is finite, positions differ in their last bits."""
    s = _recs(1500, 0x5EED0D30)
    s[:, 1] = np.linspace(0, 1, 1500).astype(np.float32) * _f32(1e-30)
    return s, ((2, 2, 2, 3), (0, 0, 0, 0), (1, 1, 1, 2))


def case_inf_extent():
    """x extent -3e38 .. 3e38 overflows to inf: inv = 0, and the splat at boundsMax makes inf * 0 = NaN."""
    s = _recs(1200, 0x5EED0D40)
    s[:600, 0] *= _f32(1e37)
    s[0, 0], s[1, 0] = _f32(-3e38), _f32(3e38)
    return s, ((2, 2, 2, 3), (0, 0, 0, 0), (1, 1, 1, 2))


def case_chunks():
    """Chunk edges: a planar ground at y = 300 (min + 1e-5 rounds back to min: 0 / 0), all-zero SH chunks, opacity 0 / 1,
    scales 0, subnormal, 1e30 and near float rounding midpoints after pow(s, 1/8), colour outside [0, 1]."""
    from test_gpu_pack import _near_midpoint_scales
    rng = np.random.default_rng(11)
    s = _recs(2048, 0x5EED0D50)
    s[:, 0:3] = rng.uniform(-4, 4, (2048, 3)).astype(np.float32)
    s[:512, 1] = _f32(300.0)                                     # ground plane, far from the others
    s[:512, 0] += _f32(100.0)
    s[512:1024, 9:54] = 0.0                                      # degree-0 capture: no f_rest
    s[1024:1100, 54] = _f32(0.0)
    s[1100:1176, 54] = _f32(1.0)
    s[1176:1200, 55:58] = _f32(0.0)
    s[1200:1224, 55:58] = np.float32(1e-40)
    s[1224:1248, 55:58] = _f32(1e30)
    mid = _near_midpoint_scales(48)
    s[1248:1264, 55:58] = mid.reshape(16, 3)
    s[1300:1400, 6:9] = rng.uniform(-0.5, 1.5, (100, 3)).astype(np.float32)
    s[1400:1656, 0:3] -= _f32(100.0)                             # the first chunk in Morton order ...
    s[1400:1656, 6] = _f32(300.0)                                # ... has one equal large colour channel: 0 / 0 again
    return s, LOSSY + ((1, 2, 0, 1), (3, 0, 1, 3), (0, 0, 0, 0))


def _on_integer(scale, k=40, seed=0):
    """Float32 values v with fl(v * scale) an integer, and one ulp to either side, in [0, 1]."""
    m = np.random.default_rng(seed).integers(1, int(scale), k)
    v = (m / np.float64(scale)).astype(np.float32)
    v = v[(v * np.float32(scale)) == np.round(v * np.float32(scale))]
    return np.clip(np.concatenate([v, np.nextafter(v, np.float32(0)), np.nextafter(v, np.float32(2))]), 0, 1).astype(np.float32)


def case_quantisers():
    """One chunk (n = 256) whose position, colour and SH ranges are exactly [0, 1], so each value reaches its encoder
    unchanged: products with 65535.5 / 2047.5 / 1023.5 / 63.5 / 31.5 / 255.5 on an integer and one ulp to either side;
    rotations likewise against 1023.5 and 3.5; chunk halves at 65504, 65519.9, 65520 and at f16 rounding ties."""
    n = 256
    s = _recs(n, 0x5EED0D60)
    vals = {sc: _on_integer(sc, seed=int(sc)) for sc in (65535.5, 2047.5, 1023.5, 63.5, 31.5, 255.5)}
    pool = np.concatenate(list(vals.values()))
    rng = np.random.default_rng(5)
    for cols in (slice(0, 3), slice(6, 9), slice(9, 54), slice(58, 61)):
        w = cols.stop - cols.start
        s[:, cols] = rng.choice(pool, (n, w))
    s[:, 61] = rng.choice(np.array([0, 1 / 3, 2 / 3, 1], np.float32), n)
    s[0, 0:3], s[1, 0:3] = 0.0, 1.0
    s[0, 6:9], s[1, 6:9] = 0.0, 1.0
    s[0, 9:54], s[1, 9:54] = 0.0, 1.0
    out = [(s, ((2, 2, 2, 3), (1, 1, 1, 2), (3, 3, 2, 3), (1, 0, 2, 2), (2, 1, 2, 2)))]
    # chunk halves: the same scene with its colour / SH ranges moved onto f16 edges and ties
    t = s.copy()
    t[0, 6], t[1, 6] = _f32(65504.0), _f32(65519.9)
    t[:, 7] += _f32(2.0)
    t[0, 7], t[1, 7] = _f32(1.00048828125), _f32(65520.0)        # a tie f32tof16 rounds up (nearest-even would go down)
    t[0, 8], t[1, 8] = _f32(-1.00244140625), _f32(2.0009765625)  # 1 + 5 * 2^-11, 2 + 2^-10: ties again
    t[0, 9:54], t[1, 9:54] = _f32(-0.50048828125 / 2), _f32(1.00048828125)
    t[0, 54], t[1, 54] = _f32(0.0), _f32(1.0)
    out.append((t, ((1, 1, 1, 1), (2, 2, 1, 2), (0, 0, 1, 1))))
    return out


CASES = {
    "formats": case_formats,
    **{"count-%d" % n: case_count(n) for n in (1, 255, 256, 257, 511, 32768, 32769, 70001)},
    "morton": case_morton,
    "zero-bounds": case_zero_bounds,
    "degree0": case_degree0,
    "thin-axis": case_thin_axis,
    "inf-extent": case_inf_extent,
    "chunks": case_chunks,
    "quantisers": lambda: case_quantisers()[0],
    "f16-halves": lambda: case_quantisers()[1],
}


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def sample_ids(size, seed):
    return np.sort(np.random.default_rng(seed).choice(size, min(size, SAMPLE), replace=False)).astype(np.int64)


def compute(name, L=None):
    """Case `name` computed by the compiled reference (which must be present): {key: array} as the fixture stores it,
    but with every blob whole."""
    L = L or ref_cs()
    splats, formats = CASES[name]()
    out = {"input_sha256": digest(splats), "n": np.int64(splats.shape[0])}
    for f in formats:
        blobs, bounds, conv = ref_pack(L, splats, f)
        p = label(f) + "/"
        out[p + "bounds"] = bounds
        out[p + "morton_conv"] = conv["morton"]
        out[p + "conv_rec"] = np.flatnonzero(conv["rec"]).astype(np.int64)
        out[p + "conv_rec_bits"] = conv["rec"][conv["rec"] != 0]
        out[p + "conv_rows"] = np.flatnonzero(conv["rows"]).astype(np.int64)
        out[p + "tex_rows"] = np.int64(len(conv["rows"]))
        for b, data in blobs.items():
            if data is None:
                continue
            out[p + b + "_sha256"] = digest(data)
            out[p + b + "_size"] = np.int64(data.size)
            out[p + b] = data
    return out


def stored(name, L=None):
    """What the fixture keeps: blobs up to SMALL bytes whole, larger ones as sha256 plus a seeded sample."""
    d = compute(name, L)
    for key in [k for k in d if k.split("/")[-1] in BLOBS]:
        data = d[key]
        if data.size > SMALL:
            idx = sample_ids(data.size, int.from_bytes(hashlib.sha256(key.encode()).digest()[:4], "little"))
            d[key + "_sample_idx"], d[key + "_sample"] = idx, data[idx]
            del d[key]
    return d


def fixture(name):
    return GOLD / ("ref_cs_pack_%s.npz" % name)


def write_npz(path, data):
    """np.savez with fixed member timestamps and order, so that the bytes depend on the arrays only."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for key in sorted(data):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(data[key]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(), zipfile.ZIP_DEFLATED)


def reference(name):
    """Case `name`: computed by the compiled reference when it is present, else read from its fixture."""
    L = ref_cs()
    if L is not None:
        return compute(name, L)
    with np.load(fixture(name)) as f:
        return {k: f[k] for k in f.files}


def conventions(ref, f, name, size):
    """convention_mask for blob `name` of format f from a stored or computed case."""
    p = label(f) + "/"
    n = int(ref["n"])
    rec = np.zeros(n, np.uint8)
    rec[ref[p + "conv_rec"]] = ref[p + "conv_rec_bits"]
    rows = np.zeros(int(ref[p + "tex_rows"]), np.uint8)
    rows[ref[p + "conv_rows"]] = 1
    return convention_mask(name, size, f, n, {"morton": ref[p + "morton_conv"], "rec": rec, "rows": rows}, 2048)


if __name__ == "__main__":
    L = ref_cs()
    if L is None:
        raise SystemExit("oracle/_ref/libref_cs.so is not built")
    unknown = sorted(set(sys.argv[1:]) - set(CASES))
    if unknown:
        raise SystemExit("unknown case(s) %s; the cases are %s" % (unknown, sorted(CASES)))
    for name in sys.argv[1:] or CASES:
        write_npz(fixture(name), stored(name, L))
        print("wrote", fixture(name))


# ---- comparison, shared by tests/test_reference_cs.py and tests/test_gpu_pack_reference.py -----------------------------
def packer_formats(f):
    """The formats a packer is run with for reference combination f: a clustered SH format as Cluster4k, whose palette and
    indices are not compared and whose other bytes do not depend on the palette size."""
    return tuple(f) if f[3] <= 3 else (f[0], f[1], f[2], 8)


def differences(asset, ref, f):
    """Where packed `asset` differs from the reference's case data `ref` for formats f: a list of messages, each saying
    whether the differing bytes are reference truth or a stated convention (convention_mask)."""
    p = label(f) + "/"
    msgs = []
    for key, mine in (("bounds", np.concatenate([asset.boundsMin, asset.boundsMax]).astype(np.float32)),):
        if not np.array_equal(mine.view(np.uint32), ref[p + key].view(np.uint32)):
            msgs.append("bounds %s != reference %s" % (mine, ref[p + key]))
    for b in BLOBS:
        if p + b + "_sha256" not in ref:
            continue
        mine = getattr(asset, b)
        if mine is None or mine.size != int(ref[p + b + "_size"]):
            msgs.append("%s: %s bytes, the reference writes %d" % (b, None if mine is None else mine.size, int(ref[p + b + "_size"])))
            continue
        mine = mine.copy()
        if b == "otherData" and f[3] > 3:                           # the palette index: not written by the reference harness
            st = 4 + VSIZE[f[1]] + 2
            mine[:int(ref["n"]) * st].reshape(-1, st)[:, st - 2:] = 0
        if np.array_equal(digest(mine), ref[p + b + "_sha256"]):
            continue
        if p + b in ref:
            d = np.flatnonzero(mine != ref[p + b])
        else:
            idx = ref[p + b + "_sample_idx"]
            d = idx[mine[idx] != ref[p + b + "_sample"]]
        conv = conventions(ref, f, b, mine.size)
        truth = d[~conv[d]] if d.size else d
        msgs.append("%s differs from the reference (sha256)%s: %d differing bytes seen, %d of them reference truth, first at %s" %
                    (b, "" if p + b in ref else " [sampled]", d.size, truth.size, d[:1].tolist()))
    return msgs
