"""The host asset packer (csrc/asset_creator.cpp) against THE REFERENCE IMPORTER'S OWN C#.

oracle/_ref/libref_cs.so is package/Editor/GaussianSplatAssetCreator.cs's packing jobs and the helpers they call
(GaussianUtils, GaussianSplatAsset's sizes and layouts, InputSplatData, LinearizeDataJob), syntactically rewritten to C++ and
compiled with g++ against a shim of Unity.Mathematics / Unity.Collections (oracle/refcs/).  Where that library is built the
reference's bytes are computed on the spot; elsewhere they are read from tests/golden/ref_cs_pack_*.npz
(tests/golden/make_ref_cs_golden.py).  Every blob must equal the reference's byte for byte -- except Unity's BC7 colour and
the k-means palette and indices, which the reference does not contain.  Bytes the reference leaves to an unspecified choice
(an out-of-range float -> integer conversion, Burst's pow) are named "convention" in a failure, not reference truth."""
import struct
import sys
import tempfile
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).parent / "golden"))
import make_ref_cs_golden as M  # noqa: E402

@pytest.fixture(scope="module")
def cases():
    """{case: (input records, formats, reference data)}, each scene built once."""
    out = {}
    for name, build in M.CASES.items():
        splats, formats = build()
        ref = M.reference(name)
        assert np.array_equal(M.digest(splats), ref["input_sha256"]), "case %s: the scene is no longer the one the reference bytes are for" % name
        out[name] = (splats, formats, ref)
    return out


def _f16(x):
    return int(np.float16(x).view(np.uint16))


def _chunk_halves(ref, f, word):
    """(min, max) f16 bit patterns of ChunkInfo word `word` (0..3 colour, 10..12 scale, 13..15 SH) of every chunk."""
    c = ref[M.label(f) + "/chunkData"].view(np.uint32).reshape(-1, 16)
    return c[:, word] & 0xFFFF, c[:, word] >> 16


def check_property(name, splats, formats, ref):
    """The property that makes case `name` that case, so that a changed scene cannot quietly become an ordinary one."""
    n = splats.shape[0]
    pos = splats[:, 0:3]
    b = ref[M.label(formats[0]) + "/bounds"]
    if name == "formats":
        assert n > 4096
        for k, values in enumerate((range(4), range(4), range(4), range(9))):
            assert {f[k] for f in formats} == set(values)
    elif name.startswith("count-"):
        want = int(name[len("count-"):])
        assert n == want
        rows = int(ref[M.label(formats[0]) + "/tex_rows"])
        assert rows == {32768: 16, 32769: 32}.get(n, rows) and rows % 16 == 0
        if n > 65536:
            assert rows >= 48                                        # the Morton 16x16 swizzle past the first row of tiles
    elif name == "morton":
        for k in range(3):
            assert (pos[:, k] == b[3 + k]).sum() >= 2                # splats on boundsMax of every axis: code 2^21 - 1
        assert len(np.unique(pos.view(np.uint32), axis=0)) < n - 250  # duplicated positions: equal codes
        zero = pos == 0
        assert (zero & np.signbit(pos)).sum() > 50 and (zero & ~np.signbit(pos)).sum() > 50
        d, inv, k = pos[1000:1060, 0] - b[0], np.float32(1) / (b[3] - b[0]), np.float32(2097151.0)
        assert (np.floor(d * inv * k) != np.floor(d * (inv * k))).all()   # codes that depend on the product's association
    elif name == "degree0":
        assert not splats[:, 9:54].any()
    elif name == "zero-bounds":
        assert (b[:3] == 0).all() and np.signbit(b[:3]).any()          # a -0 bound: which equal value the fold keeps matters
        first = [pos[np.flatnonzero(pos[:, k] == 0)[0], k] for k in range(3)]
        assert any(np.signbit(first[k]) != np.signbit(b[k]) for k in range(3))
    elif name == "thin-axis":
        assert 0 < b[4] - b[1] <= 1e-30
    elif name == "inf-extent":
        with np.errstate(over="ignore"):
            assert np.isinf(np.float32(b[3]) - np.float32(b[0]))        # inv = 1 / inf = 0
        assert int(ref[M.label(formats[0]) + "/morton_conv"]) > 0     # and inf * 0 = NaN reaches the Morton cast
    elif name == "chunks":
        c = ref[M.label(formats[0]) + "/chunkData"].view(np.float32).reshape(-1, 16)
        assert ((c[:, 6] == c[:, 7]) & (np.abs(c[:, 6]) >= 256)).any()  # posY: min + 1e-5 == min, so 0 / 0
        lo, hi = _chunk_halves(ref, formats[0], 0)
        assert ((lo == hi) & (lo == _f16(300.0))).any()                 # colour R: the same
        assert (np.abs(splats[:, 9:54]).max(1) == 0).sum() >= 512        # degree-0 SH chunks
        assert (splats[:, 54] == 0).any() and (splats[:, 54] == 1).any()
        sc = splats[:, 55:58]
        assert (sc == 0).any() and ((sc > 0) & (sc < np.finfo(np.float32).tiny)).any() and (sc >= 1e30).any()
        assert ((splats[:, 6:9] < 0) | (splats[:, 6:9] > 1)).any()
    elif name == "quantisers":
        assert n == 256                                                   # one chunk, ranges exactly [0, 1]
        for sc in (65535.5, 2047.5, 1023.5, 63.5, 31.5, 255.5):
            prod = splats[:, np.r_[0:3, 6:54, 58:61]] * np.float32(sc)
            assert ((prod == np.round(prod)) & (prod > 0)).sum() >= 10, sc
    elif name == "f16-halves":
        assert n == 256
        assert _chunk_halves(ref, formats[0], 0)[1][0] == 0x7BFF           # 65519.9 -> 65504, the largest half
        lo, hi = _chunk_halves(ref, formats[0], 1)
        assert lo[0] == 0x3C01 and hi[0] == 0x7C00                        # the tie 1 + 2^-11 rounded up; 65520 -> inf
        assert _chunk_halves(ref, formats[0], 2)[0][0] == 0xBC03           # -(1 + 5 * 2^-11): a tie, up in magnitude
        assert _chunk_halves(ref, formats[0], 13)[1][0] == 0x3C01          # SH: the same tie as a chunk maximum


@pytest.mark.parametrize("name", list(M.CASES))
def test_every_case_keeps_its_property(cases, name):
    splats, formats, ref = cases[name]
    check_property(name, splats, formats, ref)


@pytest.mark.parametrize("name", list(M.CASES))
def test_host_packer_matches_the_reference_importer(g, cases, name):
    splats, formats, ref = cases[name]
    bad = []
    for f in formats:
        asset = g.create_asset(splats.copy(), formats=M.packer_formats(f))
        bad += ["%s: %s" % (M.label(f), m) for m in M.differences(asset, ref, f)]
    assert not bad, "\n".join(bad)


# ---- LinearizeDataJob against gsa_ply_read ------------------------------------------------------------------------------
def linearize_records():
    """Raw PLY-space records: quaternion (0,0,0,0) and negative w, log-scales +-88, opacity logits +-100, f_dc beyond +-10."""
    rng = np.random.default_rng(17)
    n = 64
    r = np.zeros((n, 62), np.float32)
    r[:, 0:3] = rng.normal(size=(n, 3))
    r[:, 6:9] = rng.uniform(-14, 14, (n, 3))
    r[:, 9:54] = rng.normal(0, 0.1, (n, 45))
    r[:, 54] = rng.uniform(-8, 8, n)
    r[:, 55:58] = rng.uniform(-9, 2, (n, 3))
    r[:, 58:62] = rng.normal(size=(n, 4))
    r[0, 58:62] = 0.0
    r[1:9, 58] = -np.abs(r[1:9, 58])                                     # rot_0 = w < 0
    r[9, 55:58], r[10, 55:58] = 88.0, -88.0
    r[11, 54], r[12, 54] = 100.0, -100.0
    r[13, 6:9], r[14, 6:9] = 10.5, -10.5
    return r


def reference_linearize(raw):
    """ReorderSHs (f_rest channel-major -> per-coefficient RGB) then the reference's LinearizeDataJob."""
    L = M.ref_cs()
    if L is None:
        with np.load(M.GOLD / "ref_cs_linearize.npz") as f:
            assert np.array_equal(f["input"], raw)
            return f["output"]
    out = raw.copy()
    out[:, 9:54] = raw[:, 9:54].reshape(-1, 3, 15).transpose(0, 2, 1).reshape(-1, 45)
    L.ref_cs_linearize(out.ctypes.data, out.shape[0])
    return out


def _ulps(a, b):
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def test_ply_linearize_matches_the_reference(g, tmp_path):
    raw = linearize_records()
    path = tmp_path / "edge.ply"
    g.write_ply(str(path), raw)
    ours, ref = g.read_ply(str(path)), reference_linearize(raw)
    assert np.array_equal(ours[:, :9].view(np.uint32), ref[:, :9].view(np.uint32))          # position, normal: untouched
    assert np.array_equal(ours[:, 9:54].view(np.uint32), ref[:, 9:54].view(np.uint32))       # SH: reordered only
    # rotation: the packed smallest-three words exactly (the zero quaternion's NaNs as NaNs)
    rq_o, rq_r = ours[:, 58:62], ref[:, 58:62]
    assert np.array_equal(np.isnan(rq_o), np.isnan(rq_r)) and np.isnan(rq_r[0, :3]).all()
    ok = ~np.isnan(rq_r)
    assert np.array_equal(rq_o[ok].view(np.uint32), rq_r[ok].view(np.uint32))
    # exp-derived fields: libm expf against the managed (float)Math.Exp(double) -- within 2 ulp
    assert _ulps(ours[:, 55:58], ref[:, 55:58]).max() <= 2
    assert _ulps(ours[:, 54:55], ref[:, 54:55]).max() <= 2
    assert ref[11, 54] == 1.0 and ref[12, 54] == 0.0 and np.isfinite(ref[9, 55:58]).all() and (ref[10, 55:58] > 0).all()
    assert np.array_equal(ours[:, 6:9].view(np.uint32), ref[:, 6:9].view(np.uint32))        # SH0ToColor: no exp


# ---- the shim's stated third-party semantics -----------------------------------------------------------------------------
def _lib():
    L = M.ref_cs()
    if L is None:
        pytest.skip("oracle/_ref/libref_cs.so is not built (the reference's sources are absent)")
    return L


def test_shim_f32tof16_rounds_half_up_and_half3_converts_each_component():
    L = _lib()
    assert L.ref_cs_f32tof16(1.00048828125) == 0x3C01 and L.ref_cs_f32tof16(1.00146484375) == 0x3C02   # ties go up
    assert L.ref_cs_f32tof16(65504.0) == 0x7BFF and L.ref_cs_f32tof16(65520.0) == 0x7C00 and L.ref_cs_f32tof16(-0.0) == 0x8000
    assert L.ref_cs_f32tof16(float("nan")) & 0x7FFF == 0x7E00
    v = np.random.default_rng(2).uniform(-65504, 65504, 4000).astype(np.float32)
    got = np.array([L.ref_cs_f32tof16(float(x)) for x in v], np.uint32)
    rne = v.astype(np.float16).view(np.uint16).astype(np.uint32)
    tie = (v.view(np.uint32) & 0x1FFF) == 0x1000                        # normal halves: exactly half of bit 13 dropped
    assert np.array_equal(got[~tie], rne[~tie]) and (got[tie] >= rne[tie]).all()
    h = np.zeros(3, np.uint16)
    L.ref_cs_half3(np.array([1.00048828125, -2.0, 0.5], np.float32).ctypes.data, h.ctypes.data)
    assert h.tolist() == [0x3C01, 0xC000, 0x3800]


def test_shim_pow_is_managed_double_pow_narrowed():
    L = _lib()
    for x in (1e-40, 0.0, 1e30, 0.3, 2.0):
        assert L.ref_cs_pow(x, 0.125) == np.float32(float(np.float32(x)) ** 0.125)


def test_shim_min_max_saturate_on_nan_and_signed_zero():
    L = _lib()
    bits = lambda x: struct.pack("<f", x)  # noqa: E731
    nan = float("nan")
    assert bits(L.ref_cs_min(0.0, -0.0)) == bits(-0.0) and bits(L.ref_cs_min(-0.0, 0.0)) == bits(0.0)   # the second of equals
    assert bits(L.ref_cs_max(0.0, -0.0)) == bits(-0.0) and bits(L.ref_cs_max(-0.0, 0.0)) == bits(0.0)
    assert L.ref_cs_min(2.0, nan) == 2.0 and L.ref_cs_min(nan, 2.0) == 2.0                            # NaN is ignored
    assert L.ref_cs_max(2.0, nan) == 2.0 and L.ref_cs_max(nan, 2.0) == 2.0
    assert L.ref_cs_saturate(nan) == 1.0 and L.ref_cs_saturate(-3.0) == 0.0 and L.ref_cs_saturate(0.25) == 0.25


def test_shim_float_to_unsigned_truncates_in_range_and_marks_the_rest():
    import ctypes as C
    L = _lib()
    flag = C.c_int()
    for x, want in ((2047.99, 2047), (0.999, 0), (-0.5, 0), (4294967040.0, 4294967040)):
        assert L.ref_cs_to_uint(x, C.byref(flag)) == want and flag.value == 0
    for x in (float("nan"), -1.0, 4294967296.0):
        L.ref_cs_to_uint(x, C.byref(flag))
        assert flag.value == 1
    assert L.ref_cs_to_ulong(65535.9, C.byref(flag)) == 65535 and flag.value == 0


# ---- the fixtures ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(M.CASES) + ["linearize"])
def test_generator_reproduces_the_fixture_bytes(name):
    if M.ref_cs() is None:
        pytest.skip("oracle/_ref/libref_cs.so is not built (the reference's sources are absent)")
    with tempfile.TemporaryDirectory() as d:
        out = Path(d) / "f.npz"
        M.write_npz(out, linearize_fixture() if name == "linearize" else M.stored(name))
        want = M.GOLD / ("ref_cs_linearize.npz" if name == "linearize" else M.fixture(name).name)
        assert out.read_bytes() == want.read_bytes()


def linearize_fixture():
    raw = linearize_records()
    return {"input": raw, "output": reference_linearize(raw)}


if __name__ == "__main__":   # python tests/test_reference_cs.py: (re)write the linearize fixture
    M.write_npz(M.GOLD / "ref_cs_linearize.npz", linearize_fixture())
