"""GS_PIX_B10G11R11_UFLOAT camera targets without a GPU: the packed-target oracle's (tests/packed_oracle.c) float11 / float10
codec against a numpy restatement of the header's contract (every code, every value and midpoint between neighbours with one
float32 ulp either side, the specials and 10^6 random bit patterns), its packed composite against the CPU oracle's float
composite followed by the encode, and the Python and C++ side's constant and image mapping."""
import re
from pathlib import Path

import numpy as np
import pytest

import packed_oracle as P

ROOT = Path(__file__).resolve().parents[1]
M11, M10 = 6, 5


def np_decode(c, m):
    """The header's decode: exponent 0 denormal, 31 +Inf (mantissa 0) or NaN."""
    c = np.asarray(c, np.int64)
    e, mant = c >> m, c & ((1 << m) - 1)
    v = np.where(e == 0, np.ldexp(mant.astype(np.float64), -14 - m), np.ldexp((mant + (1 << m)).astype(np.float64), e - 15 - m))
    v = np.where(e == 31, np.where(mant == 0, np.inf, np.nan), v)
    return v.astype(np.float32)


def np_encode(x, m):
    """The header's encode, through exact rational arithmetic on float64: NaN all ones, <= 0 to 0, +Inf to Inf, else round to
    nearest even with IEEE overflow."""
    with np.errstate(invalid="ignore"):   # signalling NaNs among random bit patterns
        x = np.asarray(x, np.float32).astype(np.float64)
    inf = 31 << m
    out = np.zeros(x.shape, np.int64)
    pos = np.isfinite(x) & (x > 0)
    xp = np.where(pos, x, 1.0)
    e = np.maximum(np.floor(np.log2(xp)).astype(np.int64), -14)
    # floor(log2) of float64 may be off by one at the edges of a binade: correct it exactly
    e = np.where(np.ldexp(1.0, e) > xp, e - 1, e)
    e = np.where(np.ldexp(1.0, e + 1) <= xp, e + 1, e)
    e = np.maximum(e, -14)
    n = np.rint(np.ldexp(xp, m - e)).astype(np.int64)   # np.rint: ties to even
    code = ((e + 15) << m) + n - (1 << m)   # below 2^-13 (e = -14) this is n: denormals and the first binade alike
    out = np.where(pos, np.minimum(code, inf), out)
    out = np.where(np.isposinf(x), inf, out)
    out = np.where(np.isnan(x), inf | ((1 << m) - 1), out)
    return out.astype(np.uint32)


@pytest.fixture(scope="module")
def L():
    return P.lib()


def _enc(L, m):
    return L.gso_f32_to_uf11 if m == M11 else L.gso_f32_to_uf10


def _dec(L, m):
    return L.gso_uf11_to_f32 if m == M11 else L.gso_uf10_to_f32


def _f32_bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("m", [M11, M10], ids=["float11", "float10"])
def test_decode_every_code(L, m):
    codes = np.arange(1 << (m + 5), dtype=np.uint32)
    got = np.array([_dec(L, m)(int(c)) for c in codes], np.float32)
    want = np_decode(codes, m)
    nan = np.isnan(want)
    assert nan.sum() == (1 << m) - 1 and np.isnan(got[nan]).all()
    assert np.array_equal(_f32_bits(got[~nan]), _f32_bits(want[~nan]))
    # the quiet NaN keeps the mantissa, so that the device and the oracle agree bit for bit
    assert np.array_equal(_f32_bits(got[nan]), (0x7FC00000 | ((codes[nan] & ((1 << m) - 1)) << (23 - m))).astype(np.uint32))
    # round trip of every non-NaN code
    assert all(_enc(L, m)(float(v)) == c for c, v in zip(codes[~nan], want[~nan]))


@pytest.mark.parametrize("m", [M11, M10], ids=["float11", "float10"])
def test_encode_values_midpoints_and_their_neighbours(L, m):
    codes = np.arange(31 << m, dtype=np.uint32)   # every finite code
    vals = np_decode(codes, m).astype(np.float64)
    nxt = np.append(vals[1:], 2.0 ** 16)           # the value above the largest finite one is Inf's place, 2^16
    mids = ((vals + nxt) / 2).astype(np.float32)   # exact in float32: each midpoint needs one more mantissa bit
    assert np.array_equal(mids.astype(np.float64), (vals + nxt) / 2)
    xs = np.concatenate([vals.astype(np.float32), mids, np.nextafter(mids, np.float32(0)), np.nextafter(mids, np.float32(np.inf))])
    got = np.array([_enc(L, m)(float(x)) for x in xs], np.uint32)
    assert np.array_equal(got, np_encode(xs, m))
    # ties go to the even neighbour; one ulp either side to the nearer one
    n = codes.size
    mid_got, below, above = got[n:2 * n], got[2 * n:3 * n], got[3 * n:]
    assert np.array_equal(mid_got, np.where(codes % 2 == 0, codes, codes + 1))
    assert np.array_equal(below, codes) and np.array_equal(above, codes + 1)


def test_specials(L):
    e11, e10 = L.gso_f32_to_uf11, L.gso_f32_to_uf10
    for e, inf, maxf, over in ((e11, 0x7C0, 65024.0, 65280.0), (e10, 0x3E0, 64512.0, 65024.0)):
        m = 6 if e is e11 else 5
        assert e(0.0) == 0 and e(-0.0) == 0 and e(-1.0) == 0 and e(-1e-30) == 0 and e(float("-inf")) == 0
        assert e(float("inf")) == inf and e(float("nan")) == inf | ((1 << m) - 1)
        assert e(maxf) == inf - 1
        assert e(over) == inf and e(float(np.nextafter(np.float32(over), np.float32(0)))) == inf - 1
        assert e(1e30) == inf and e(3.4e38) == inf
        tiny = 2.0 ** (-14 - m)   # the smallest denormal
        assert e(tiny) == 1 and e(tiny / 2) == 0 and e(float(np.nextafter(np.float32(tiny / 2), np.float32(1)))) == 1
        assert e(2.0 ** -14) == 1 << m and e(2.0 ** -14 - tiny) == (1 << m) - 1
        assert e(1e-45) == 0   # a float32 denormal
    assert L.gso_uf11_to_f32(0x7C0) == float("inf") and L.gso_uf10_to_f32(0x3E0) == float("inf")
    assert L.gso_uf11_to_f32(0x7BF) == 65024.0 and L.gso_uf10_to_f32(0x3DF) == 64512.0


@pytest.mark.parametrize("m", [M11, M10], ids=["float11", "float10"])
def test_random_bit_patterns(L, m):
    u = np.random.default_rng(0xB10 + m).integers(0, 2 ** 32, 10 ** 6, dtype=np.uint64).astype(np.uint32)
    xs = u.view(np.float32)
    fn = _enc(L, m)
    got = np.fromiter((fn(float(x)) for x in xs), np.uint32, xs.size)
    assert np.array_equal(got, np_encode(xs, m))


def test_packed_composite_is_the_float_composite_then_the_encode(O, L):
    rng = np.random.default_rng(77)
    H, W = 37, 53
    rt = rng.random((H, W, 4), np.float32)
    rt[..., :3] *= rt[..., 3:]              # premultiplied
    rt[rng.random((H, W)) < 0.2, 3] = 0.0   # no coverage: the texel keeps its bits
    rt[rng.random((H, W)) < 0.05, :] = 0.0
    rt[0, 0, 3] = np.nan
    # random codes, with denormals, the largest finite values, Inf and NaN among them
    tgt = rng.integers(0, 2 ** 32, (H, W), dtype=np.uint64).astype(np.uint32)
    tgt[1, :8] = [0x001, 0x7BF | (0x7BF << 11) | (0x3DF << 22), 0x7C0, 0x7C0 << 11, 0x3E0 << 22, 0x7C3, 0x3FF << 22, 0]
    got = P.composite_b10g11r11(rt, tgt)
    rgb = np.stack([np_decode(tgt & 0x7FF, 6), np_decode((tgt >> 11) & 0x7FF, 6), np_decode(tgt >> 22, 5)], -1)
    f = O.composite(rt, np.concatenate([rgb, np.zeros((H, W, 1), np.float32)], -1))
    want = np_encode(f[..., 0], 6) | (np_encode(f[..., 1], 6) << 11) | (np_encode(f[..., 2], 5) << 22)
    blended = rt[..., 3] > 0
    want = np.where(blended, want, tgt)
    assert np.array_equal(got, want)
    assert (got[~blended] == tgt[~blended]).all() and (got[blended] != tgt[blended]).any()


def test_python_codec_matches_the_oracle(L):
    from unitygaussiansplatting_b200 import pack_b10g11r11, unpack_b10g11r11
    rng = np.random.default_rng(5)
    u = rng.integers(0, 2 ** 32, (3000, 3), dtype=np.uint64).astype(np.uint32)
    rgb = np.concatenate([u.view(np.float32), rng.random((3000, 3), np.float32) * 70000], 0)
    packed = pack_b10g11r11(rgb)
    want = np.array([L.gso_f32_to_uf11(float(r)) | (L.gso_f32_to_uf11(float(g)) << 11) | (L.gso_f32_to_uf10(float(b)) << 22)
                     for r, g, b in rgb], np.uint32)
    assert np.array_equal(packed, want)
    codes = rng.integers(0, 2 ** 32, 5000, dtype=np.uint64).astype(np.uint32)
    back = unpack_b10g11r11(codes)
    want = np.array([[L.gso_uf11_to_f32(int(c)), L.gso_uf11_to_f32(int(c) >> 11), L.gso_uf10_to_f32(int(c) >> 22)] for c in codes], np.float32)
    assert np.array_equal(_f32_bits(back), _f32_bits(want))


def test_header_constant_and_image_mapping():
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import CudaArrayImage, _image
    hdr = (ROOT / "include" / "gsplat_b200.h").read_text()
    assert int(re.search(r"GS_PIX_B10G11R11_UFLOAT\s*=\s*(\d+)", hdr).group(1)) == N.GS_PIX_B10G11R11_UFLOAT == 2
    host = np.zeros((6, 10), np.uint32)
    im = _image(host, 10, 6)
    assert (im.format, im.memory, im.width, im.height, im.row_pitch_bytes, im.data) == (2, N.GS_MEM_HOST, 10, 6, 40, host.ctypes.data)
    a = CudaArrayImage(0x1000, 10, 6, np.uint32)
    assert a.shape == (6, 10)
    im = _image(a, 10, 6)
    assert (im.format, im.memory, im.data, im.row_pitch_bytes) == (2, N.GS_MEM_ARRAY, 0x1000, 0)
    im = _image(CudaArrayImage(0x1000, 10, 6, np.uint32, layer=1, origin=(3, 4)), 10, 6)
    assert (im.format, im.memory) == (2, N.GS_MEM_ARRAY_RECT)
    # RGBA images are mapped as before; a wrong shape is refused
    assert _image(np.zeros((6, 10, 4), np.float16), 10, 6).format == N.GS_PIX_RGBA16F
    assert _image(np.zeros((6, 10, 4), np.float32), 10, 6).format == N.GS_PIX_RGBA32F
    with pytest.raises(ValueError):
        _image(np.zeros((6, 10, 4), np.uint32), 10, 6)
    with pytest.raises(ValueError):
        _image(CudaArrayImage(0x1000, 10, 6, np.uint32), 6, 10)
    with pytest.raises(ValueError):
        CudaArrayImage(0x1000, 10, 6, np.int16)


def test_host_mirror_builds_a_packed_camera_target(tmp_path):
    import subprocess
    src = tmp_path / "packed.cpp"
    src.write_text(r'''
#include "unitygaussiansplatting_b200/host/GaussianSplatRenderer.hpp"
int main() {
  uint32_t px[6];
  const GsImage im = GaussianSplatting::PackedCameraTarget(px, 3, 2, GS_MEM_HOST);
  const GsImage a = GaussianSplatting::ArrayImage(px, 3, 2, GS_PIX_B10G11R11_UFLOAT);
  return (GS_PIX_B10G11R11_UFLOAT == 2 && im.data == px && im.width == 3 && im.height == 2 && im.row_pitch_bytes == 0 &&
          im.format == 2 && im.memory == GS_MEM_HOST && a.format == 2 && a.memory == GS_MEM_ARRAY) ? 0 : 1;
}
''')
    exe = tmp_path / "packed"
    r = subprocess.run(["g++", "-std=c++17", "-I", str(ROOT), "-o", str(exe), str(src)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    assert subprocess.run([str(exe)]).returncode == 0
