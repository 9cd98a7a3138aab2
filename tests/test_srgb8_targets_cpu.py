"""GS_PIX_R8G8B8A8_SRGB camera targets without a GPU: the codec's generated tables against 50-digit decimal arithmetic (every
decode entry, every encode threshold and the float32 just below it), the sRGB8 oracle (tests/srgb8_oracle.c) and the Python
codec at those places, on the specials and on random bit patterns, the oracle's composite against the CPU oracle's RGBA32F
composite followed by the encode, and the Python and C++ side's constant and image mapping."""
import re
import subprocess
from decimal import Decimal, getcontext
from pathlib import Path

import numpy as np
import pytest

import srgb8_oracle as S

ROOT = Path(__file__).resolve().parents[1]
TABLES = ROOT / "unitygaussiansplatting_b200" / "csrc" / "gs_srgb8_tables.h"
getcontext().prec = 50
D = Decimal


def eotf(v):
    return v / D("12.92") if v <= D("0.04045") else ((v + D("0.055")) / D("1.055")) ** D("2.4")


def oetf(x):
    return x * D("12.92") if x <= D("0.0031308") else D("1.055") * x ** (D(1) / D("2.4")) - D("0.055")


def exact(f):
    return D(float(np.float32(f)))


def below(f):
    return np.nextafter(np.float32(f), np.float32(-np.inf))


def above(f):
    return np.nextafter(np.float32(f), np.float32(np.inf))


def table(name):
    """A table of the generated header, as float32."""
    body = re.search(r"#define %s \{(.*?)\}" % name, TABLES.read_text(), re.S).group(1)
    return np.array([float.fromhex(t[:-1]) for t in re.findall(r"-?0x[0-9a-f.]+p[-+]\d+f", body)], np.float32)


@pytest.fixture(scope="module")
def L():
    return S.lib()


@pytest.fixture(scope="module")
def thresholds():
    t = table("GS_SRGB8_THRESHOLDS")
    assert t.size == 257 and t[0] == 0.0 and t[256] == 2.0   # the sentinels
    return t[1:256]                                          # T_1 .. T_255


def _f32_bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def test_decode_table_is_the_nearest_float_to_the_eotf(L):
    from unitygaussiansplatting_b200 import decode_srgb8
    dec = table("GS_SRGB8_DECODE")
    assert dec.size == 256
    for c in range(256):
        want = eotf(D(c) / D(255))
        f = dec[c]
        err = abs(exact(f) - want)
        assert err < abs(exact(below(f)) - want) and err < abs(exact(above(f)) - want), "entry %d" % c
    assert np.array_equal(_f32_bits([L.gso_srgb8_decode(c) for c in range(256)]), _f32_bits(dec)), "the oracle's decode"
    codes = np.arange(256, dtype=np.uint8)
    py = decode_srgb8(np.stack([codes, codes, codes, codes], -1))
    assert np.array_equal(_f32_bits(py[:, :3]), _f32_bits(np.repeat(dec[:, None], 3, 1))), "the Python decode"
    # alpha: the float32 nearest a / 255
    for a in range(256):
        f = np.float32(py[a, 3])
        assert abs(exact(f) - D(a) / D(255)) < abs(exact(below(f)) - D(a) / D(255)) and \
            abs(exact(f) - D(a) / D(255)) < abs(exact(above(f)) - D(a) / D(255)), "alpha %d" % a
        assert _f32_bits(L.gso_unorm8_decode(a)) == _f32_bits(f)


def test_every_threshold_and_the_float_below_it(L, thresholds):
    """T_j is the smallest float32 with 255 OETF(T_j) >= j - 0.5: it reaches the boundary, the float below does not, and the
    oracle and the Python codec step from j - 1 to j exactly there."""
    from unitygaussiansplatting_b200 import encode_srgb8
    assert np.all(np.diff(thresholds) > 0)
    for j, t in enumerate(thresholds, start=1):
        bound = (D(j) - D("0.5")) / D(255)
        assert oetf(exact(t)) >= bound, "T_%d does not reach its boundary" % j
        assert oetf(exact(below(t))) < bound, "the float below T_%d reaches its boundary" % j
        assert L.gso_srgb8_encode(float(t)) == j and L.gso_srgb8_encode(float(below(t))) == j - 1, "oracle at T_%d" % j
    xs = np.concatenate([thresholds, below(thresholds)])
    rgba = np.stack([xs, xs, xs, np.zeros_like(xs)], -1)
    got = encode_srgb8(rgba)[:, :3]
    want = np.concatenate([np.arange(1, 256), np.arange(0, 255)])
    assert np.array_equal(got, np.repeat(want[:, None], 3, 1).astype(np.uint8)), "the Python codec"


def test_no_boundary_in_the_junction_step(thresholds):
    """The OETF falls by 2.9e-8 at its junction; the nearest boundaries are T_10 and T_11, on either side of it."""
    J = D("0.0031308")
    drop = J * D("12.92") - (D("1.055") * J ** (D(1) / D("2.4")) - D("0.055"))
    assert D("2.8e-8") < drop < D("3.0e-8")
    xj = np.float32(0.0031308)   # the last float32 of the linear segment
    if exact(xj) > J:
        xj = below(xj)
    assert oetf(exact(above(xj))) < oetf(exact(xj))
    assert thresholds[9] < xj and above(xj) < thresholds[10]
    assert abs(float(oetf(exact(thresholds[9]))) - 0.0373) < 1e-4 and abs(float(oetf(exact(thresholds[10]))) - 0.0412) < 1e-4


def test_specials(L):
    from unitygaussiansplatting_b200 import encode_srgb8
    nan_payloads = np.array([0x7FC00000, 0x7F800001, 0x7FFFFFFF, 0xFFC00000, 0xFF800001, 0x7FA00000], np.uint32).view(np.float32)
    one = np.float32(1.0)
    cases = [(0.0, 0, 0), (-0.0, 0, 0), (np.inf, 255, 255), (-np.inf, 0, 0), (1.0, 255, 255), (2.0, 255, 255),
             (float(below(one)), 255, 255), (0.5, None, 128), (1e-45, 0, 0), (-1e-45, 0, 0), (1.1754942e-38, 0, 0),
             (float(np.float32(0.5 / 255)), None, 1), (float(below(np.float32(0.5 / 255))), None, 0)]
    for x in nan_payloads:
        cases.append((x, 0, 0))
    for x, rgb, a in cases:
        if rgb is not None:
            assert L.gso_srgb8_encode(float(x)) == rgb, x
        assert L.gso_unorm8_encode(float(x)) == a, x
    with np.errstate(invalid="ignore"):
        xs = np.array([c[0] for c in cases], np.float32)
        xs[-len(nan_payloads):] = nan_payloads
    got = encode_srgb8(np.stack([xs] * 4, -1))
    for (x, rgb, a), row in zip(cases, got):
        if rgb is not None:
            assert (row[:3] == rgb).all(), x
        assert row[3] == a, x
    # the float just below 1 is above T_255
    assert L.gso_srgb8_encode(float(below(one))) == 255
    # alpha rounds 255 x to nearest: 127.5 is the only representable tie
    assert L.gso_unorm8_encode(float(below(np.float32(0.5)))) == 127 and L.gso_unorm8_encode(float(above(np.float32(0.5)))) == 128


def test_python_codec_matches_the_oracle_on_random_bit_patterns(L):
    from unitygaussiansplatting_b200 import encode_srgb8
    rng = np.random.default_rng(0x5A6B)
    u = rng.integers(0, 2 ** 32, (200000, 4), dtype=np.uint64).astype(np.uint32)
    x = np.concatenate([u.view(np.float32), rng.random((100000, 4), np.float32), (rng.random((20000, 4)) * 0.01).astype(np.float32)], 0)
    got = encode_srgb8(x)
    want = np.concatenate([S.encode(x[:, :3]), S.encode(x[:, 3:], alpha=True)], -1)
    assert np.array_equal(got, want)


def test_srgb8_composite_is_the_float_composite_then_the_encode(O, L):
    from unitygaussiansplatting_b200 import decode_srgb8, encode_srgb8
    rng = np.random.default_rng(78)
    H, W = 37, 53
    rt = rng.random((H, W, 4), np.float32)
    rt[..., :3] *= rt[..., 3:]              # premultiplied
    rt[rng.random((H, W)) < 0.2, 3] = 0.0   # no coverage: the texel keeps its bytes
    rt[rng.random((H, W)) < 0.05, :] = 0.0
    rt[0, 0, 3] = np.nan
    rt[0, 1] = [0.0, 0.0, 0.0, 1.0]         # opaque black
    tgt = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
    tgt[1, :4] = [[0, 0, 0, 0], [255, 255, 255, 255], [1, 2, 3, 4], [254, 128, 127, 128]]
    got = S.composite_srgb8(rt, tgt)
    f = O.composite(rt, decode_srgb8(tgt))
    want = encode_srgb8(f)
    blended = rt[..., 3] > 0
    want = np.where(blended[..., None], want, tgt)
    assert np.array_equal(got, want)
    assert (got[~blended] == tgt[~blended]).all() and (got[blended] != tgt[blended]).any()


def test_header_constant_and_image_mapping():
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import CudaArrayImage, _image
    hdr = (ROOT / "include" / "gsplat_b200.h").read_text()
    assert int(re.search(r"GS_PIX_R8G8B8A8_SRGB\s*=\s*(\d+)", hdr).group(1)) == N.GS_PIX_R8G8B8A8_SRGB == 3
    host = np.zeros((6, 10, 4), np.uint8)
    im = _image(host, 10, 6)
    assert (im.format, im.memory, im.width, im.height, im.row_pitch_bytes, im.data) == (3, N.GS_MEM_HOST, 10, 6, 40, host.ctypes.data)
    a = CudaArrayImage(0x1000, 10, 6, np.uint8)
    assert a.shape == (6, 10, 4)
    im = _image(a, 10, 6)
    assert (im.format, im.memory, im.data, im.row_pitch_bytes) == (3, N.GS_MEM_ARRAY, 0x1000, 0)
    im = _image(CudaArrayImage(0x1000, 10, 6, np.uint8, layer=1), 10, 6)
    assert (im.format, im.memory) == (3, N.GS_MEM_ARRAY_LAYER)
    im = _image(CudaArrayImage(0x1000, 10, 6, np.uint8, layer=1, origin=(3, 4)), 10, 6)
    assert (im.format, im.memory) == (3, N.GS_MEM_ARRAY_RECT)
    # the other mappings and refusals stay as they were
    assert _image(np.zeros((6, 10, 4), np.float16), 10, 6).format == N.GS_PIX_RGBA16F
    assert _image(np.zeros((6, 10, 4), np.float32), 10, 6).format == N.GS_PIX_RGBA32F
    assert _image(np.zeros((6, 10), np.uint32), 10, 6).format == N.GS_PIX_B10G11R11_UFLOAT
    for bad in (np.zeros((6, 10, 4), np.uint32), np.zeros((6, 10, 4), np.int16), np.zeros((6, 10), np.uint8), np.zeros((6, 10, 3), np.uint8)):
        with pytest.raises(ValueError):
            _image(bad, 10, 6)
    with pytest.raises(ValueError):
        _image(CudaArrayImage(0x1000, 10, 6, np.uint8), 6, 10)
    with pytest.raises(ValueError):
        CudaArrayImage(0x1000, 10, 6, np.int8)


def test_torch_uint8_tensor_maps_to_srgb8():
    torch = pytest.importorskip("torch")
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    t = torch.zeros((6, 10, 4), dtype=torch.uint8)
    im = _image(t, 10, 6)
    assert (im.format, im.memory, im.row_pitch_bytes, im.data) == (N.GS_PIX_R8G8B8A8_SRGB, N.GS_MEM_HOST, 40, t.data_ptr())
    assert _image(torch.zeros((6, 10, 4), dtype=torch.float16), 10, 6).format == N.GS_PIX_RGBA16F
    assert _image(torch.zeros((6, 10, 4), dtype=torch.float32), 10, 6).format == N.GS_PIX_RGBA32F
    with pytest.raises(ValueError):
        _image(torch.zeros((6, 10), dtype=torch.uint8), 10, 6)


def test_host_mirror_builds_an_srgb8_camera_target(tmp_path):
    src = tmp_path / "srgb8.cpp"
    src.write_text(r'''
#include "unitygaussiansplatting_b200/host/GaussianSplatRenderer.hpp"
int main() {
  uint8_t px[6 * 4];
  const GsImage im = GaussianSplatting::Srgb8CameraTarget(px, 3, 2, GS_MEM_DEVICE, 16);
  const GsImage a = GaussianSplatting::ArrayImage(px, 3, 2, GS_PIX_R8G8B8A8_SRGB);
  const GsImage p = GaussianSplatting::PackedCameraTarget(px, 3, 2, GS_MEM_HOST);
  return (GS_PIX_R8G8B8A8_SRGB == 3 && im.data == px && im.width == 3 && im.height == 2 && im.row_pitch_bytes == 16 &&
          im.format == 3 && im.memory == GS_MEM_DEVICE && a.format == 3 && a.memory == GS_MEM_ARRAY && p.format == 2) ? 0 : 1;
}
''')
    exe = tmp_path / "srgb8"
    r = subprocess.run(["g++", "-std=c++17", "-I", str(ROOT), "-o", str(exe), str(src)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    assert subprocess.run([str(exe)]).returncode == 0
