"""gs_pack_asset / gs_kmeans on the GPU against the host packer (csrc/asset_creator.cpp, csrc/asset_cluster_bc7.cpp): the
same bytes for every preset and format, the same k-means means and labels, and an asset that renders like an uploaded one."""
import ctypes as C

import numpy as np
import pytest

from conftest import default_camera

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def P(g):
    from unitygaussiansplatting_b200 import pack
    return pack


def _host(g, splats, quality="Medium", formats=None):
    return g.create_asset(splats.copy(), quality, formats)


def _same(a, b):
    assert (a.splatCount, a.posFormat, a.scaleFormat, a.colorFormat, a.shFormat) == (b.splatCount, b.posFormat, b.scaleFormat,
                                                                                      b.colorFormat, b.shFormat)
    for name in ("posData", "otherData", "colorData", "shData", "chunkData"):
        x, y = getattr(a, name), getattr(b, name)
        assert (x is None) == (y is None), name
        if x is not None:
            assert x.nbytes == y.nbytes, name
            diff = np.flatnonzero(x != y)
            assert diff.size == 0, "%s differs at %d bytes, first at byte %d" % (name, diff.size, diff[0])
    assert np.array_equal(a.boundsMin.view(np.uint32), b.boundsMin.view(np.uint32))
    assert np.array_equal(a.boundsMax.view(np.uint32), b.boundsMax.view(np.uint32))


def _check(g, ctx, splats, quality="Medium", formats=None):
    before = splats.copy()
    gpu = g.pack_asset(splats, quality, formats, context=ctx)
    assert np.array_equal(splats.view(np.uint32), before.view(np.uint32)), "pack_asset modified its input"
    _same(gpu, _host(g, splats, quality, formats))
    return gpu


@pytest.mark.parametrize("quality", ["Medium", "High", "VeryHigh"])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_lossless_presets_match_host(g, ctx, quality, kind):
    _check(g, ctx, g.generate_input_splats(kind, 5001, 0x5EED0100 + kind), quality)


@pytest.mark.parametrize("quality", ["Medium", "High", "VeryHigh"])
def test_single_splat(g, ctx, quality):
    _check(g, ctx, g.generate_input_splats(1, 1, 7), quality)


@pytest.mark.parametrize("quality,n", [("VeryLow", 4097), ("Low", 16385)])
def test_clustered_presets_smallest_n(g, ctx, quality, n):
    _check(g, ctx, g.generate_input_splats(1, n, 0x5EED0200), quality)


@pytest.mark.parametrize("kind", [0, 2])
def test_verylow_other_scene_kinds(g, ctx, kind):
    _check(g, ctx, g.generate_input_splats(kind, 6000, 0x5EED0300 + kind), "VeryLow")


def test_verylow_300k(g, ctx):
    _check(g, ctx, g.generate_input_splats(1, 300_001, 0x5EED0400), "VeryLow")


# every vector, colour and SH format, including Float32 SH with chunks (the reference's inconsistent combination)
CUSTOM = [
    (0, 3, 2, 0),    # pos Float32, scale Norm6, Norm8x4, SH Float32 -> chunked
    (1, 2, 0, 1),    # Norm16, Norm11, Float32x4, Float16
    (3, 0, 1, 3),    # Norm6, Float32, Float16x4, Norm6
    (2, 1, 3, 2),    # Norm11, Norm16, BC7, Norm11
    (0, 0, 0, 7),    # all float, Cluster8k
]


@pytest.mark.parametrize("formats", CUSTOM)
def test_custom_formats_match_host(g, ctx, formats):
    n = 8193 if formats[3] > 3 else 2049
    _check(g, ctx, g.generate_input_splats(1, n, 0x5EED0500 + formats[3]), formats=formats)


def test_full_size_medium(g, ctx):
    _check(g, ctx, g.generate_input_splats(1, 6_131_954, 0x5EED0600), "Medium")


# ---- hazards -------------------------------------------------------------------------------------------------------------
def test_ties_and_signed_zeros(g, ctx):
    """Duplicate positions and +-0 everywhere: which of two equal values a min / max keeps depends on the order of the fold."""
    s = g.generate_input_splats(1, 5000, 0x5EED0700)
    rng = np.random.default_rng(3)
    s[1000:2000, 0:3] = s[0:1000, 0:3]                       # duplicated positions
    zero = rng.random((5000, 62)) < 0.2
    sign = np.where(rng.random((5000, 62)) < 0.5, np.float32(-0.0), np.float32(0.0))
    for cols in (slice(0, 3), slice(6, 9), slice(9, 54), slice(54, 55), slice(55, 58)):
        s[:, cols] = np.where(zero[:, cols], sign[:, cols], s[:, cols])
    s[4000:4256, 9:54] = rng.choice(np.array([0.0, -0.0, 0.25, -0.25], np.float32), (256, 45))
    for q in ("VeryLow", "Medium", "High"):
        _check(g, ctx, s, q)
    _check(g, ctx, s, formats=CUSTOM[0])


def test_all_splats_at_one_point(g, ctx):
    """Zero extent: inv = 1 / 0 = inf, every Morton code 0, order = input order."""
    s = g.generate_input_splats(2, 5000, 0x5EED0800)
    s[:, 0:3] = np.float32([1.5, -2.0, 0.25])
    for q in ("Medium", "VeryHigh", "VeryLow"):
        _check(g, ctx, s, q)


def _near_midpoint_scales(count, seed=5):
    """Float32 scales whose float64 s^(1/8) lies within 2^-45 (relative) of a float32 rounding midpoint -- the values the
    device lists for the host's std::pow.  Found by search: about one value in two million qualifies."""
    rng = np.random.default_rng(seed)
    found = []
    while len(found) < count:
        s = rng.uniform(1e-3, 2.0, 4_000_000).astype(np.float32)
        r = s.astype(np.float64) ** 0.125
        f = r.astype(np.float32)
        below = 0.5 * (f.astype(np.float64) + np.nextafter(f, np.float32(-np.inf)).astype(np.float64))
        above = 0.5 * (f.astype(np.float64) + np.nextafter(f, np.float32(np.inf)).astype(np.float64))
        tol = np.abs(r) * 2.0 ** -45
        found.extend(s[(np.abs(r - below) <= tol) | (np.abs(r - above) <= tol)].tolist())
    return np.array(found[:count], np.float32)


def test_pow_guard(g, ctx):
    from unitygaussiansplatting_b200 import pack
    special = _near_midpoint_scales(12)
    s = g.generate_input_splats(1, 4000, 0x5EED0900)
    s[::333, 55:58][: special.size // 3] = special[: (special.size // 3) * 3].reshape(-1, 3)
    _check(g, ctx, s, "Medium")
    stats = pack.pack_stats(ctx)
    assert stats[0] >= special.size // 3 * 3, "every near-midpoint scale must be recomputed on the host (%d)" % stats[0]


def test_nan_input_gives_well_formed_asset(g, ctx):
    s = g.generate_input_splats(1, 3000, 0x5EED0A00)
    s[5, 0] = np.nan
    s[17, 9:20] = np.inf
    s[300, 55] = np.nan
    a = g.pack_asset(s, "Medium", context=ctx)
    h = _host(g, s)
    for name in ("posData", "otherData", "colorData", "shData", "chunkData"):
        assert getattr(a, name).nbytes == getattr(h, name).nbytes


# ---- k-means -------------------------------------------------------------------------------------------------------------
def _kmeans_host(data, k, batch, passes):
    from unitygaussiansplatting_b200 import _native as N
    means = np.zeros((k, data.shape[1]), np.float32)
    labels = np.zeros(data.shape[0], np.int32)
    assert N.asset_lib().gsa_kmeans(data.shape[1], data.ctypes.data, data.shape[0], batch, passes, means.ctypes.data, k,
                                    labels.ctypes.data) == 0
    return means, labels


@pytest.mark.parametrize("n,k,dim,batch,passes", [(260, 7, 45, 64, 1.2), (3000, 37, 13, 256, 0.8), (50_000, 4096, 45, 2048, 1.2)])
def test_kmeans_matches_host(ctx, P, n, k, dim, batch, passes):
    rng = np.random.default_rng(n + dim)
    centres = rng.standard_normal((max(5, k // 8), dim)).astype(np.float32)
    data = (centres[rng.integers(0, centres.shape[0], n)] + 0.3 * rng.standard_normal((n, dim))).astype(np.float32)
    hm, hl = _kmeans_host(data, k, batch, passes)
    dm, dl = P.kmeans(data, k, batch, passes, context=ctx)
    assert np.array_equal(dl, hl)
    assert np.array_equal(dm.view(np.uint32), hm.view(np.uint32)), "centres must match to the bit"


# ---- end to end ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("quality", ["Medium", "VeryLow"])
def test_device_asset_renders_like_uploaded(g, ctx, quality):
    import torch
    s = g.generate_input_splats(1, 20000, 0x5EED0B00)
    t = torch.from_numpy(s.copy()).cuda()
    t_before = t.clone()
    packed, r_dev = g.pack_asset(t, quality, context=ctx, keep_on_device=True)
    assert torch.equal(t, t_before), "pack_asset modified its input tensor"
    host = _host(g, s, quality)
    _same(packed, host)
    r_up = g.GaussianSplatRenderer(host, ctx)
    for step in range(6):
        ang = step * 0.6
        cam = default_camera(g, 320, 200, pos=(6 * np.sin(ang), 0.5, -6 * np.cos(ang)), forward=(-np.sin(ang), 0.0, np.cos(ang)))
        rts = []
        for r in (r_dev, r_up):
            rt = np.zeros((200, 320, 4), np.float16)
            r.SortAndRenderSplats(cam, rt=rt)
            rts.append(rt)
        assert np.array_equal(r_dev.readback_order(), r_up.readback_order())
        assert np.array_equal(rts[0].view(np.uint16), rts[1].view(np.uint16))
        r_dev.CalcViewData(cam)
        r_up.CalcViewData(cam)
        assert np.array_equal(r_dev.readback_view(), r_up.readback_view())
    r_dev.Dispose()
    r_up.Dispose()


# ---- errors --------------------------------------------------------------------------------------------------------------
def test_errors_are_status_codes(g, ctx):
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    s = g.generate_input_splats(1, 100, 1)
    with pytest.raises(g.GsError) as e:
        g.pack_asset(s, formats=(4, 0, 0, 0), context=ctx)
    assert e.value.code == -4
    with pytest.raises(g.GsError) as e:
        g.pack_asset(s, "VeryLow", context=ctx)   # a 4k palette needs more than 4096 splats
    assert e.value.code == -4 and "palette" in str(e.value)
    d = N.GsPackDesc()
    d.splats, d.splat_count, d.memory = s.ctypes.data, 100, N.GS_MEM_HOST
    out = N.GsPackedAsset()
    assert lib.gs_pack_asset(ctx.handle, C.byref(d), C.byref(out), None) == -1 and lib.gs_last_error(ctx.handle)
    assert lib.gs_pack_asset(ctx.handle, None, C.byref(out), None) == -1
    assert lib.gs_pack_asset(None, C.byref(d), C.byref(out), None) == -1
    assert lib.gs_pack_asset(ctx.handle, C.byref(d), None, None) == -1
    d.splats = None
    h = C.c_void_p()
    assert lib.gs_pack_asset(ctx.handle, C.byref(d), None, C.byref(h)) == -1 and not h.value
    m = np.zeros((7, 45), np.float32)
    lab = np.zeros(5, np.int32)
    x = np.zeros((5, 45), np.float32)
    assert lib.gs_kmeans(ctx.handle, 45, x.ctypes.data, 5, 64, 1.2, m.ctypes.data, 7, lab.ctypes.data) == -1   # k > n
    assert lib.gs_kmeans(ctx.handle, 45, None, 5, 64, 1.2, m.ctypes.data, 7, lab.ctypes.data) == -1
    assert lib.gs_kmeans(ctx.handle, 200, x.ctypes.data, 5, 64, 1.2, m.ctypes.data, 1, lab.ctypes.data) == -1  # dim > 128
    assert b"dim" in lib.gs_last_error(ctx.handle)
