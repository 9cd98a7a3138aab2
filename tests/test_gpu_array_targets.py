"""CUDA arrays as images (GS_MEM_ARRAY): what a graphics API's render texture looks like once it is imported into CUDA
(cudaExternalMemoryGetMappedMipmappedArray / cudaGraphicsSubResourceGetMappedArray).  The library renders into and composites
onto such an array in place, through surface objects.

Arrays are made by images.Cudart, through the CUDA runtime torch already loaded.  Every GPU test compares the array result
byte for byte with the same call on a torch device tensor: the linear path is pinned to the oracle elsewhere, so equality is the
parity contract."""
import ctypes as C
import re
import sys
from pathlib import Path

import numpy as np
import pytest

from images import KIND_FLOAT, KIND_UNSIGNED, SURFACE_LOAD_STORE, Image, bits, ca, to_device, to_host  # noqa: F401
from util import camera

ROOT = Path(__file__).resolve().parents[1]
GOLD = Path(__file__).parent / "golden"


def test_header_and_python_agree_on_gs_mem_array():
    from unitygaussiansplatting_b200 import _native as N
    text = (ROOT / "include" / "gsplat_b200.h").read_text()
    m = re.search(r"typedef enum GsMemory \{([^}]*)\} GsMemory;", text)
    assert m, "GsMemory enum not found in the header"
    values = dict((k, int(v)) for k, v in re.findall(r"(GS_MEM_\w+)\s*=\s*(\d+)", m.group(1)))
    assert values == {"GS_MEM_HOST": N.GS_MEM_HOST, "GS_MEM_DEVICE": N.GS_MEM_DEVICE, "GS_MEM_ARRAY": N.GS_MEM_ARRAY}
    assert N.GS_MEM_ARRAY == 2


def _noise(w, h, dtype=np.float16):
    """Random halves / floats: content every pixel of a render target must overwrite."""
    return np.random.default_rng(w * 7919 + h).random((h, w, 4), np.float32).astype(dtype)


def _lattice_case(g):
    sys.path.insert(0, str(GOLD))
    import make_golden
    kind, n, seed, quality, _w, _h, pos, sh = make_golden.CASES["lattice_1k_medium"]
    return g.synthetic_asset(kind, n, seed, quality), camera(g, 256, 256, pos=pos), sh


# ---- 1, 2: gs_frame into an array --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["lattice_1k_medium_256x256", "clustered_333x211"])
def test_frame_into_rgba16f_array_equals_tensor(g, O, ctx, ca, scene):
    if scene.startswith("lattice"):
        asset, cam, sh = _lattice_case(g)
    else:
        asset, cam, sh = g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED00A1, "Medium"), camera(g, 333, 211), 3
    h, w = cam.pixelHeight, cam.pixelWidth
    r = g.GaussianSplatRenderer(asset, ctx)
    r.m_SHOrder = sh
    t = to_device(np.zeros((h, w, 4), np.float16))
    r.SortAndRenderSplats(cam, rt=t)
    want = to_host(ctx, t)
    r.ResetOrder()
    im = Image(g, ca, "array", _noise(w, h))     # random content: every pixel must be overwritten
    r.SortAndRenderSplats(cam, rt=im.image)
    got = im.read(ctx)
    assert want.any()
    assert np.array_equal(bits(got), bits(want))
    if scene.startswith("lattice"):   # and straight against the oracle
        fp, _keep = g.make_frame_params(cam, sh_order=sh)
        ref = O.frame(asset, fp, threads=O.max_threads())
        assert np.array_equal(got.astype(np.float32), ref["rt"])
    r.Dispose()


@pytest.mark.gpu
def test_frame_into_rgba32f_array_fp32_blend_equals_tensor(g, ctx, ca):
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED00A2, "Medium")
    cam = camera(g, 333, 211)
    r = g.GaussianSplatRenderer(asset, ctx)
    r.blend_mode = 1
    t = to_device(np.zeros((211, 333, 4), np.float32))
    r.SortAndRenderSplats(cam, rt=t)
    want = to_host(ctx, t)
    r.ResetOrder()
    im = Image(g, ca, "array", _noise(333, 211, np.float32))
    r.SortAndRenderSplats(cam, rt=im.image)
    got = im.read(ctx)
    assert want.any() and np.array_equal(bits(got), bits(want))
    r.Dispose()


# ---- 3: GS_FLAG_LOAD_RT ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_renderers_share_one_array_render_target(g, ctx, ca):
    a = g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED0091, "Medium")
    b = g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0092, "VeryHigh")
    cam = camera(g, 400, 300)

    def draw(rt):
        ra, rb = g.GaussianSplatRenderer(a, ctx), g.GaussianSplatRenderer(b, ctx)
        ra.localToWorldMatrix = g.trs(position=(1.5, 0.0, 3.0)).astype(np.float32)
        rb.localToWorldMatrix = g.trs(position=(-1.0, 0.2, 0.5), scale=(0.7, 0.7, 0.7)).astype(np.float32)
        active = g.SortAndRenderSplatsMulti([ra, rb], cam, rt)
        assert active == [rb, ra]
        return ra, rb

    t = to_device(np.zeros((300, 400, 4), np.float16))
    keep = draw(t)
    want = to_host(ctx, t)
    im = Image(g, ca, "array", _noise(400, 300))
    keep += draw(im.image)
    got = im.read(ctx)
    assert want.any() and np.array_equal(bits(got), bits(want))
    for r in keep:
        r.Dispose()


# ---- 4: the extras variant (selection + scene depth) ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_selection_and_scene_depth_into_array(g, ctx, ca):
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 40000, 0x5EED00A4, "Medium")
    n = asset.splatCount
    sel = np.zeros((n + 31) // 32, np.uint32)
    ids = np.arange(0, n, 5)
    np.bitwise_or.at(sel, ids >> 5, np.uint32(1) << (ids & 31).astype(np.uint32))
    cam = camera(g, 400, 300)
    P = cam.gpuProjectionMatrix(True).astype(np.float64)
    clip = P @ np.array([0.0, 0.0, -6.0, 1.0])
    depth = np.zeros((300, 400), np.float32)
    depth[:, :240] = np.float32(clip[2] / clip[3])
    r = g.GaussianSplatRenderer(asset, ctx)
    r.m_SelectedBits, r.sceneDepth = sel, depth
    t = to_device(np.zeros((300, 400, 4), np.float16))
    r.SortAndRenderSplats(cam, rt=t)
    want = to_host(ctx, t)
    r.ResetOrder()
    im = Image(g, ca, "array", _noise(400, 300))
    r.SortAndRenderSplats(cam, rt=im.image)
    got = im.read(ctx)
    assert want.any() and np.array_equal(bits(got), bits(want))
    r.Dispose()


# ---- 5: staged calls -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_staged_render_into_array_equals_fused_frame(g, ctx, ca):
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED0006, "Medium")
    cam = camera(g, 300, 200)
    a, b = g.GaussianSplatRenderer(asset, ctx), g.GaussianSplatRenderer(asset, ctx)
    t = to_device(np.zeros((200, 300, 4), np.float16))
    a.SortAndRenderSplats(cam, rt=t)
    want = to_host(ctx, t)
    im = Image(g, ca, "array", _noise(300, 200))
    b.SortPoints(cam); b.CalcViewData(cam); b.DrawSplats(cam, im.image)
    got = im.read(ctx)
    assert want.any() and np.array_equal(bits(got), bits(want))
    a.Dispose(); b.Dispose()


# ---- 6: composite --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tgt_dtype", [np.float16, np.float32])
def test_composite_all_four_target_kinds(g, ctx, ca, tgt_dtype):
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0002, "Medium")
    cam = camera(g, 320, 200)
    r = g.GaussianSplatRenderer(asset, ctx)
    rt_t = to_device(np.zeros((200, 320, 4), np.float16))
    r.SortAndRenderSplats(cam, rt=rt_t)
    rt_np = to_host(ctx, rt_t)
    assert (rt_np[..., 3] == 0).any() and (rt_np[..., 3] > 0).any()   # both sides of the SrcAlpha == 0 early-out occur
    rt_a = Image(g, ca, "array", rt_np).image
    bg = np.random.default_rng(11).random((200, 320, 4), np.float32).astype(np.float16).astype(tgt_dtype)
    want = None
    for src in (rt_t, rt_a):
        for kind in ("tensor", "array"):
            tgt = Image(g, ca, "device" if kind == "tensor" else "array", bg)
            r.Composite(src, tgt.image)
            got = tgt.read(ctx)
            if want is None:
                want = got
                untouched = rt_np[..., 3] == 0
                assert np.array_equal(bits(got)[untouched], bits(bg)[untouched]) and not np.array_equal(got, bg)
            assert np.array_equal(bits(got), bits(want)), "rt %s, target %s" % ("tensor" if src is rt_t else "array", kind)
    # gs_frame with an array camera target, with the render target in library scratch and with an array render target
    for with_rt in (False, True):
        r.ResetOrder(); r.m_FrameCounter = 0
        tgt = Image(g, ca, "array", bg)
        rt = Image(g, ca, "array", _noise(320, 200)) if with_rt else None
        r.SortAndRenderSplats(cam, rt=rt and rt.image, camera_target=tgt.image)
        assert np.array_equal(bits(tgt.read(ctx)), bits(want)), "gs_frame, rt %s" % ("array" if with_rt else "scratch")
        if with_rt:
            assert np.array_equal(bits(rt.read(ctx)), bits(rt_np))
    r.Dispose()


# ---- 7: row ranges ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_row_range_into_array_keeps_other_rows(g, ctx, ca):
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED00A7, "Medium")
    cam = camera(g, 333, 211)
    r = g.GaussianSplatRenderer(asset, ctx)
    full_t = to_device(np.zeros((211, 333, 4), np.float16))
    r.SortAndRenderSplats(cam, rt=full_t)
    full = to_host(ctx, full_t)
    sentinel = np.float16(-7.5)
    r.rows = (3, 11)                          # 16-pixel rows 3..10: pixel rows [48, 176)
    r.ResetOrder(); r.m_FrameCounter = 0
    t = to_device(np.full((211, 333, 4), sentinel))
    r.SortAndRenderSplats(cam, rt=t)
    want = to_host(ctx, t)
    r.ResetOrder(); r.m_FrameCounter = 0
    im = Image(g, ca, "array", np.full((211, 333, 4), sentinel))
    r.SortAndRenderSplats(cam, rt=im.image)
    got = im.read(ctx)
    assert np.array_equal(bits(got), bits(want))
    assert np.array_equal(bits(got[48:176]), bits(full[48:176])) and full[48:176].any()
    assert (got[:48] == sentinel).all() and (got[176:] == sentinel).all()
    r.Dispose()


# ---- 8: the Unity render-thread event ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_unity_event_with_array_rt_equals_direct_frame(g, ctx, ca):
    from unitygaussiansplatting_b200 import _native as N
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0051, "Medium")
    cam = camera(g, 200, 150)
    r = g.GaussianSplatRenderer(asset, ctx)
    direct = np.zeros((150, 200, 4), np.float16)
    r.SortAndRenderSplats(cam, rt=direct)
    r.ResetOrder()
    im = Image(g, ca, "array", _noise(200, 150))
    fp, _keep = g.make_frame_params(cam, r.localToWorldMatrix, r.m_SplatScale, r.m_OpacityScale, r.m_SHOrder, r.m_SHOnly)
    ev = N.GsUnityFrameEvent()
    ev.ctx, ev.asset = C.cast(ctx.handle, C.c_void_p).value, C.cast(r._asset, C.c_void_p).value
    C.memmove(C.byref(ev.params), C.byref(fp), C.sizeof(fp))
    ev.options.blend_mode = 0
    ev.do_sort, ev.status = 1, -5
    ev.has_rt, ev.has_camera_target = 1, 0
    ev.rt.data, ev.rt.width, ev.rt.height = im.image.handle, 200, 150
    ev.rt.row_pitch_bytes, ev.rt.format, ev.rt.memory = 0, N.GS_PIX_RGBA16F, N.GS_MEM_ARRAY
    fn = N.native().gs_unity_get_render_event_func()
    fn(N.GS_UNITY_EVENT_FRAME, C.addressof(ev))
    assert ev.status == 0
    fn(N.GS_UNITY_EVENT_SYNC, C.addressof(ev))
    assert ev.status == 0
    got = im.read(ctx)
    assert direct.any() and np.array_equal(bits(got), bits(direct))
    r.Dispose()


# ---- 9: groups -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("members", [2, 3])
def test_emulated_group_with_array_members_equals_one_gpu(g, ctx, ca, members):
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 40000, 0x5EED00A9, "Medium")
    cam = camera(g, 400, 300)
    r = g.GaussianSplatRenderer(asset, ctx)
    want = np.zeros((300, 400, 4), np.float16)
    r.SortAndRenderSplats(cam, rt=want)
    r.Dispose()
    grp = GaussianSplatGroup.create(asset, [0] * members, emulate=True)
    arrays = [Image(g, ca, "array", _noise(400, 300)) for _ in range(members - 1)]   # rts[0] (and rts[1] for 3 members)
    rest = [np.zeros_like(want)]
    grp.SortAndRenderSplats(cam, rts=[im.image for im in arrays] + rest)
    grp.sync()
    assert want.any()
    for im in arrays:
        assert np.array_equal(bits(im.read(ctx)), bits(want))
    assert np.array_equal(bits(rest[0]), bits(want))
    grp.close()


# ---- 10: rejections ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_array_rejections_leave_the_array_untouched(g, ctx, ca):
    import torch
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED00AA, "Medium")
    cam = camera(g, 128, 128)
    r = g.GaussianSplatRenderer(asset, ctx)
    fp = r.frame_params(cam)

    def frame(handle, fmt=N.GS_PIX_RGBA16F, memory=N.GS_MEM_ARRAY, pitch=0, band_packed=0):
        im = N.GsImage(handle, 128, 128, pitch, fmt, memory)
        opt = r._options()
        opt.band_packed = band_packed
        return lib.gs_frame(ctx.handle, r._asset, C.byref(fp), C.byref(opt), 1, C.byref(im), None)

    pattern = np.random.default_rng(3).random((128, 128, 4), np.float32).astype(np.float16)

    def filled(width=128, kind=KIND_FLOAT, flags=SURFACE_LOAD_STORE, fill=pattern):
        return ca.array(width, 128, dtype=fill.dtype, flags=flags, kind=kind, fill=fill)

    def unchanged(h, fill=pattern):
        return np.array_equal(ca.download(h).view(np.uint8), fill.view(np.uint8))

    bytes8 = np.random.default_rng(4).integers(0, 256, (128, 128, 4), np.uint8)
    h = filled(kind=KIND_UNSIGNED, fill=bytes8)                               # uint8 x 4
    assert frame(h) == -4 and "channel format" in lib.gs_last_error(ctx.handle).decode()
    ctx.sync()
    assert unchanged(h, bytes8)
    wide = np.concatenate([pattern, pattern[:, :1]], axis=1)
    h = filled(width=129, fill=wide)                                           # 129 x 128 for a 128 x 128 image
    assert frame(h) == -1
    ctx.sync()
    assert unchanged(h, wide)
    no_surface = filled(flags=0)                                               # no cudaArraySurfaceLoadStore
    assert frame(no_surface) == -1 and "cudaArraySurfaceLoadStore" in lib.gs_last_error(ctx.handle).decode()
    good = filled()
    assert frame(good, pitch=128 * 8) == -1                                    # non-zero pitch
    assert frame(good, memory=3) == -1                                         # unknown memory kind
    opt = r._options()                                                         # band-packed output (all of one partition's rows)
    opt.partition_index, opt.partition_count, opt.band_rows, opt.band_packed = 0, 2, 1, 1
    im = N.GsImage(good, 128, 64, 0, N.GS_PIX_RGBA16F, N.GS_MEM_ARRAY)
    assert lib.gs_frame(ctx.handle, r._asset, C.byref(fp), C.byref(opt), 1, C.byref(im), None) == -1
    assert "band_packed" in lib.gs_last_error(ctx.handle).decode()
    gathered = torch.zeros((2, 64, 128, 4), dtype=torch.float16, device="cuda")   # gs_unshuffle_bands into an array
    im = N.GsImage(good, 128, 128, 0, N.GS_PIX_RGBA16F, N.GS_MEM_ARRAY)
    assert lib.gs_unshuffle_bands(ctx.handle, C.c_void_p(gathered.data_ptr()), 2, 1, 64, N.GS_PIX_RGBA16F, C.byref(im)) == -1
    ctx.sync()
    assert unchanged(good) and unchanged(no_surface)
    # and the same array, correctly described, is accepted
    assert frame(good) == 0
    ctx.sync()
    assert not unchanged(good)
    r.Dispose()
