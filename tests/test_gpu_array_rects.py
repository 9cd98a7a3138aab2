"""A rectangle of a CUDA array as an image or a depth buffer (GS_MEM_ARRAY_RECT): an HDRP render target allocated larger than
the camera, whose camera draws into the rectangle at its origin, and the tiles of an atlas or a light-field quilt, one per
camera.  The library draws into, composites onto and depth-tests against the rectangle in place, and leaves every texel
outside it, and every other layer, as it was.

Arrays are made by images.Cudart, and several images in one array are an images.SharedArray.  Every result inside a rectangle is compared
byte for byte with the same call on linear device memory (or, for several cameras, with the camera loop it stands for), and
every texel outside the rectangles is checked to still hold its sentinel."""
import ctypes as C

import numpy as np
import pytest

from frame_loops import call_cameras, frame_args
from images import SENTINEL, SURFACE_LOAD_STORE, SharedArray, background, bits, ca, check_regions, launches, to_device, to_host  # noqa: F401
from util import camera

INVALID, UNSUPPORTED = -1, -4
W, H = 200, 120    # a screen that is not a multiple of 16 on either axis
# (array width, array height, x, y): at the origin of a larger array, at an odd offset, flush with the far corner
PLACEMENTS = {"origin": (301, 157, 0, 0), "odd": (301, 157, 37, 19), "far-corner": (301, 157, 101, 37)}


def _assets(g):
    return (g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED0E01, "Medium"),
            g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0E02, "VeryHigh"))


# ---- 1. every single-camera entry point, at every placement, in a 2-D array and in a layer ------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,blend", [(np.float16, 0), (np.float16, 1), (np.float32, 0), (np.float32, 1)],
                         ids=["rgba16f-rop", "rgba16f-fp32", "rgba32f-rop", "rgba32f-fp32"])
def test_rect_equals_linear_target(g, ctx, ca, dtype, blend):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    a, b = _assets(g)
    cam = camera(g, W, H)
    bg = background(H, W, dtype, 5)
    zeros = np.zeros((H, W, 4), dtype)
    sel = np.zeros((a.splatCount + 31) // 32, np.uint32)
    sel[::5] = 0x00FF00FF

    def renderer(asset, **kn):
        r = g.GaussianSplatRenderer(asset, ctx)
        r.blend_mode = blend
        for key, v in kn.items():
            setattr(r, key, v)
        return r

    r = renderer(a)
    r2 = renderer(b, localToWorldMatrix=g.trs(position=(-1.0, 0.2, 0.5)).astype(np.float32))
    ra, rb = renderer(a), renderer(b, localToWorldMatrix=g.trs(position=(1.5, 0.0, 3.0)).astype(np.float32))

    def frame(rt, tg=None, selected=None):
        r.m_SelectedBits = selected
        r.ResetOrder()
        r.SortAndRenderSplats(cam, rt=rt, camera_target=tg)
        r.m_SelectedBits = None

    def load(rt):
        r2.load_rt = True
        r2.ResetOrder()
        r2.SortAndRenderSplats(cam, rt=rt)
        r2.load_rt = False

    def objects(rt, tg):
        for x in (ra, rb):
            x.ResetOrder()
            x.m_FrameCounter = 0
        assert g.renderer.draws_in_one_call(g.GatherSplatsForCamera([ra, rb], cam))
        g.SortAndRenderSplatsMulti([ra, rb], cam, rt, tg)

    def counted(fn, *args):
        n0 = launches(ctx)
        fn(*args)
        return launches(ctx) - n0

    ctx.set_timing(True)
    try:
        # the definitions, on linear device memory, and the launches of the same calls on whole 2-D arrays
        t = to_device(zeros); frame(t); want_f = to_host(ctx, t)
        t = to_device(zeros); frame(t, selected=sel); want_sel = to_host(ctx, t)
        t = to_device(want_f); load(t); want_load = to_host(ctx, t)
        t, tg = to_device(zeros), to_device(bg); frame(t, tg); want_ftg = (to_host(ctx, t), to_host(ctx, tg))
        t, tg = to_device(zeros), to_device(bg); objects(t, tg); want_obj = (to_host(ctx, t), to_host(ctx, tg))
        assert want_f.any() and not np.array_equal(bits(want_sel), bits(want_f)) and not np.array_equal(bits(want_load), bits(want_f))
        whole = SharedArray(g, ca, W, H, 0, dtype)
        whole.fill(0, 0, 0, want_f)
        n_load_whole = counted(load, g.CudaArrayImage(whole.handle, W, H, dtype))
        whole_tg = SharedArray(g, ca, W, H, 0, dtype)
        whole_tg.fill(0, 0, 0, bg)
        n_obj_whole = counted(objects, g.CudaArrayImage(whole.handle, W, H, dtype), g.CudaArrayImage(whole_tg.handle, W, H, dtype))

        for pname, (aw, ah, x, y) in PLACEMENTS.items():
            for layers, k in ((0, None), (3, 1)):
                what = "%s, %s" % (pname, "layer %d" % k if layers else "2-D")
                A = SharedArray(g, ca, aw, ah, layers, dtype)
                frame(A.view(k, (x, y), (W, H)))
                A.check(ctx, [(k, x, y, want_f)], "gs_frame " + what)
                A = SharedArray(g, ca, aw, ah, layers, dtype)
                frame(A.view(k, (x, y), (W, H)), selected=sel)
                A.check(ctx, [(k, x, y, want_sel)], "gs_frame with a selection " + what)
                A = SharedArray(g, ca, aw, ah, layers, dtype)
                A.fill(k, x, y, want_f)
                assert counted(load, A.view(k, (x, y), (W, H))) == n_load_whole, what
                A.check(ctx, [(k, x, y, want_load)], "GS_FLAG_LOAD_RT " + what)
                A, B = SharedArray(g, ca, aw, ah, layers, dtype), SharedArray(g, ca, aw, ah, layers, dtype)
                B.fill(k, x, y, bg)
                frame(A.view(k, (x, y), (W, H)), B.view(k, (x, y), (W, H)))
                A.check(ctx, [(k, x, y, want_ftg[0])], "gs_frame rt " + what)
                B.check(ctx, [(k, x, y, want_ftg[1])], "gs_frame camera target " + what)
                A, B = SharedArray(g, ca, aw, ah, layers, dtype), SharedArray(g, ca, aw, ah, layers, dtype)
                B.fill(k, x, y, bg)
                assert counted(objects, A.view(k, (x, y), (W, H)), B.view(k, (x, y), (W, H))) == n_obj_whole, what
                A.check(ctx, [(k, x, y, want_obj[0])], "gs_frame_objects rt " + what)
                B.check(ctx, [(k, x, y, want_obj[1])], "gs_frame_objects camera target " + what)

        # staged gs_render, then gs_composite, with rt and camera target disjoint rectangles of one array
        t = to_device(zeros)
        r.ResetOrder(); r.SortPoints(cam); r.CalcViewData(cam); r.DrawSplats(cam, t)
        want_r = to_host(ctx, t)
        tg = to_device(bg)
        r.Composite(t, tg)
        want_c = to_host(ctx, tg)
        for layers, k in ((0, None), (3, 2)):
            A = SharedArray(g, ca, 420, 130, layers, dtype)
            A.fill(k, 211, 7, bg)
            rt_im, tg_im = A.view(k, (3, 5), (W, H)), A.view(k, (211, 7), (W, H))
            r.ResetOrder(); r.SortPoints(cam); r.CalcViewData(cam); r.DrawSplats(cam, rt_im)
            r.Composite(rt_im, tg_im)
            A.check(ctx, [(k, 3, 5, want_r), (k, 211, 7, want_c)], "gs_render + gs_composite, %d layers" % layers)

        # the Unity render-thread event (gs_frame) with a GS_MEM_ARRAY_RECT render target
        fp, _keep = g.make_frame_params(cam, r.localToWorldMatrix, r.m_SplatScale, r.m_OpacityScale, r.m_SHOrder, r.m_SHOnly)
        A = SharedArray(g, ca, 301, 157, 0, dtype)
        rt_im = _image(A.view(None, (37, 19), (W, H)), W, H)   # points to the rectangle's descriptor, which rt_im keeps alive
        ev = N.GsUnityFrameEvent()
        ev.ctx, ev.asset = C.cast(ctx.handle, C.c_void_p).value, C.cast(r._asset, C.c_void_p).value
        C.memmove(C.byref(ev.params), C.byref(fp), C.sizeof(fp))
        ev.options.blend_mode = blend
        ev.do_sort, ev.status, ev.has_rt, ev.has_camera_target = 1, -5, 1, 0
        ev.rt = rt_im
        r.ResetOrder()
        fn = N.native().gs_unity_get_render_event_func()
        fn(N.GS_UNITY_EVENT_FRAME, C.addressof(ev))
        assert ev.status == 0
        fn(N.GS_UNITY_EVENT_SYNC, C.addressof(ev))
        assert ev.status == 0
        A.check(ctx, [(0, 37, 19, want_f)], "Unity event")
    finally:
        ctx.set_timing(False)
    for x in (r, r2, ra, rb):
        x.Dispose()


# ---- 2. a quilt: several cameras in disjoint tiles of one array, one camera run --------------------------------------------------
# (x, y, w, h) of each camera's tile: three 128 x 96 views above three 96 x 64 views
TILES = [(0, 0, 128, 96), (130, 0, 128, 96), (260, 0, 128, 96), (0, 100, 96, 64), (100, 100, 96, 64), (200, 100, 96, 64)]


def _quilt_cameras(g):
    return [camera(g, w, h, pos=(-0.6 + 0.24 * i, 0.5 + 0.05 * (i % 2), -6.0 + 0.2 * i), forward=(0.1 * (i - 2.5), 0.0, 1.0))
            for i, (_, _, w, h) in enumerate(TILES)]


def _quilt_renderers(g, ctx, assets):
    rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]
    rs[1].localToWorldMatrix = g.trs(position=(-0.6, 0.1, 0.2)).astype(np.float32)
    return rs


@pytest.mark.gpu
@pytest.mark.parametrize("layered", [False, True], ids=["2-D", "layer"])
def test_quilt_is_one_camera_run(g, ctx, ca, layered):
    assets = _assets(g)
    cams = _quilt_cameras(g)
    layers, k = (3, 1) if layered else (0, None)
    bgs = [background(h, w, np.float16, 20 + i) for i, (_, _, w, h) in enumerate(TILES)]
    ctx.set_timing(True)
    try:
        # the definition: the camera loop, gs_frame_objects per camera into images of its own
        loop = _quilt_renderers(g, ctx, assets)
        rts = [to_device(np.zeros((h, w, 4), np.float16)) for (_, _, w, h) in TILES]
        tgs = [to_device(bg) for bg in bgs]
        n0 = launches(ctx)
        for c, cam in enumerate(cams):
            assert len(g.SortAndRenderSplatsMulti(loop, cam, rts[c], tgs[c])) == 2
        n_loop = launches(ctx) - n0
        want_rt, want_tg = [to_host(ctx, t) for t in rts], [to_host(ctx, t) for t in tgs]
        want_order = [r.readback_order() for r in loop]
        assert all(x.any() for x in want_rt)

        # the same cameras in one gs_frame_cameras call into separate arrays
        sep = _quilt_renderers(g, ctx, assets)
        sep_rt = [SharedArray(g, ca, w, h, 0) for (_, _, w, h) in TILES]
        sep_tg = [SharedArray(g, ca, w, h, 0) for (_, _, w, h) in TILES]
        for t, bg in zip(sep_tg, bgs):
            t.fill(0, 0, 0, bg)
        n0 = launches(ctx)
        actives = g.SortAndRenderCameras(sep, cams, [a.view(None, (0, 0), (a.w, a.h)) for a in sep_rt], [a.view(None, (0, 0), (a.w, a.h)) for a in sep_tg])
        n_sep = launches(ctx) - n0
        assert g.renderer.cameras_in_one_call(actives)

        # and into the tiles of one colour array, with the camera targets in the tiles of another
        call = _quilt_renderers(g, ctx, assets)
        A, B = SharedArray(g, ca, 400, 170, layers), SharedArray(g, ca, 400, 170, layers)
        for (x, y, _, _), bg in zip(TILES, bgs):
            B.fill(k, x, y, bg)
        n0 = launches(ctx)
        g.SortAndRenderCameras(call, cams, [A.view(k, (x, y), (w, h)) for (x, y, w, h) in TILES],
                               [B.view(k, (x, y), (w, h)) for (x, y, w, h) in TILES])
        n_call = launches(ctx) - n0
        A.check(ctx, [(k, x, y, want) for (x, y, _, _), want in zip(TILES, want_rt)], "quilt render targets")
        B.check(ctx, [(k, x, y, want) for (x, y, _, _), want in zip(TILES, want_tg)], "quilt camera targets")
        for r, o in zip(call, want_order):
            assert np.array_equal(r.readback_order(), o), "draw order differs"
        assert n_call == n_sep < n_loop, (n_call, n_sep, n_loop)
        for r in loop + sep + call:
            r.Dispose()
    finally:
        ctx.set_timing(False)


@pytest.mark.gpu
@pytest.mark.parametrize("first", ["rect", "whole"])
def test_intersecting_rects_are_the_camera_loop(g, ctx, ca, first):
    """Two cameras whose render targets share texels: the second starts a new run and draws over the first, as the loop does.
    first = "whole": the first camera's target is the whole array, which intersects every rectangle of it."""
    assets = _assets(g)
    if first == "rect":
        aw, ah, tiles = 200, 150, [(0, 0, 128, 96), (64, 48, 128, 96)]
    else:
        aw, ah, tiles = 128, 96, [(0, 0, 128, 96), (16, 8, 96, 64)]
    cams = [camera(g, w, h, pos=(0.3 * i, 0.5, -6.0)) for i, (_, _, w, h) in enumerate(tiles)]

    def images(A):
        ims = [A.view(None, (x, y), (w, h)) for (x, y, w, h) in tiles]
        if first == "whole":
            ims[0] = g.CudaArrayImage(A.handle, aw, ah)
        return ims

    ctx.set_timing(True)
    try:
        loop = _quilt_renderers(g, ctx, assets)
        L = SharedArray(g, ca, aw, ah)
        n0 = launches(ctx)
        for cam, im in zip(cams, images(L)):
            g.SortAndRenderSplatsMulti(loop, cam, im)
        n_loop = launches(ctx) - n0
        ctx.sync()
        want = L.read(ctx)
        call = _quilt_renderers(g, ctx, assets)
        A = SharedArray(g, ca, aw, ah)
        n0 = launches(ctx)
        g.SortAndRenderCameras(call, cams, images(A))
        n_call = launches(ctx) - n0
        ctx.sync()
        assert np.array_equal(bits(A.read(ctx)), bits(want))
        assert n_call == n_loop, (n_call, n_loop)
        for r, q in zip(loop, call):
            assert np.array_equal(r.readback_order(), q.readback_order())
        for r in loop + call:
            r.Dispose()
    finally:
        ctx.set_timing(False)


# ---- 3. scene depth in a rectangle -----------------------------------------------------------------------------------------------
def _wall(g, cam, w, h):
    clip = cam.gpuProjectionMatrix(True).astype(np.float64) @ np.array([0.0, 0.0, -6.0, 1.0])
    depth = np.zeros((h, w), np.float32)
    depth[:, :int(w * 0.6)] = np.float32(clip[2] / clip[3])
    depth[::37, ::23] = np.nan
    return depth


@pytest.mark.gpu
def test_depth_rect_equals_tensor_depth(g, ctx, ca):
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 40000, 0x5EED0095, "Medium")
    cam = camera(g, W, H)
    depth = _wall(g, cam, W, H)
    x, y = 37, 19
    # the rest of every depth array holds 1.0, which hides every splat: a wrong offset or layer shows
    flat, layered = SharedArray(g, ca, 301, 157, 0, np.float32, "depth", 1.0), SharedArray(g, ca, 301, 157, 3, np.float32, "depth", 1.0)
    flat.fill(None, x, y, depth)
    layered.fill(2, x, y, depth)
    r = g.GaussianSplatRenderer(asset, ctx)

    def draw(d):
        r.sceneDepth = d
        r.ResetOrder()
        t = to_device(np.zeros((H, W, 4), np.float16))
        r.SortAndRenderSplats(cam, rt=t)
        return to_host(ctx, t)

    want = draw(to_device(depth))
    assert not np.array_equal(bits(want), bits(draw(None))), "the wall hides nothing"
    for d in (flat.view(None, (x, y), (W, H)), layered.view(2, (x, y), (W, H))):
        assert np.array_equal(bits(draw(d)), bits(want))
    assert not draw(layered.view(1, (x, y), (W, H))).any()

    # two cameras of one gs_frame_cameras call, each depth-tested against its tile of one depth array
    cams = [camera(g, W, H, pos=(s * 0.032, 0.5, -6.0)) for s in (-1, 1)]
    depths = [_wall(g, c, W, H) for c in cams]
    depths[1] = np.ascontiguousarray(depths[1][:, ::-1])
    tiles = [(0, 0), (210, 30)]
    atlas = SharedArray(g, ca, 420, 160, 0, np.float32, "depth", 1.0)
    for (tx, ty), d in zip(tiles, depths):
        atlas.fill(None, tx, ty, d)

    def cameras(ds):
        ts = [to_device(np.zeros((H, W, 4), np.float16)) for _ in cams]
        r.ResetOrder()
        assert call_cameras(g, ctx, [[r], [r]], cams, 0, ts, [None, None], [[{"scene_depth": d}] for d in ds], check=False) == 0
        return [to_host(ctx, t) for t in ts]

    want = cameras([to_device(d) for d in depths])
    got = cameras([atlas.view(None, t, (W, H)) for t in tiles])
    for e in range(2):
        assert np.array_equal(bits(got[e]), bits(want[e])), "camera %d" % e
    r.Dispose()


# ---- 4. groups -------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_emulated_group_into_rects_equals_one_gpu(g, ctx, ca):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    assets = _assets(g)
    mats = [g.trs(position=(0.3, 0.0, 1.0)).astype(np.float32), g.trs(position=(-0.6, 0.1, 0.2)).astype(np.float32)]
    cam = camera(g, W, H)
    bg = background(H, W, np.float16, 13)
    rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]
    for r, m in zip(rs, mats):
        r.localToWorldMatrix = m
    rt, tg = to_device(np.zeros((H, W, 4), np.float16)), to_device(bg)
    g.SortAndRenderSplatsMulti(rs, cam, rt, tg)
    want_rt, want_tg = to_host(ctx, rt), to_host(ctx, tg)
    for r in rs:
        r.Dispose()

    grp = GaussianSplatGroup.create(assets[0], [0, 0], emulate=True)
    objs = [grp, grp.add_object(assets[1])]
    for o, m in zip(objs, mats):
        o.localToWorldMatrix = m
    # member i draws into the rectangle at (37 i, 19) of layer i of its own array, and composites onto the rectangle at (11, 7 i)
    # of a 2-D array
    A = [SharedArray(g, ca, 301, 157, 2) for _ in range(2)]
    B = [SharedArray(g, ca, 260, 140, 0) for _ in range(2)]
    for i in range(2):
        B[i].fill(0, 11, 7 * i, bg)
    grp.SortAndRenderSplatsMulti(objs, cam, rts=[A[i].view(i, (37 * i, 19), (W, H)) for i in range(2)],
                                 camera_targets=[B[i].view(None, (11, 7 * i), (W, H)) for i in range(2)])
    grp.sync()
    for i in range(2):
        A[i].check(ctx, [(i, 37 * i, 19, want_rt)], "member %d rt" % i)
        B[i].check(ctx, [(0, 11, 7 * i, want_tg)], "member %d camera target" % i)
    # a depth rectangle is refused: the members share the frame parameters, and an array belongs to one device
    da = SharedArray(g, ca, 301, 157, 0, np.float32, "depth", 0.0)
    grp.sceneDepth = da.view(None, (3, 4), (W, H))
    hosts = [np.full((H, W, 4), SENTINEL, np.float16) for _ in range(2)]
    with pytest.raises(N.GsError) as e:
        grp.SortAndRenderSplats(cam, rts=hosts)
    assert e.value.code == INVALID
    for x in hosts:
        assert (x == np.float16(SENTINEL)).all()
    grp.close()


# ---- 5. refusals -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rect_refusals_enqueue_nothing(g, ctx, ca):
    import torch
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    lib = N.native()
    w, h = 128, 96
    cam = camera(g, w, h)
    rs = [g.GaussianSplatRenderer(a, ctx) for a in _assets(g)]
    r = rs[0]
    for x in rs:
        x.ResetOrder()
    orders = [x.readback_order() for x in rs]
    r.CalcViewData(cam)   # gs_render's precondition, so that only the image or the depth buffer can refuse it
    descs = []

    def rect(array, x=0, y=0, layer=0, reserved=0):
        descs.append(N.GsArrayRect(array, layer, x, y, reserved))
        return C.addressof(descs[-1])

    def image(data, memory=N.GS_MEM_ARRAY_RECT, pitch=0, fmt=N.GS_PIX_RGBA16F, height=h):
        return N.GsImage(data, w, height, pitch, fmt, memory)

    good = ca.array(200, 150, 0, fill=SENTINEL)
    good3 = ca.array(200, 150, 2, fill=SENTINEL)
    arrays = {
        "good": good, "good3": good3,
        "3-D": ca.array(200, 150, 2, flags=SURFACE_LOAD_STORE, fill=SENTINEL),   # a 3-D array that is not layered
        "no surface": ca.array(200, 150, 0, flags=0, fill=SENTINEL),
        "wide": ca.array(200, 150, 0, np.float32, fill=SENTINEL),               # 4 x 32-bit for an RGBA16F image
    }
    image_cases = [   # (what, image, status, words of the message)
        ("null array", image(rect(0)), INVALID, "null"),
        ("reserved", image(rect(good, reserved=1)), INVALID, "reserved"),
        ("layer of a 2-D array", image(rect(good, layer=1)), INVALID, "layer"),
        ("layer out of range", image(rect(good3, layer=2)), INVALID, "layer"),
        ("layer 2^31", image(rect(good3, layer=1 << 31)), INVALID, "layer"),
        ("3-D array", image(rect(arrays["3-D"])), INVALID, "3-D"),
        ("no surface flag", image(rect(arrays["no surface"])), INVALID, "cudaArraySurfaceLoadStore"),
        ("past the right edge", image(rect(good, x=73)), INVALID, "inside"),
        ("past the bottom edge", image(rect(good3, y=55, layer=1)), INVALID, "inside"),
        ("origin that wraps", image(rect(good, x=2 ** 32 - 64)), INVALID, "inside"),
        ("row pitch", image(rect(good), pitch=w * 8), INVALID, "row_pitch_bytes"),
        ("channel format", image(rect(arrays["wide"])), UNSUPPORTED, "channel format"),
        ("memory kind 6", image(rect(good), memory=6), INVALID, "memory kind"),
    ]
    d2 = ca.array(200, 150, 0, np.float32, 1, fill=0.0)
    d3 = ca.array(200, 150, 2, np.float32, 1, fill=0.0)
    depth_cases = [
        ("depth: null array", rect(0), INVALID),
        ("depth: reserved", rect(d2, reserved=1), INVALID),
        ("depth: layer of a 2-D array", rect(d2, layer=1), INVALID),
        ("depth: layer out of range", rect(d3, layer=2), INVALID),
        ("depth: 3-D array", rect(ca.array(200, 150, 2, np.float32, 1, flags=SURFACE_LOAD_STORE)), INVALID),
        ("depth: no surface flag", rect(ca.array(200, 150, 0, np.float32, 1, flags=0)), INVALID),
        ("depth: past the right edge", rect(d2, x=73), INVALID),
        ("depth: past the bottom edge", rect(d3, y=55, layer=1), INVALID),
        ("depth: origin that wraps", rect(d2, y=2 ** 32 - 8), INVALID),
        ("depth: RGBA16F array", rect(ca.array(200, 150, 0, np.float16)), UNSUPPORTED),
    ]
    rt_t = to_device(np.full((h, w, 4), SENTINEL, np.float16))
    rt_lin = _image(rt_t, w, h)
    other = _image(to_device(np.zeros((h, w, 4), np.float16)), w, h)
    opt = N.GsRenderOptions()
    no = (C.POINTER(N.GsImage) * 2)(C.POINTER(N.GsImage)(), C.POINTER(N.GsImage)())
    counts = (C.c_uint32 * 2)(1, 1)

    def params(depth=None):
        assets, fps, do_sort, keep = frame_args(g, [(cam, x, x.sceneDepth) for x in rs])
        if depth is not None:
            for i in range(len(rs)):
                fps[i].scene_depth, fps[i].scene_depth_on_device = depth, N.GS_MEM_ARRAY_RECT
        return fps, assets, do_sort, keep

    def untouched(what):
        check_regions(to_host(ctx, rt_t), SENTINEL, [], what)
        for name, hd in arrays.items():
            check_regions(ca.download(hd), SENTINEL, [], "%s: %s" % (what, name))
        for x, o in zip(rs, orders):
            assert np.array_equal(x.readback_order(), o), what

    ctx.set_timing(True)
    try:
        for what, im, status, words in image_cases:
            fps, assets, do_sort, keep = params()
            n0 = launches(ctx)
            assert lib.gs_frame(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), 1, C.byref(im), None) == status, what
            assert words in lib.gs_last_error(ctx.handle).decode(), what
            assert lib.gs_render(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), C.byref(im)) == status, what
            assert lib.gs_frame_objects(ctx.handle, 2, assets, fps, do_sort, C.byref(opt), C.byref(im), None) == status, what
            assert lib.gs_frame_objects(ctx.handle, 2, assets, fps, do_sort, C.byref(opt), C.byref(rt_lin), C.byref(im)) == status, what
            ims = (C.POINTER(N.GsImage) * 2)(C.pointer(other), C.pointer(im))
            assert lib.gs_frame_cameras(ctx.handle, 2, counts, assets, fps, do_sort, C.byref(opt), ims, no) == status, what
            assert launches(ctx) == n0, what
            untouched(what)
        for what, d, status in depth_cases:
            fps, assets, do_sort, keep = params(d)
            n0 = launches(ctx)
            assert lib.gs_frame(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), 1, C.byref(rt_lin), None) == status, what
            assert lib.gs_render(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), C.byref(rt_lin)) == status, what
            assert lib.gs_frame_objects(ctx.handle, 2, assets, fps, do_sort, C.byref(opt), C.byref(rt_lin), None) == status, what
            ims = (C.POINTER(N.GsImage) * 2)(C.pointer(rt_lin), C.pointer(other))
            assert lib.gs_frame_cameras(ctx.handle, 2, counts, assets, fps, do_sort, C.byref(opt), ims, no) == status, what
            assert launches(ctx) == n0, what
            untouched(what)
        # band-packed output and gs_unshuffle_bands output are linear memory only
        fps, assets, do_sort, keep = params()
        bopt = N.GsRenderOptions()
        bopt.partition_index, bopt.partition_count, bopt.band_rows, bopt.band_packed = 0, 2, 1, 1
        im = image(rect(good), height=64)
        assert lib.gs_frame(ctx.handle, assets[0], C.byref(fps[0]), C.byref(bopt), 1, C.byref(im), None) == INVALID
        assert "band_packed" in lib.gs_last_error(ctx.handle).decode()
        gathered = torch.zeros((2, 64, w, 4), dtype=torch.float16, device="cuda")
        im = image(rect(good))
        assert lib.gs_unshuffle_bands(ctx.handle, C.c_void_p(gathered.data_ptr()), 2, 1, 64, N.GS_PIX_RGBA16F, C.byref(im)) == INVALID
        untouched("band_packed / gs_unshuffle_bands")
        # and a correct rectangle of the same array is accepted: drawn inside, nothing outside
        A = SharedArray(g, ca, 200, 150)
        fps, assets, do_sort, keep = params()
        im = _image(A.view(None, (72, 54), (w, h)), w, h)
        assert lib.gs_frame(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), 1, C.byref(im), None) == 0
        inside = A.read(ctx)[0, 54:, 72:]
        assert not np.array_equal(bits(inside), bits(A.start[0, 54:, 72:]))
        A.check(ctx, [(0, 72, 54, inside)], "the rectangle accepted")
    finally:
        ctx.set_timing(False)
    for x in rs:
        x.Dispose()
