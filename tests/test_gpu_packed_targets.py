"""GS_PIX_B10G11R11_UFLOAT camera targets on the GPU: the HDR colour buffer of URP and HDRP cameras, one uint32 texel per pixel
(R and G unsigned float11, B unsigned float10, no alpha), composited onto in host memory, device memory, a 2-D CUDA array of
one 32-bit unsigned channel, a layer of a layered one and a rectangle of either.

Every result is compared bit for bit: the device codec with the packed-target oracle's (tests/packed_oracle.c) over every float32
bit pattern, gs_composite with its gso_composite_b10g11r11, and each fused entry point with its definition (the draw into a render target, then gs_composite).
Texels outside a rectangle, other layers, and pixels the splats do not cover keep their bits."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import packed_oracle as P
from frame_loops import frame_args
from images import KIND_FLOAT, SharedArray, ca, launches, to_device, to_host  # noqa: F401
from util import camera

ROOT = Path(__file__).resolve().parents[1]
UNSUPPORTED = -4
PACKED = 2
W, H = 200, 120   # not a multiple of 16 on either axis


def codes(shape, seed):
    """Random texels, with denormals, the largest finite values, Inf and NaN codes among them."""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 2 ** 32, shape, dtype=np.uint64).astype(np.uint32)
    flat = t.reshape(-1)
    special = [0x001 | (0x002 << 11) | (0x01F << 22), 0x7BF | (0x7BF << 11) | (0x3DF << 22), 0x7C0 | (0x7C0 << 11) | (0x3E0 << 22),
               0x03F, 0x7C0, 0x3E0 << 22, 0]
    flat[:flat.size:97][:len(special)] = special
    return t


def packed(g, ca, w, h, layers=0, seed=1):
    """A packed camera-target array (layers 0: a 2-D array) whose every texel starts as a random code."""
    return SharedArray(g, ca, w, h, layers, np.uint32, "packed", codes((max(layers, 1), h, w), seed))


def _assets(g):
    return (g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED0B01, "Medium"),
            g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0B02, "VeryHigh"))


# ---- 1. the codec --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_codec_equals_the_oracle_over_every_float(tmp_path):
    from unitygaussiansplatting_b200 import build
    so = P.path()
    exe = tmp_path / "packed_float_test"
    subprocess.run([build._nvcc(), *build.nvcc_flags(), "-I", str(build.CSRC), "-I", str(ROOT / "tests"), "-o", str(exe),
                    str(ROOT / "tests" / "packed_float_test.cu"), str(so), "-Xlinker", "-rpath=" + str(so.parent)],
                   check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    r = subprocess.run([str(exe)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout


# ---- 2. gs_composite onto every kind of packed target -----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,blend", [(np.float16, 0), (np.float32, 1)], ids=["rgba16f", "rgba32f"])
def test_composite_equals_the_oracle(g, ctx, ca, dtype, blend):
    asset = _assets(g)[0]
    cam = camera(g, W, H)
    r = g.GaussianSplatRenderer(asset, ctx)
    r.blend_mode = blend
    t = to_device(np.zeros((H, W, 4), dtype))
    r.SortAndRenderSplats(cam, rt=t)
    rt = to_host(ctx, t)
    covered = rt[..., 3] > 0
    assert covered.any() and not covered.all()
    start = codes((H, W), 3)
    want = P.composite_b10g11r11(rt.astype(np.float32), start)
    assert np.array_equal(want[~covered], start[~covered]) and not np.array_equal(want[covered], start[covered])

    host = start.copy()
    r.Composite(rt, host)                      # host rt, host target
    assert np.array_equal(host, want), "host target"
    dev = to_device(start)
    r.Composite(t, dev)                        # device rt, device target
    assert np.array_equal(to_host(ctx, dev), want), "device target"
    for what, layers, layer, x, y, aw, ah in (("2-D array", 0, None, None, None, W, H), ("layer", 3, 1, None, None, W, H),
                                                ("rectangle", 0, None, 37, 19, 301, 157), ("rectangle of a layer", 3, 2, 101, 37, 301, 157)):
        A = packed(g, ca, aw, ah, layers, seed=11)
        A.fill(layer, x or 0, y or 0, start)
        r.Composite(t, A.view(layer, None if x is None else (x, y), (W, H)))
        A.check(ctx, [(layer, x or 0, y or 0, want)], what)
    r.Dispose()


# ---- 3. the fused entry points --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_frame_and_frame_objects_equal_draw_then_composite(g, ctx, ca):
    a, b = _assets(g)
    cam = camera(g, W, H)
    r = g.GaussianSplatRenderer(a, ctx)
    ra, rb = g.GaussianSplatRenderer(a, ctx), g.GaussianSplatRenderer(b, ctx)
    rb.localToWorldMatrix = g.trs(position=(1.5, 0.0, 3.0)).astype(np.float32)
    start = codes((H, W), 4)

    def frame(rt, tg):
        r.ResetOrder()
        r.SortAndRenderSplats(cam, rt=rt, camera_target=tg)

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
        for name, fn in (("gs_frame", frame), ("gs_frame_objects", objects)):
            # the definition: the draw into rt, then gs_composite onto the packed target
            t = to_device(np.zeros((H, W, 4), np.float16))
            fn(t, None)
            want_rt = to_host(ctx, t)
            tg = to_device(start)
            r.Composite(t, tg)
            want = to_host(ctx, tg)
            assert not np.array_equal(want, start)
            # RGBA16F camera targets: the launch count the packed ones must match
            n16 = counted(fn, to_device(np.zeros((H, W, 4), np.float16)), to_device(np.zeros((H, W, 4), np.float16)))
            n16_alone = counted(fn, None, to_device(np.zeros((H, W, 4), np.float16)))
            for kind in ("host", "device", "2-D array", "layer", "rectangle"):
                what = "%s onto a %s target" % (name, kind)
                for with_rt in (True, False):
                    t = to_device(np.zeros((H, W, 4), np.float16)) if with_rt else None
                    if kind == "host":
                        tg = start.copy()
                        fn(t, tg)
                        assert np.array_equal(tg, want), what
                    elif kind == "device":
                        tg = to_device(start)
                        assert counted(fn, t, tg) == (n16 if with_rt else n16_alone), what
                        assert np.array_equal(to_host(ctx, tg), want), what
                    else:
                        layers, layer, x, y, aw, ah = {"2-D array": (0, None, None, None, W, H), "layer": (2, 1, None, None, W, H),
                                                       "rectangle": (2, 1, 37, 19, 301, 157)}[kind]
                        A = packed(g, ca, aw, ah, layers, seed=12)
                        A.fill(layer, x or 0, y or 0, start)
                        assert counted(fn, t, A.view(layer, None if x is None else (x, y), (W, H))) == (n16 if with_rt else n16_alone), what
                        A.check(ctx, [(layer, x or 0, y or 0, want)], what)
                    if with_rt:
                        assert np.array_equal(to_host(ctx, t).view(np.uint16), want_rt.view(np.uint16)), what + ": rt"
    finally:
        ctx.set_timing(False)
    for x in (r, ra, rb):
        x.Dispose()


# three 128 x 96 cameras: one onto an RGBA16F tensor, two onto disjoint rectangles of one packed array
TILES = [(0, 0, 128, 96), (130, 0, 128, 96), (0, 100, 128, 96)]


@pytest.mark.gpu
def test_frame_cameras_with_mixed_targets_is_one_run(g, ctx, ca):
    assets = _assets(g)
    cams = [camera(g, w, h, pos=(-0.5 + 0.4 * i, 0.5, -6.0), forward=(0.1 * (i - 1), 0.0, 1.0)) for i, (_, _, w, h) in enumerate(TILES)]
    bg = np.random.default_rng(9).random((96, 128, 4), np.float32).astype(np.float16)

    def renderers():
        rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]
        rs[1].localToWorldMatrix = g.trs(position=(-0.6, 0.1, 0.2)).astype(np.float32)
        return rs

    ctx.set_timing(True)
    try:
        # the definition: the camera loop, into rts, then gs_composite onto each camera's target
        loop = renderers()
        A = packed(g, ca, 260, 200, 0, seed=21)
        rts = [to_device(np.zeros((h, w, 4), np.float16)) for (_, _, w, h) in TILES]
        n0 = launches(ctx)
        for c, cam in enumerate(cams):
            g.SortAndRenderSplatsMulti(loop, cam, rts[c])
        n_loop = launches(ctx) - n0
        want_rt = [to_host(ctx, t) for t in rts]
        tg0 = to_device(bg)
        loop[0].Composite(rts[0], tg0)
        want0 = to_host(ctx, tg0)
        want_tiles = []
        for c in (1, 2):
            x, y, w, h = TILES[c]
            t = to_device(A.start[0, y:y + h, x:x + w])
            loop[0].Composite(rts[c], t)
            want_tiles.append(to_host(ctx, t))
        want_order = [r.readback_order() for r in loop]

        # the same call onto RGBA16F targets: tiles of one RGBA16F array
        sep = renderers()
        h16 = ca.array(260, 200, 0, np.float16, fill=0.25)
        n0 = launches(ctx)
        actives = g.SortAndRenderCameras(sep, cams, [to_device(np.zeros((h, w, 4), np.float16)) for (_, _, w, h) in TILES],
                                         [to_device(bg)] + [g.CudaArrayImage(h16, w, h, np.float16, origin=(x, y)) for (x, y, w, h) in TILES[1:]])
        n16 = launches(ctx) - n0
        assert g.renderer.cameras_in_one_call(actives)
        assert n16 < n_loop + 3, "the cameras were not drawn as one run"   # + the loop's three composites, made apart above

        call = renderers()
        rts = [to_device(np.zeros((h, w, 4), np.float16)) for (_, _, w, h) in TILES]
        tg0 = to_device(bg)
        n0 = launches(ctx)
        g.SortAndRenderCameras(call, cams, rts, [tg0] + [A.view(origin=(x, y), size=(w, h)) for (x, y, w, h) in TILES[1:]])
        n_call = launches(ctx) - n0
        assert n_call == n16, (n_call, n16)
        for c in range(3):
            assert np.array_equal(to_host(ctx, rts[c]).view(np.uint16), want_rt[c].view(np.uint16)), "camera %d rt" % c
        assert np.array_equal(to_host(ctx, tg0).view(np.uint16), want0.view(np.uint16))
        A.check(ctx, [(None, x, y, want) for (x, y, _, _), want in zip(TILES[1:], want_tiles)], "packed tiles")
        for r, o in zip(call, want_order):
            assert np.array_equal(r.readback_order(), o)
        for r in loop + sep + call:
            r.Dispose()
    finally:
        ctx.set_timing(False)


# ---- 4. the render-thread events ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_unity_events_with_a_packed_array_target(g, ctx, ca):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    a, b = _assets(g)
    cam = camera(g, W, H)
    r = g.GaussianSplatRenderer(a, ctx)
    start = codes((H, W), 6)
    fn = N.native().gs_unity_get_render_event_func()

    # GS_UNITY_EVENT_FRAME against gs_frame
    r.ResetOrder()
    tg = to_device(start)
    r.SortAndRenderSplats(cam, camera_target=tg)
    want = to_host(ctx, tg)
    fp, _keep = g.make_frame_params(cam, r.localToWorldMatrix, r.m_SplatScale, r.m_OpacityScale, r.m_SHOrder, r.m_SHOnly)
    A = packed(g, ca, 301, 157, 0, seed=31)
    A.fill(None, 37, 19, start)
    tg_im = _image(A.view(origin=(37, 19), size=(W, H)), W, H)
    ev = N.GsUnityFrameEvent()
    ev.ctx, ev.asset = C.cast(ctx.handle, C.c_void_p).value, C.cast(r._asset, C.c_void_p).value
    C.memmove(C.byref(ev.params), C.byref(fp), C.sizeof(fp))
    ev.options.blend_mode = r.blend_mode
    ev.do_sort, ev.status, ev.has_rt, ev.has_camera_target = 1, -5, 0, 1
    ev.camera_target = tg_im
    r.ResetOrder()
    fn(N.GS_UNITY_EVENT_FRAME, C.addressof(ev))
    assert ev.status == 0
    fn(N.GS_UNITY_EVENT_SYNC, C.addressof(ev))
    assert ev.status == 0
    A.check(ctx, [(None, 37, 19, want)], "GS_UNITY_EVENT_FRAME")

    # GS_UNITY_EVENT_FRAME_OBJECTS against gs_frame_objects
    rs = [g.GaussianSplatRenderer(x, ctx) for x in (a, b)]
    rs[1].localToWorldMatrix = g.trs(position=(1.5, 0.0, 3.0)).astype(np.float32)
    tg = to_device(start)
    active = g.SortAndRenderSplatsMulti(rs, cam, None, tg)
    want = to_host(ctx, tg)
    k = len(active)
    for x in active:
        x.ResetOrder()
    assets_arr, fps, ds, keep = frame_args(g, [(cam, x, x.sceneDepth) for x in active])
    B = packed(g, ca, W, H, 3, seed=32)
    B.fill(2, 0, 0, start)
    ev = N.GsUnityFrameObjectsEvent()
    ev.ctx, ev.object_count = C.cast(ctx.handle, C.c_void_p).value, k
    ev.assets, ev.fps, ev.do_sort = C.addressof(assets_arr), C.addressof(fps), C.addressof(ds)
    ev.options.blend_mode = active[0].blend_mode
    ev.status, ev.has_rt, ev.has_camera_target = -5, 0, 1
    tg_im = _image(B.view(layer=2), W, H)
    ev.camera_target = tg_im
    fn(N.GS_UNITY_EVENT_FRAME_OBJECTS, C.addressof(ev))
    assert ev.status == 0
    B.check(ctx, [(2, 0, 0, want)], "GS_UNITY_EVENT_FRAME_OBJECTS")
    for x in [r] + rs:
        x.Dispose()


# ---- 5. a group ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_emulated_group_onto_packed_targets_equals_one_gpu(g, ctx, ca):
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    assets = _assets(g)
    mats = [g.trs(position=(0.3, 0.0, 1.0)).astype(np.float32), g.trs(position=(-0.6, 0.1, 0.2)).astype(np.float32)]
    cam = camera(g, W, H)
    start = codes((H, W), 8)
    rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]
    for r, m in zip(rs, mats):
        r.localToWorldMatrix = m
    rt, tg = to_device(np.zeros((H, W, 4), np.float16)), to_device(start)
    g.SortAndRenderSplatsMulti(rs, cam, rt, tg)
    want_rt, want = to_host(ctx, rt), to_host(ctx, tg)
    for r in rs:
        r.Dispose()

    grp = GaussianSplatGroup.create(assets[0], [0, 0, 0], emulate=True)
    objs = [grp, grp.add_object(assets[1])]
    for o, m in zip(objs, mats):
        o.localToWorldMatrix = m
    # member 0 composites onto a device tensor, member 1 onto a rectangle of a packed array, member 2 onto host memory
    A = packed(g, ca, 301, 157, 0, seed=41)
    A.fill(None, 37, 19, start)
    dev, host = to_device(start), start.copy()
    rts = [to_device(np.zeros((H, W, 4), np.float16)) for _ in range(3)]
    grp.SortAndRenderSplatsMulti(objs, cam, rts=rts, camera_targets=[dev, A.view(origin=(37, 19), size=(W, H)), host])
    grp.sync()
    for t in rts:
        assert np.array_equal(to_host(ctx, t).view(np.uint16), want_rt.view(np.uint16))
    assert np.array_equal(to_host(ctx, dev), want)
    A.check(ctx, [(None, 37, 19, want)], "member 1")
    assert np.array_equal(host, want)
    grp.close()


# ---- 6. refusals -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_packed_refusals_write_nothing(g, ctx, ca):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    from unitygaussiansplatting_b200.renderer import _image
    lib = N.native()
    asset = _assets(g)[0]
    cam = camera(g, W, H)
    r = g.GaussianSplatRenderer(asset, ctx)
    r.ResetOrder()
    r.CalcViewData(cam)   # gs_render's precondition, so that only the image can refuse it
    start = codes((H, W), 51)
    rt16 = to_device(np.random.default_rng(2).random((H, W, 4), np.float32).astype(np.float16))
    rt16_host = to_host(ctx, rt16)

    def refused(code, call, images):
        before = [im.copy() for im in images]
        with pytest.raises(N.GsError) as e:
            call()
        assert e.value.code == code, (e.value.code, str(e.value))
        ctx.sync()
        for im, b in zip(images, before):
            assert np.array_equal(im, b)

    # a packed image as a render target: gs_render, gs_frame, gs_frame_objects, gs_composite's source
    host = start.copy()
    refused(UNSUPPORTED, lambda: r.DrawSplats(cam, host), [host])
    refused(UNSUPPORTED, lambda: r.SortAndRenderSplats(cam, rt=host), [host])
    tg = start.copy()
    refused(UNSUPPORTED, lambda: r.SortAndRenderSplats(cam, rt=host, camera_target=tg), [host, tg])
    refused(UNSUPPORTED, lambda: g.SortAndRenderSplatsMulti([r], cam, host, tg), [host, tg])
    A = packed(g, ca, W, H, 0, seed=52)
    refused(UNSUPPORTED, lambda: r.SortAndRenderSplats(cam, rt=A.view()), [])
    A.check(ctx, [], "a packed array as rt")
    refused(UNSUPPORTED, lambda: r.Composite(host, tg), [host, tg])
    # band_packed output
    r.band_packed, r.partition = True, (0, 2, 1)
    try:
        hb = np.zeros((64, W), np.uint32)
        refused(UNSUPPORTED, lambda: r.DrawSplats(cam, hb), [hb])
    finally:
        r.band_packed, r.partition = False, (0, 0, 1)
    # gs_unshuffle_bands into a packed image
    out = start.copy()
    im = _image(out, W, H)
    gathered = to_device(np.zeros((2, 64, W), np.uint32))
    assert lib.gs_unshuffle_bands(ctx.handle, C.c_void_p(gathered.data_ptr()), 2, 1, 64, PACKED, C.byref(im)) == UNSUPPORTED
    assert np.array_equal(out, start)
    # a packed target array with a float channel, and an RGBA16F target given a uint32 array
    fa = ca.array(W, H, 0, np.uint32, 1, kind=KIND_FLOAT)
    refused(UNSUPPORTED, lambda: r.Composite(rt16, g.CudaArrayImage(fa, W, H, np.uint32)), [])
    ua = packed(g, ca, W, H, 0, seed=53)
    refused(UNSUPPORTED, lambda: r.Composite(rt16, g.CudaArrayImage(ua.handle, W, H, np.float16)), [])
    refused(UNSUPPORTED, lambda: g.SortAndRenderSplatsMulti([r], cam, None, g.CudaArrayImage(fa, W, H, np.uint32)), [])
    ua.check(ctx, [], "a uint32 array as an RGBA16F target")
    assert np.array_equal(to_host(ctx, rt16).view(np.uint16), rt16_host.view(np.uint16))
    r.Dispose()

    # a group's render targets
    grp = GaussianSplatGroup.create(asset, [0, 0], emulate=True)
    hosts = [start.copy() for _ in range(2)]
    refused(UNSUPPORTED, lambda: grp.SortAndRenderSplatsMulti([grp], cam, rts=hosts), hosts)
    grp.close()
