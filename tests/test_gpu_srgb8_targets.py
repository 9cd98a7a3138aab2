"""GS_PIX_R8G8B8A8_SRGB camera targets on the GPU: the 8-bit colour buffer of LDR cameras and of the reference's validator, four
bytes per pixel (R, G, B sRGB-encoded, A linear UNorm), composited onto in host memory, device memory, a 2-D CUDA array of four
8-bit unsigned channels, a layer of a layered one and a rectangle of either.

Every result is compared bit for bit: the device codec with the sRGB8 oracle's (tests/srgb8_oracle.c) over every float32 bit
pattern, gs_composite with its gso_composite_srgb8, each fused entry point with its definition (the draw into a render target,
then gs_composite), each render-thread event with its direct call, and an emulated GPU group with one GPU.  Texels outside a
rectangle, other layers, and pixels the splats do not cover keep their bytes."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import srgb8_oracle as S
from frame_loops import Twins, frame_args, mixed_assets, mixed_setup
from images import KIND_FLOAT, KIND_UNSIGNED, Image, SharedArray, bits, ca, launches, to_device, to_host  # noqa: F401
from util import camera

ROOT = Path(__file__).resolve().parents[1]
UNSUPPORTED, INVALID = -4, -1
SRGB8 = 3
W, H = 200, 120   # not a multiple of 16 on either axis


def codes(shape, seed):
    """Random texels (H, W, 4) uint8 (or (layers, H, W, 4)), with 0, 255 and the codes beside them among them."""
    t = np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)
    flat = t.reshape(-1, 4)
    special = [[0, 0, 0, 0], [255, 255, 255, 255], [1, 254, 128, 127], [255, 0, 255, 0], [10, 11, 12, 128]]
    flat[:flat.shape[0]:97][:len(special)] = special
    return t


def srgb8(g, ca, w, h, layers=0, seed=1):
    """An sRGB8 camera-target array (layers 0: a 2-D array) whose every texel starts as a random code."""
    return SharedArray(g, ca, w, h, layers, np.uint8, "colour", codes((max(layers, 1), h, w, 4), seed))


def _assets(g):
    return (g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED0C01, "Medium"),
            g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0C02, "VeryHigh"))


# ---- 1. the codec --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_codec_equals_the_oracle_over_every_float(tmp_path):
    from unitygaussiansplatting_b200 import build
    so = S.path()
    exe = tmp_path / "srgb8_test"
    subprocess.run([build._nvcc(), *build.nvcc_flags(), "-I", str(build.CSRC), "-I", str(ROOT / "tests"), "-o", str(exe),
                    str(ROOT / "tests" / "srgb8_test.cu"), str(so), "-Xlinker", "-rpath=" + str(so.parent)],
                   check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    r = subprocess.run([str(exe)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout


# ---- 2. gs_composite onto every kind of sRGB8 target ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("blend", [0, 1], ids=["rop", "fp32"])
@pytest.mark.parametrize("dtype", [np.float16, np.float32], ids=["rgba16f", "rgba32f"])
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
    start = codes((H, W, 4), 3)
    want = S.composite_srgb8(rt.astype(np.float32), start)
    assert np.array_equal(want[~covered], start[~covered]) and not np.array_equal(want[covered], start[covered])

    host = start.copy()
    r.Composite(rt, host)                      # host rt, host target
    assert np.array_equal(host, want), "host target"
    dev = to_device(start)
    r.Composite(t, dev)                        # device rt, device target
    assert np.array_equal(to_host(ctx, dev), want), "device target"
    for what, layers, layer, x, y, aw, ah in (("2-D array", 0, None, None, None, W, H), ("layer", 3, 1, None, None, W, H),
                                                ("rectangle", 0, None, 37, 19, 301, 157), ("rectangle of a layer", 3, 2, 101, 37, 301, 157)):
        A = srgb8(g, ca, aw, ah, layers, seed=11)
        A.fill(layer, x or 0, y or 0, start)
        r.Composite(t, A.view(layer, None if x is None else (x, y), (W, H)))
        A.check(ctx, [(layer, x or 0, y or 0, want)], what)
    r.Dispose()


@pytest.mark.gpu
def test_pitched_host_and_device_targets(g, ctx):
    """A linear image whose rows lie further apart than its width: the composite follows the pitch and leaves the padding."""
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    lib = N.native()
    asset = _assets(g)[0]
    cam = camera(g, W, H)
    r = g.GaussianSplatRenderer(asset, ctx)
    t = to_device(np.zeros((H, W, 4), np.float16))
    r.SortAndRenderSplats(cam, rt=t)
    start = codes((H, W + 5, 4), 4)
    want = start.copy()
    want[:, :W] = S.composite_srgb8(to_host(ctx, t).astype(np.float32), start[:, :W])
    rt_im = _image(t, W, H)
    for kind in ("host", "device"):
        buf = start.copy() if kind == "host" else to_device(start)
        im = N.GsImage()
        im.data = buf.ctypes.data if kind == "host" else buf.data_ptr()
        im.width, im.height, im.row_pitch_bytes, im.format = W, H, (W + 5) * 4, SRGB8
        im.memory = N.GS_MEM_HOST if kind == "host" else N.GS_MEM_DEVICE
        N.check(ctx.handle, lib.gs_composite(ctx.handle, C.byref(rt_im), C.byref(im)))
        got = buf if kind == "host" else to_host(ctx, buf)
        ctx.sync()
        assert np.array_equal(got, want), kind
    r.Dispose()


# ---- 3. the fused entry points --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_frame_and_frame_objects_equal_draw_then_composite(g, ctx, ca):
    a, b = _assets(g)
    cam = camera(g, W, H)
    r = g.GaussianSplatRenderer(a, ctx)
    ra, rb = g.GaussianSplatRenderer(a, ctx), g.GaussianSplatRenderer(b, ctx)
    rb.localToWorldMatrix = g.trs(position=(1.5, 0.0, 3.0)).astype(np.float32)
    start = codes((H, W, 4), 5)

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
            # the definition: the draw into rt, then gs_composite onto the sRGB8 target
            t = to_device(np.zeros((H, W, 4), np.float16))
            fn(t, None)
            want_rt = to_host(ctx, t)
            tg = to_device(start)
            r.Composite(t, tg)
            want = to_host(ctx, tg)
            assert not np.array_equal(want, start)
            # RGBA16F camera targets: the launch count the sRGB8 ones must match
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
                        A = srgb8(g, ca, aw, ah, layers, seed=12)
                        A.fill(layer, x or 0, y or 0, start)
                        assert counted(fn, t, A.view(layer, None if x is None else (x, y), (W, H))) == (n16 if with_rt else n16_alone), what
                        A.check(ctx, [(layer, x or 0, y or 0, want)], what)
                    if with_rt:
                        assert np.array_equal(bits(to_host(ctx, t)), bits(want_rt)), what + ": rt"
    finally:
        ctx.set_timing(False)
    for x in (r, ra, rb):
        x.Dispose()


# four 128 x 96 cameras: one onto an RGBA16F tensor, one onto a B10G11R11 tensor, two onto an atlas of sRGB8 rectangles of one array
TILES = [(0, 0, 128, 96), (0, 0, 128, 96), (130, 0, 128, 96), (0, 100, 128, 96)]


@pytest.mark.gpu
def test_frame_cameras_with_mixed_targets_is_one_run(g, ctx, ca):
    assets = _assets(g)
    cams = [camera(g, w, h, pos=(-0.5 + 0.3 * i, 0.5, -6.0), forward=(0.07 * (i - 1.5), 0.0, 1.0)) for i, (_, _, w, h) in enumerate(TILES)]
    rng = np.random.default_rng(9)
    bg16 = rng.random((96, 128, 4), np.float32).astype(np.float16)
    bg_packed = g.pack_b10g11r11(rng.random((96, 128, 3), np.float32))

    def renderers():
        rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]
        rs[1].localToWorldMatrix = g.trs(position=(-0.6, 0.1, 0.2)).astype(np.float32)
        return rs

    ctx.set_timing(True)
    try:
        # the definition: the camera loop, into rts, then gs_composite onto each camera's target
        loop = renderers()
        A = srgb8(g, ca, 260, 200, 0, seed=21)
        rts = [to_device(np.zeros((h, w, 4), np.float16)) for (_, _, w, h) in TILES]
        n0 = launches(ctx)
        for c, cam in enumerate(cams):
            g.SortAndRenderSplatsMulti(loop, cam, rts[c])
        n_loop = launches(ctx) - n0
        want_rt = [to_host(ctx, t) for t in rts]
        want = []
        for c, start in ((0, bg16), (1, bg_packed)):
            tg = to_device(start)
            loop[0].Composite(rts[c], tg)
            want.append(to_host(ctx, tg))
        want_tiles = []
        for c in (2, 3):
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
                                         [to_device(bg16), to_device(bg16)] +
                                         [g.CudaArrayImage(h16, w, h, np.float16, origin=(x, y)) for (x, y, w, h) in TILES[2:]])
        n16 = launches(ctx) - n0
        assert g.renderer.cameras_in_one_call(actives)
        assert n16 < n_loop + 4, "the cameras were not drawn as one run"   # + the loop's four composites, made apart above

        call = renderers()
        rts = [to_device(np.zeros((h, w, 4), np.float16)) for (_, _, w, h) in TILES]
        tg0, tg1 = to_device(bg16), to_device(bg_packed)
        n0 = launches(ctx)
        g.SortAndRenderCameras(call, cams, rts, [tg0, tg1] + [A.view(origin=(x, y), size=(w, h)) for (x, y, w, h) in TILES[2:]])
        n_call = launches(ctx) - n0
        assert n_call == n16, (n_call, n16)
        for c in range(4):
            assert np.array_equal(bits(to_host(ctx, rts[c])), bits(want_rt[c])), "camera %d rt" % c
        assert np.array_equal(bits(to_host(ctx, tg0)), bits(want[0])), "RGBA16F target"
        assert np.array_equal(to_host(ctx, tg1), want[1]), "B10G11R11 target"
        A.check(ctx, [(None, x, y, w_) for (x, y, _, _), w_ in zip(TILES[2:], want_tiles)], "sRGB8 atlas")
        for r, o in zip(call, want_order):
            assert np.array_equal(r.readback_order(), o)
        for r in loop + sep + call:
            r.Dispose()
    finally:
        ctx.set_timing(False)


# ---- 4. the render-thread events ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_frame_and_frame_objects_events_with_srgb8_array_targets(g, ctx, ca):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    a, b = _assets(g)
    cam = camera(g, W, H)
    r = g.GaussianSplatRenderer(a, ctx)
    start = codes((H, W, 4), 6)
    fn = N.native().gs_unity_get_render_event_func()

    # GS_UNITY_EVENT_FRAME (1) against gs_frame
    r.ResetOrder()
    tg = to_device(start)
    r.SortAndRenderSplats(cam, camera_target=tg)
    want = to_host(ctx, tg)
    assert not np.array_equal(want, start)
    fp, _keep = g.make_frame_params(cam, r.localToWorldMatrix, r.m_SplatScale, r.m_OpacityScale, r.m_SHOrder, r.m_SHOnly)
    A = srgb8(g, ca, 301, 157, 0, seed=31)
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

    # GS_UNITY_EVENT_FRAME_OBJECTS (3) against gs_frame_objects
    rs = [g.GaussianSplatRenderer(x, ctx) for x in (a, b)]
    rs[1].localToWorldMatrix = g.trs(position=(1.5, 0.0, 3.0)).astype(np.float32)
    tg = to_device(start)
    active = g.SortAndRenderSplatsMulti(rs, cam, None, tg)
    want = to_host(ctx, tg)
    k = len(active)
    for x in active:
        x.ResetOrder()
    assets_arr, fps, ds, keep = frame_args(g, [(cam, x, x.sceneDepth) for x in active])
    B = srgb8(g, ca, W, H, 3, seed=32)
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


@pytest.mark.gpu
def test_frame_cameras_event_with_srgb8_array_targets(g, ctx, ca):
    """GS_UNITY_EVENT_FRAME_CAMERAS (4) against gs_frame_cameras: a stereo pair onto the layers of an sRGB8 eye-texture array and
    a third camera onto a rectangle of an sRGB8 array, with device, host and no render targets."""
    tw = Twins(g, ctx, mixed_assets(g, 2), mixed_setup)
    cams = [camera(g, 160, 112, pos=(-0.032, 0.5, -6.0)), camera(g, 160, 112, pos=(0.032, 0.5, -6.0)),
            camera(g, 144, 96, pos=(0.3, 0.4, -5.5))]
    rt_kinds = ["device", "host", None]

    def images():
        eyes = srgb8(g, ca, 160, 112, 2, seed=41)
        atlas = srgb8(g, ca, 300, 200, 0, seed=42)
        rts = [Image(g, ca, k, np.full((c.pixelHeight, c.pixelWidth, 4), 7, np.float16)) if k else None for k, c in zip(rt_kinds, cams)]
        return eyes, atlas, rts, [eyes.view(layer=0), eyes.view(layer=1), atlas.view(origin=(101, 57), size=(144, 96))]

    (de, da, drts, dtgts), (ee, ea, erts, etgts) = images(), images()
    g.SortAndRenderCameras(tw.loop, cams, [x and x.image for x in drts], dtgts)
    g.SortAndRenderCameras(tw.call, cams, [x and x.image for x in erts], etgts, via_event=True)
    for c in range(2):
        want = drts[c].read(ctx)
        assert want.any()
        assert np.array_equal(bits(erts[c].read(ctx)), bits(want)), "camera %d render target" % c
    want_eyes, want_atlas = de.read(ctx), da.read(ctx)
    assert not np.array_equal(want_eyes, de.start) and not np.array_equal(want_atlas, da.start)
    assert np.array_equal(ee.read(ctx), want_eyes), "eye layers"
    assert np.array_equal(ea.read(ctx), want_atlas), "atlas"
    tw.check_state()
    tw.dispose()


@pytest.mark.gpu
def test_group_frame_objects_event_with_srgb8_targets(g, ctx, ca):
    """GS_UNITY_EVENT_GROUP_FRAME_OBJECTS (5) + GS_UNITY_EVENT_GROUP_SYNC against gs_group_frame_objects + gs_group_sync on an
    emulated group of 2, member 0 onto a rectangle of an sRGB8 array, member 1 onto a layer of one."""
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    assets = mixed_assets(g, 2)
    mats = [g.trs(position=(0.3, 0.0, 1.0)).astype(np.float32), g.trs(position=(-0.6, 0.1, 0.2)).astype(np.float32)]
    cam = camera(g, W, H)
    start = codes((H, W, 4), 43)
    results = []
    for k in range(2):   # the direct call, then the event
        grp = GaussianSplatGroup.create(assets[0], [0, 0], emulate=True)
        objs = [grp, grp.add_object(assets[1])]
        for o, m in zip(objs, mats):
            o.localToWorldMatrix = m
        A, B = srgb8(g, ca, 301, 157, 0, seed=44), srgb8(g, ca, W, H, 2, seed=45)
        A.fill(None, 37, 19, start)
        B.fill(1, 0, 0, start)
        rts = [to_device(np.zeros((H, W, 4), np.float16)), None]
        grp.SortAndRenderSplatsMulti(objs, cam, rts=rts, camera_targets=[A.view(origin=(37, 19), size=(W, H)), B.view(layer=1)],
                                     via_event=k == 1)
        grp.sync(via_event=k == 1)
        results.append((to_host(ctx, rts[0]), A.read(ctx), B.read(ctx)))
        grp.close()
    (rt0, a0, b0), (rt1, a1, b1) = results
    assert rt0.any() and not np.array_equal(a0[0, 19:19 + H, 37:37 + W], start)
    assert np.array_equal(bits(rt1), bits(rt0))
    assert np.array_equal(a1, a0) and np.array_equal(b1, b0)


# ---- 5. a group ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("members", [2, 4])
def test_emulated_group_onto_srgb8_targets_equals_one_gpu(g, ctx, ca, members):
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    assets = _assets(g)
    mats = [g.trs(position=(0.3, 0.0, 1.0)).astype(np.float32), g.trs(position=(-0.6, 0.1, 0.2)).astype(np.float32)]
    cam = camera(g, W, H)
    start = codes((H, W, 4), 8)
    rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]
    for r, m in zip(rs, mats):
        r.localToWorldMatrix = m
    rt, tg = to_device(np.zeros((H, W, 4), np.float16)), to_device(start)
    g.SortAndRenderSplatsMulti(rs, cam, rt, tg)
    want_rt, want = to_host(ctx, rt), to_host(ctx, tg)
    assert not np.array_equal(want, start)
    for r in rs:
        r.Dispose()

    grp = GaussianSplatGroup.create(assets[0], [0] * members, emulate=True)
    objs = [grp, grp.add_object(assets[1])]
    for o, m in zip(objs, mats):
        o.localToWorldMatrix = m
    # members onto a device tensor, a rectangle of an sRGB8 array, host memory and a layer of an sRGB8 array
    A = srgb8(g, ca, 301, 157, 0, seed=41)
    A.fill(None, 37, 19, start)
    B = srgb8(g, ca, W, H, 2, seed=42)
    B.fill(1, 0, 0, start)
    dev, host = to_device(start), start.copy()
    targets = [dev, A.view(origin=(37, 19), size=(W, H)), host, B.view(layer=1)][:members]
    rts = [to_device(np.zeros((H, W, 4), np.float16)) for _ in range(members)]
    grp.SortAndRenderSplatsMulti(objs, cam, rts=rts, camera_targets=targets)
    grp.sync()
    for t in rts:
        assert np.array_equal(bits(to_host(ctx, t)), bits(want_rt))
    assert np.array_equal(to_host(ctx, dev), want)
    A.check(ctx, [(None, 37, 19, want)], "member 1")
    if members == 4:
        assert np.array_equal(host, want)
        B.check(ctx, [(1, 0, 0, want)], "member 3")
    grp.close()


# ---- 6. refusals -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_srgb8_refusals_write_nothing(g, ctx, ca):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    from unitygaussiansplatting_b200.renderer import _image
    lib = N.native()
    asset = _assets(g)[0]
    cam = camera(g, W, H)
    r = g.GaussianSplatRenderer(asset, ctx)
    r.ResetOrder()
    r.CalcViewData(cam)   # gs_render's precondition, so that only the image can refuse it
    start = codes((H, W, 4), 51)
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

    # an sRGB8 image as a render target: gs_render, gs_frame, gs_frame_objects, gs_composite's source
    host = start.copy()
    refused(UNSUPPORTED, lambda: r.DrawSplats(cam, host), [host])
    refused(UNSUPPORTED, lambda: r.SortAndRenderSplats(cam, rt=host), [host])
    tg = start.copy()
    refused(UNSUPPORTED, lambda: r.SortAndRenderSplats(cam, rt=host, camera_target=tg), [host, tg])
    refused(UNSUPPORTED, lambda: g.SortAndRenderSplatsMulti([r], cam, host, tg), [host, tg])
    A = srgb8(g, ca, W, H, 0, seed=52)
    refused(UNSUPPORTED, lambda: r.SortAndRenderSplats(cam, rt=A.view()), [])
    A.check(ctx, [], "an sRGB8 array as rt")
    refused(UNSUPPORTED, lambda: r.Composite(host, tg), [host, tg])
    # band_packed output
    r.band_packed, r.partition = True, (0, 2, 1)
    try:
        hb = np.zeros((64, W, 4), np.uint8)
        refused(UNSUPPORTED, lambda: r.DrawSplats(cam, hb), [hb])
    finally:
        r.band_packed, r.partition = False, (0, 0, 1)
    # gs_unshuffle_bands into an sRGB8 image
    out = start.copy()
    im = _image(out, W, H)
    gathered = to_device(np.zeros((2, 64, W, 4), np.uint8))
    assert lib.gs_unshuffle_bands(ctx.handle, C.c_void_p(gathered.data_ptr()), 2, 1, 64, SRGB8, C.byref(im)) == UNSUPPORTED
    assert np.array_equal(out, start)
    # an sRGB8 target array of the wrong channels: one 8-bit channel, one 32-bit unsigned channel, four 32-bit floats
    for what, arr in (("uchar1", ca.array(W, H, 0, np.uint8, 1)), ("uint32", ca.array(W, H, 0, np.uint32, 1)),
                      ("float4", ca.array(W, H, 0, np.uint8, 4, bits=32, kind=KIND_FLOAT))):
        refused(UNSUPPORTED, lambda: r.Composite(rt16, g.CudaArrayImage(arr, W, H, np.uint8)), [])
        refused(UNSUPPORTED, lambda: g.SortAndRenderSplatsMulti([r], cam, None, g.CudaArrayImage(arr, W, H, np.uint8)), [])
    # an RGBA16F target given an sRGB8 array
    refused(UNSUPPORTED, lambda: r.Composite(rt16, g.CudaArrayImage(A.handle, W, H, np.float16)), [])
    A.check(ctx, [], "an sRGB8 array as an RGBA16F target")
    # a wrong size: an array larger than the image, and a row pitch that is not a whole number of texels
    big = srgb8(g, ca, W + 1, H, 0, seed=54)
    refused(INVALID, lambda: r.Composite(rt16, g.CudaArrayImage(big.handle, W, H, np.uint8)), [])
    big.check(ctx, [], "an array of the wrong size")
    out = np.ascontiguousarray(np.broadcast_to(start.reshape(H, W * 4)[:, :1], (H, W * 4 + 2)))
    im = N.GsImage()
    im.data, im.width, im.height, im.row_pitch_bytes, im.format, im.memory = out.ctypes.data, W, H, W * 4 + 2, SRGB8, N.GS_MEM_HOST
    before = out.copy()
    assert lib.gs_composite(ctx.handle, C.byref(_image(rt16, W, H)), C.byref(im)) == INVALID
    ctx.sync()
    assert np.array_equal(out, before)
    assert np.array_equal(bits(to_host(ctx, rt16)), bits(rt16_host))
    r.Dispose()

    # a group's render targets
    grp = GaussianSplatGroup.create(asset, [0, 0], emulate=True)
    hosts = [start.copy() for _ in range(2)]
    refused(UNSUPPORTED, lambda: grp.SortAndRenderSplatsMulti([grp], cam, rts=hosts), hosts)
    grp.close()
