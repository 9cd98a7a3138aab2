"""The render-thread events of the camera run and the GPU group against their direct calls: GS_UNITY_EVENT_FRAME_CAMERAS
against gs_frame_cameras, GS_UNITY_EVENT_GROUP_FRAME_OBJECTS + GS_UNITY_EVENT_GROUP_SYNC against gs_group_frame_objects +
gs_group_sync.  Each case draws once through the event and once through the direct call, on fresh but identical state (two
copies of every asset, or two groups), and requires identical bytes in every render target and camera target, identical
persistent draw orders and sorted keys of every asset, and the same kernel launches and bin-list entries.  A refused payload
reports the direct call's code and text and writes no image.  Named test_zz_* so it runs after the parity tests proper."""
import ctypes as C

import numpy as np
import pytest

from frame_loops import Twins, _camera_args, _image, call_cameras, mixed_assets, mixed_setup, opt
from images import SENTINEL, Cudart, Image, SharedArray, background, bits, ca, to_device, to_host  # noqa: F401
from util import camera

pytestmark = pytest.mark.gpu

INVALID = -1


def event_cameras(g, ctx, per_cam, cams, blend, rts, tgts, extras=None, flags=0, counts=None):
    """call_cameras through GS_UNITY_EVENT_FRAME_CAMERAS: the same arguments in a GsUnityFrameCamerasEvent, images by value.
    Returns the payload's status."""
    from unitygaussiansplatting_b200 import _native as N
    assets, fps, ds, keep = _camera_args(g, per_cam, cams, extras)
    ims = [(_image(rt, cam), _image(tg, cam)) for rt, tg, cam in zip(rts, tgts, cams)]
    counts = (C.c_uint32 * len(cams))(*(counts if counts is not None else [len(rs) for rs in per_cam]))
    a, b = N.image_array([x for x, _ in ims]), N.image_array([y for _, y in ims])
    ev = N.GsUnityFrameCamerasEvent(ctx=ctx.handle.value, camera_count=len(cams), object_counts=C.addressof(counts),
                                    assets=C.addressof(assets), fps=C.addressof(fps), do_sort=C.addressof(ds),
                                    options=opt(N, blend, flags), rts=C.addressof(a), camera_targets=C.addressof(b),
                                    status=N.GS_ERR_NOT_READY)
    assert ev.status == N.GS_ERR_NOT_READY          # what the managed side records; the library writes it when the event runs
    return N.unity_event(N.GS_UNITY_EVENT_FRAME_CAMERAS, ev)


def event_cameras_ok(*args, **kw):
    rc = event_cameras(*args, **kw)
    assert rc == 0, "status %d" % rc


def counted(contexts, draw):
    """Runs draw() with timing on; per context, the kernels it launched and the bin-list entries of its last draw."""
    for c in contexts:
        c.set_timing(True)
    try:
        before = [c.stage_times().kernel_launches for c in contexts]
        draw()
        after = [c.stage_times() for c in contexts]
        return [(t.kernel_launches - n, t.tile_entries) for t, n in zip(after, before)]
    finally:
        for c in contexts:
            c.set_timing(False)


def _eye(g, W, H, side):
    return camera(g, W, H, pos=(side * 0.032, 0.5, -6.0))


# ---- GS_UNITY_EVENT_FRAME_CAMERAS ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("blend", [0, 1], ids=["rop", "fp32"])
def test_stereo_pair_into_layers_with_depth_layers(g, ctx, ca, blend):
    """The two eyes of a single-pass-instanced XR eye texture: render targets on layers 0 and 1 of one RGBA16F layered array,
    camera targets on layers of another, and each eye depth-tested against its layer of a float32 eye-depth array."""
    W, H = 256, 192
    tw = Twins(g, ctx, mixed_assets(g, 2), mixed_setup)
    eyes = [_eye(g, W, H, s) for s in (-1.0, 1.0)]
    lo, hi = tw.pick(tw.gathered(g, [range(2), range(2)], eyes))
    depth = SharedArray(g, ca, W, H, 2, np.float32, role="depth", start=0.0)
    for e in range(2):
        ramp = np.broadcast_to(np.linspace(0.0, 0.06 + 0.02 * e, W, dtype=np.float32), (H, W))
        depth.fill(e, 0, 0, ramp)
    extras = [[{"scene_depth": depth.view(layer=e)}] * 2 for e in range(2)]
    bg = background(H, W, np.float16, 21)
    arrays = []
    for _ in range(2):   # (render targets, camera targets) of the direct call, then of the event
        rt, tg = SharedArray(g, ca, W, H, 2), SharedArray(g, ca, W, H, 2)
        for e in range(2):
            tg.fill(e, 0, 0, bg)
        arrays.append((rt, tg))

    def draw(k, fn):
        rt, tg = arrays[k]
        return counted([ctx], lambda: fn(g, ctx, lo if k == 0 else hi, eyes, blend, [rt.view(layer=e) for e in range(2)],
                                         [tg.view(layer=e) for e in range(2)], extras))

    direct = draw(0, call_cameras)
    event = draw(1, event_cameras_ok)
    (rt0, tg0), (rt1, tg1) = arrays
    want_rt, want_tg = rt0.read(ctx), tg0.read(ctx)
    assert want_rt[0].any() and want_rt[1].any() and not np.array_equal(bits(want_rt[0]), bits(want_rt[1]))
    assert np.array_equal(bits(rt1.read(ctx)), bits(want_rt)), "render targets"
    assert np.array_equal(bits(tg1.read(ctx)), bits(want_tg)), "camera targets"
    tw.check_state()
    assert event == direct
    tw.dispose()


def test_quilt_of_rect_tiles(g, ctx, ca):
    """A 2 x 2 quilt: four cameras, each drawing into its GS_MEM_ARRAY_RECT tile of one array and compositing onto its tile of
    another."""
    W, H = 160, 112
    tw = Twins(g, ctx, mixed_assets(g, 3), mixed_setup)
    cams = [camera(g, W, H, pos=(0.25 * (i % 2) - 0.125, 0.45 + 0.1 * (i // 2), -6.0)) for i in range(4)]
    subsets = [[0, 1], [1, 2], [0, 2], [0, 1, 2]]
    lo, hi = tw.pick(tw.gathered(g, subsets, cams))
    origins = [(W * (i % 2), H * (i // 2)) for i in range(4)]
    bg = background(2 * H, 2 * W, np.float16, 22)
    arrays = [(SharedArray(g, ca, 2 * W, 2 * H), SharedArray(g, ca, 2 * W, 2 * H, start=bg)) for _ in range(2)]

    def views(a):
        return [a.view(origin=o, size=(W, H)) for o in origins]

    direct = counted([ctx], lambda: call_cameras(g, ctx, lo, cams, 0, views(arrays[0][0]), views(arrays[0][1])))
    event = counted([ctx], lambda: event_cameras_ok(g, ctx, hi, cams, 0, views(arrays[1][0]), views(arrays[1][1])))
    (rt0, tg0), (rt1, tg1) = arrays
    want_rt = rt0.read(ctx)
    for x, y in origins:
        assert want_rt[0, y:y + H, x:x + W].any(), "tile at (%d, %d)" % (x, y)
    assert np.array_equal(bits(rt1.read(ctx)), bits(want_rt)), "render targets"
    assert np.array_equal(bits(tg1.read(ctx)), bits(tg0.read(ctx))), "camera targets"
    tw.check_state()
    assert event == direct
    tw.dispose()


def test_host_device_and_packed_camera_targets_through_the_mirror(g, ctx, ca):
    """SortAndRenderCameras(via_event=True) against SortAndRenderCameras: three cameras whose camera targets are a host RGBA16F
    image, a device RGBA16F image and a B10G11R11 CUDA array, with host, device and no render targets."""
    tw = Twins(g, ctx, mixed_assets(g, 2), mixed_setup)
    cams = [camera(g, 200, 128, pos=(-0.3, 0.5, -6.0)), camera(g, 176, 144, pos=(0.2, 0.4, -5.5)), camera(g, 144, 96)]
    rt_kinds, tgt_kinds = ["device", "host", None], ["host", "device", "array"]

    def images():
        rts, tgts = [], []
        for c, cam in enumerate(cams):
            H, W = cam.pixelHeight, cam.pixelWidth
            bg = background(H, W, np.float16, 30 + c)
            rts.append(Image(g, ca, rt_kinds[c], np.full((H, W, 4), 7, np.float16)) if rt_kinds[c] else None)
            packed = c == 2
            tgts.append(Image(g, ca, tgt_kinds[c], g.pack_b10g11r11(bg[..., :3].astype(np.float32)) if packed else bg,
                              role="packed" if packed else "colour", start=0x1A2B3C4D if packed else SENTINEL))
        return rts, tgts

    (drts, dtgts), (erts, etgts) = images(), images()
    direct = counted([ctx], lambda: g.SortAndRenderCameras(tw.loop, cams, [x and x.image for x in drts], [x.image for x in dtgts]))
    event = counted([ctx], lambda: g.SortAndRenderCameras(tw.call, cams, [x and x.image for x in erts], [x.image for x in etgts],
                                                          via_event=True))
    for c in range(3):
        if drts[c] is not None:
            want = drts[c].read(ctx)
            assert want.any()
            assert np.array_equal(bits(erts[c].read(ctx)), bits(want)), "camera %d render target" % c
        want = dtgts[c].read(ctx)
        assert np.array_equal(bits(etgts[c].read(ctx)), bits(want)), "camera %d camera target" % c
    tw.check_state()
    assert event == direct
    tw.dispose()


def test_refused_camera_payloads_report_the_direct_calls_error(g, ctx):
    """GS_FLAG_ASYNC_READBACK and a camera without objects are refused by gs_frame_cameras: the event reports the same code and
    the same gs_last_error text, and writes no image."""
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    tw = Twins(g, ctx, mixed_assets(g, 2), mixed_setup)
    cams = [camera(g, 128, 96), camera(g, 96, 64, pos=(0.3, 0.5, -6.0))]
    for what, kw, per in [("GS_FLAG_ASYNC_READBACK", dict(flags=N.GS_FLAG_ASYNC_READBACK), [[0, 1], [1]]),
                          ("no objects", dict(counts=[2, 0]), [[0, 1], []])]:
        lo, hi = tw.pick(per)
        results = []
        for fn, rs in ((lambda *a, **k: call_cameras(*a, check=False, **k), lo), (event_cameras, hi)):
            rts = [to_device(np.full((c.pixelHeight, c.pixelWidth, 4), SENTINEL, np.float16)) for c in cams]
            tgts = [to_device(np.full((c.pixelHeight, c.pixelWidth, 4), SENTINEL, np.float16)) for c in cams]
            lib.gs_group_balance_rows(None, 0, 1, None)   # another error first: the refusal must set its own text
            rc = fn(g, ctx, rs, cams, 0, rts, tgts, **kw)
            results.append((rc, lib.gs_last_error(ctx.handle)))
            for t in rts + tgts:
                assert np.array_equal(bits(to_host(ctx, t)), bits(np.full(tuple(t.shape), SENTINEL, np.float16))), what + ": an image was written"
        assert results[0][0] == INVALID and results[1] == results[0], what
        assert (b"GS_FLAG_ASYNC_READBACK" if "ASYNC" in what else b"no objects") in results[0][1]
    tw.dispose()


# ---- GS_UNITY_EVENT_GROUP_FRAME_OBJECTS / GS_UNITY_EVENT_GROUP_SYNC ---------------------------------------------------------------
def _groups(g, assets, mats):
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    out = []
    for _ in range(2):   # the direct call's group, then the event's
        grp = GaussianSplatGroup.create(assets[0], [0, 0], emulate=True)
        objs = [grp] + [grp.add_object(a) for a in assets[1:]]
        for i, (o, m) in enumerate(zip(objs, mats)):
            o.localToWorldMatrix = m
            o.m_SortNthFrame = 1 + i
        out.append((grp, objs))
    return out


def _zero_keys(cudart, grp, objs):
    """Zeroes every asset's key buffer: a member sorts only its slab of the keys, so words no member writes then compare."""
    from unitygaussiansplatting_b200 import _native as N
    grp.sync()
    cudart.lib.cudaMemset.argtypes = [C.c_void_p, C.c_int, C.c_size_t]
    for o in objs:
        for i in range(grp.local_count):
            assert cudart.lib.cudaMemset(N.native().gs_asset_device_ptr(o._assets[i], 1), 0, o.splatCount * 4) == 0
    assert cudart.lib.cudaDeviceSynchronize() == 0


def _keys(o, i):
    from unitygaussiansplatting_b200 import _native as N
    out = np.empty(o.splatCount, np.uint32)
    N.check(None, N.native().gs_readback_keys(o._assets[i], out.ctypes.data))
    return out


def test_emulated_group_of_two_with_camera_targets(g, ctx, ca):
    """Two objects on an emulated group of 2, with render targets and camera targets, over two frames (the second sorts from
    the order the first left, and the second object sorts every other frame), each frame followed by the sync event."""
    W, H = 224, 160
    assets = mixed_assets(g, 2)
    mats = [g.trs(position=(0.3, 0.0, 1.0)).astype(np.float32), g.trs(position=(-0.6, 0.1, 0.2)).astype(np.float32)]
    groups = _groups(g, assets, mats)
    for grp, objs in groups:
        _zero_keys(ca, grp, objs)
    bg = background(H, W, np.float16, 41)
    for f, cam in enumerate([camera(g, W, H), camera(g, W, H, pos=(0.4, 0.6, -5.8))]):
        runs = []
        for k, (grp, objs) in enumerate(groups):
            rts = [to_device(np.zeros((H, W, 4), np.float16)), None]
            tgts = [Image(g, ca, "host", bg), Image(g, ca, "layer", bg)]

            def draw():
                grp.SortAndRenderSplatsMulti(objs, cam, rts=rts, camera_targets=[t.image for t in tgts], via_event=k == 1)
                grp.sync(via_event=k == 1)

            runs.append((counted(grp.contexts, draw), to_host(ctx, rts[0]), [t.read(ctx) for t in tgts]))
        (n0, rt0, tg0), (n1, rt1, tg1) = runs
        assert rt0.any() and not np.array_equal(bits(tg0[0]), bits(bg))
        assert np.array_equal(bits(rt1), bits(rt0)), "frame %d render target" % f
        for i in range(2):
            assert np.array_equal(bits(tg1[i]), bits(tg0[i])), "frame %d member %d camera target" % (f, i)
        assert n1 == n0, "frame %d: launches / bin-list entries per member" % f
        (_, direct_objs), (_, event_objs) = groups
        for o, p in zip(direct_objs, event_objs):
            for i in range(2):
                assert np.array_equal(p.readback_order(i), o.readback_order(i)), "frame %d member %d draw order" % (f, i)
                assert np.array_equal(_keys(p, i), _keys(o, i)), "frame %d member %d sorted keys" % (f, i)
    for grp, _ in groups:
        grp.close()


def test_refused_group_payload_reports_the_direct_calls_error(g, ctx, ca):
    """A CUDA-array scene depth buffer is refused by gs_group_frame_objects: the event reports the same code, member 0's
    gs_last_error holds the same text, and no image is written."""
    from unitygaussiansplatting_b200 import _native as N
    W, H = 128, 96
    assets = mixed_assets(g, 2)
    mats = [np.eye(4, dtype=np.float32)] * 2
    depth = SharedArray(g, ca, W, H, 0, np.float32, role="depth", start=0.0)
    cam = camera(g, W, H)
    errors = []
    for k, (grp, objs) in enumerate(_groups(g, assets, mats)):
        objs[1].sceneDepth = depth.view()
        rts, tgts = ([to_device(np.full((H, W, 4), SENTINEL, np.float16)) for _ in range(2)] for _ in range(2))
        with pytest.raises(g.GsError) as e:
            grp.SortAndRenderSplatsMulti(objs, cam, rts=rts, camera_targets=tgts, via_event=k == 1)
        errors.append((e.value.code, str(e.value), N.native().gs_last_error(grp.contexts[0].handle)))
        for t in rts + tgts:
            assert np.array_equal(bits(to_host(ctx, t)), bits(np.full((H, W, 4), SENTINEL, np.float16))), "an image was written"
        grp.close()
    assert errors[0][0] == INVALID and errors[1] == errors[0]
    assert b"CUDA array" in errors[0][2]


# ---- the device the events leave current -------------------------------------------------------------------------------------
def test_events_leave_the_direct_calls_device_current(g):
    """A context (and a group) on device 1 while the thread's current device is 0, as on a render thread that drives another
    GPU: the event leaves current the device the direct call leaves.  Needs two devices."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    cudart = Cudart()
    dev = C.c_int()

    def current_after(draw):
        assert cudart.lib.cudaSetDevice(0) == 0
        draw()
        assert cudart.lib.cudaGetDevice(C.byref(dev)) == 0
        return dev.value

    ctx1 = g.GaussianSplatContext(1)
    tw = Twins(g, ctx1, mixed_assets(g, 1))
    cams = [camera(g, 96, 64), camera(g, 96, 64, pos=(0.3, 0.5, -6.0))]
    rts = [[to_device(np.zeros((64, 96, 4), np.float16)).to("cuda:1") for _ in cams] for _ in range(2)]
    direct = current_after(lambda: g.SortAndRenderCameras(tw.loop, cams, rts[0], None))
    event = current_after(lambda: g.SortAndRenderCameras(tw.call, cams, rts[1], None, via_event=True))
    assert direct == event == 1
    assert np.array_equal(bits(to_host(ctx1, rts[1][0])), bits(to_host(ctx1, rts[0][0])))
    tw.dispose()
    grp = GaussianSplatGroup.create(mixed_assets(g, 1)[0], [1, 1], emulate=True)
    img = [to_device(np.zeros((64, 96, 4), np.float16)).to("cuda:1"), None]
    direct = current_after(lambda: (grp.SortAndRenderSplatsMulti([grp], cams[0], rts=img), grp.sync()))
    event = current_after(lambda: (grp.SortAndRenderSplatsMulti([grp], cams[0], rts=img, via_event=True), grp.sync(via_event=True)))
    assert direct == event == 1
    grp.close()
    ctx1.close()
