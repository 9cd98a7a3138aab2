"""The scene depth buffer in a CUDA array (GsFrameParams.scene_depth_on_device = GS_MEM_ARRAY) or in one layer of a layered one
(GS_MEM_ARRAY_LAYER): a camera depth copied into an imported R32 float texture, or one eye of an XR eye-depth array, read in place.

Every picture is compared byte for byte with the same call on a depth buffer in a device tensor holding the same texels; the
wall scene of test_gpu_parity.py::test_scene_depth_buffer is also checked against the oracle.  Layered depth arrays keep values
in their other layers that would change the picture (1.0 hides every splat), so a wrong layer shows."""
import ctypes as C

import numpy as np
import pytest

from frame_loops import call_cameras, call_frame, frame_args
from images import KIND_UNSIGNED, LAYERED, SENTINEL, Image, SharedArray, bits, ca, launches, to_device, to_host  # noqa: F401
from util import camera

INVALID, UNSUPPORTED = -1, -4


def wall_scene(g, W=400, H=300):
    """test_scene_depth_buffer's scene: 40 k clustered splats, a wall at view distance 6 over the left 60 %, plus NaN texels."""
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 40000, 0x5EED0095, "Medium")
    cam = camera(g, W, H)
    clip = cam.gpuProjectionMatrix(True).astype(np.float64) @ np.array([0.0, 0.0, -6.0, 1.0])
    depth = np.zeros((H, W), np.float32)
    depth[:, :int(W * 0.6)] = np.float32(clip[2] / clip[3])
    depth[::37, ::23] = np.nan
    return asset, cam, depth


def depths(g, ca, depth):
    """One depth picture as a device tensor, and by array kind: a 2-D array, and layer 1 of a 3-layer array whose other
    layers hold 1.0."""
    layered = Image(g, ca, "layer", depth, "depth", start=1.0, layers=3, layer=1)
    return to_device(depth), {"array": Image(g, ca, "array", depth, "depth").image, "layer": layered.image}, layered.array


def target(g, ca, kind, W, H, dtype):
    """A render target of one kind, sentinel-filled: a device tensor, a 2-D array, or layer 1 of a 2-layer array."""
    return Image(g, ca, kind, np.full((H, W, 4), SENTINEL, dtype))


# ---- 1 + 2. one object: bit-identical with tensor depth, the oracle, and the right layer ------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,blend", [(np.float16, 0), (np.float16, 1), (np.float32, 0), (np.float32, 1)],
                         ids=["rgba16f-rop", "rgba16f-fp32", "rgba32f-rop", "rgba32f-fp32"])
def test_array_depth_equals_tensor_depth(g, O, ctx, ca, dtype, blend):
    asset, cam, depth = wall_scene(g)
    H, W = depth.shape
    n = asset.splatCount
    tensor, kinds, layers = depths(g, ca, depth)
    r = g.GaussianSplatRenderer(asset, ctx)
    r.blend_mode = blend
    sel = np.zeros((n + 31) // 32, np.uint32)
    sel[::7] = 0x0F0F0F0F
    for selected in (None, sel):
        r.m_SelectedBits = selected

        def draw(depth_in, target, staged):
            r.sceneDepth = depth_in
            r.ResetOrder()
            if staged:
                r.CalcViewData(cam)
                r.DrawSplats(cam, target.image)
            else:
                r.SortAndRenderSplats(cam, rt=target.image)
            return target.read(ctx)

        for staged in (False, True):
            want = draw(tensor, target(g, ca, "device", W, H, dtype), staged)
            free = draw(None, target(g, ca, "device", W, H, dtype), staged)
            assert not np.array_equal(bits(want), bits(free)), "the wall hides nothing"
            if dtype == np.float16 and blend == 0 and selected is None and not staged:
                fp, _keep = g.make_frame_params(cam, splat_count=n, scene_depth=depth)
                assert np.array_equal(want.astype(np.float32), O.frame(asset, fp, threads=O.max_threads())["rt"])
            for dname, d in kinds.items():
                for tkind in ("device", "array", "layer"):
                    got = draw(d, target(g, ca, tkind, W, H, dtype), staged)
                    assert np.array_equal(bits(got), bits(want)), (dname, tkind, staged, selected is not None)
            # layer 0 of the 3-layer array holds 1.0: every splat is behind it
            hidden = draw(layers.view(layer=0), target(g, ca, "device", W, H, dtype), staged)
            assert not hidden.any()
    r.Dispose()


# ---- 3. several objects of one camera ---------------------------------------------------------------------------------------
def _renderers(g, ctx):
    out = []
    for i, (seed, q) in enumerate(((0x5EED0D01, "Medium"), (0x5EED0D02, "VeryHigh"), (0x5EED0D03, "Medium"))):
        r = g.GaussianSplatRenderer(g.synthetic_asset(g.SCENE_CLUSTERED, 20000, seed, q), ctx)
        r.localToWorldMatrix = g.trs(position=(0.8 * (i - 1), 0.1 * i, 0.4 * i)).astype(np.float32)
        out.append(r)
    return out


@pytest.mark.gpu
def test_objects_share_or_split_runs_by_depth_identity(g, ctx, ca):
    W, H = 320, 240
    cam = camera(g, W, H)
    rs = _renderers(g, ctx)
    _, _, d0 = wall_scene(g, W, H)
    d1 = np.where(np.arange(W)[None, :] > W // 2, d0[:, ::-1], 0.0).astype(np.float32)
    t0, t1 = to_device(d0), to_device(d1)
    a3 = ca.array(W, H, 3, np.float32, 1, fill=np.stack([d0, d1, np.ones((H, W), np.float32)]))

    def frame(depths):
        for r, d in zip(rs, depths):
            r.sceneDepth = d
            r.ResetOrder()
        rt = to_device(np.zeros((H, W, 4), np.float16))
        n0 = launches(ctx)
        active = g.SortAndRenderSplatsMulti(rs, cam, rt)
        n = launches(ctx) - n0
        return to_host(ctx, rt), n, [r.readback_order() for r in active]

    def loop(depths):
        for r, d in zip(rs, depths):
            r.sceneDepth = d
            r.ResetOrder()
        rt = to_device(np.zeros((H, W, 4), np.float16))
        active = g.GatherSplatsForCamera(rs, cam)
        for i, r in enumerate(active):
            r.load_rt = i > 0
            r.SortAndRenderSplats(cam, rt=rt)
            r.load_rt = False
        return to_host(ctx, rt), [r.readback_order() for r in active]

    def layer(k):   # a new descriptor each time: descriptors of one layer are one buffer
        return g.CudaArrayDepth(a3, W, H, layer=k)

    cases = {
        "one layer, three descriptors": ([t1, t1, t1], [layer(1), layer(1), layer(1)]),
        "two layers": ([t0, t1, t1], [layer(0), layer(1), layer(1)]),
        "an object without depth": ([t1, None, t1], [layer(1), None, layer(1)]),
    }
    for name, (lin, arr) in cases.items():
        want, n_lin, orders = frame(lin)
        ref, ref_orders = loop(lin)
        assert np.array_equal(bits(want), bits(ref)), name
        got, n_arr, got_orders = frame(arr)
        assert np.array_equal(bits(got), bits(want)), name
        assert n_arr == n_lin, (name, n_arr, n_lin)
        for a, b, c in zip(orders, ref_orders, got_orders):
            assert np.array_equal(a, b) and np.array_equal(a, c), name
    # one run against split runs: the single-descriptor case draws in fewer launches than the two-layer one
    _, n_one, _ = frame(cases["one layer, three descriptors"][1])
    _, n_two, _ = frame(cases["two layers"][1])
    assert n_one < n_two
    for r in rs:
        r.Dispose()


# ---- 4. a stereo pair: eye colour and eye depth in layers 0 / 1 -------------------------------------------------------------
@pytest.mark.gpu
def test_stereo_pair_in_depth_layers(g, ctx, ca):
    W = H = 256
    rs = _renderers(g, ctx)[:2]
    cams = [camera(g, W, H, pos=(x, 0.5, -6.0)) for x in (-0.032, 0.032)]
    _, _, d0 = wall_scene(g, W, H)
    d1 = np.ascontiguousarray(d0[:, ::-1])
    da = ca.array(W, H, 2, np.float32, 1, fill=np.stack([d0, d1]))
    td = [to_device(d0), to_device(d1)]

    def reset():
        for r in rs:
            r.ResetOrder()

    # the reference: one gs_frame_objects call per eye on linear depth, and the pair through gs_frame_cameras on linear depth
    reset()
    want = []
    for e in range(2):
        rt = to_device(np.zeros((H, W, 4), np.float16))
        for r in rs:
            r.sceneDepth = td[e]
        assert call_frame(g, ctx, rs, cams[e], 0, rt, None, check=False) == 0
        want.append(to_host(ctx, rt))
    want_orders = [r.readback_order() for r in rs]
    reset()
    lin = [to_device(np.zeros((H, W, 4), np.float16)) for _ in range(2)]
    n0 = launches(ctx)
    assert call_cameras(g, ctx, [rs, rs], cams, 0, lin, [None, None], [[{"scene_depth": d}] * 2 for d in td], check=False) == 0
    n_lin = launches(ctx) - n0
    for e in range(2):
        assert np.array_equal(bits(to_host(ctx, lin[e])), bits(want[e]))

    # eye colour in layers 0 / 1 of an RGBA16F array, eye depth in layers 0 / 1 of a float32 array
    reset()
    colour = SharedArray(g, ca, W, H, 2)
    rts = [colour.view(layer=e) for e in range(2)]
    n0 = launches(ctx)
    extras = [[{"scene_depth": g.CudaArrayDepth(da, W, H, layer=e)}] * 2 for e in range(2)]
    assert call_cameras(g, ctx, [rs, rs], cams, 0, rts, [None, None], extras, check=False) == 0
    assert launches(ctx) - n0 == n_lin
    colour.check(ctx, [(e, 0, 0, want[e]) for e in range(2)], "eyes")
    for r, o in zip(rs, want_orders):
        assert np.array_equal(r.readback_order(), o)
    for r in rs:
        r.Dispose()


# ---- 5. the Unity render event ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_unity_frame_event_with_layer_depth(g, ctx, ca):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    asset, cam, depth = wall_scene(g)
    H, W = depth.shape
    tensor, kinds, _ = depths(g, ca, depth)
    r = g.GaussianSplatRenderer(asset, ctx)
    r.sceneDepth = tensor
    r.ResetOrder()
    want = target(g, ca, "device", W, H, np.float16)
    r.SortAndRenderSplats(cam, rt=want.image)
    want = want.read(ctx)
    r.ResetOrder()
    layer = kinds["layer"]   # its GsArrayLayer must stay alive until the event has run
    fp, _keep = g.make_frame_params(cam, splat_count=asset.splatCount, scene_depth=layer)
    assert fp.scene_depth_on_device == N.GS_MEM_ARRAY_LAYER
    ev = N.GsUnityFrameEvent()
    ev.ctx, ev.asset = C.cast(ctx.handle, C.c_void_p).value, C.cast(r._asset, C.c_void_p).value
    C.memmove(C.byref(ev.params), C.byref(fp), C.sizeof(fp))
    ev.do_sort, ev.status, ev.has_rt, ev.has_camera_target = 1, -5, 1, 0
    t = target(g, ca, "layer", W, H, np.float16)
    ev.rt = _image(t.image, W, H)
    fn = N.native().gs_unity_get_render_event_func()
    fn(N.GS_UNITY_EVENT_FRAME, C.addressof(ev))
    assert ev.status == 0
    fn(N.GS_UNITY_EVENT_SYNC, C.addressof(ev))
    assert ev.status == 0
    assert np.array_equal(bits(t.read(ctx)), bits(want))
    r.Dispose()


# ---- 6. refusals ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bad_depth_arrays_are_refused_before_any_work(g, ctx, ca):
    from unitygaussiansplatting_b200 import _native as N
    W, H = 200, 120
    cam = camera(g, W, H)
    rs = _renderers(g, ctx)[:2]
    r = rs[0]

    def depth_array(w=W, h=H, layers=0, **kw):   # one float32 channel unless kw says otherwise
        return ca.array(w, h, layers, np.float32, 1, **kw)

    ok2d = depth_array(fill=0.0)
    ok3 = depth_array(layers=3, fill=0.0)

    def layer_desc(array, layer, reserved=0):
        return N.GsArrayLayer(array, layer, reserved)

    cases = [   # (what, handle or descriptor, kind, status)
        ("RGBA float32 array", ca.array(W, H, 0, np.float32), N.GS_MEM_ARRAY, UNSUPPORTED),
        ("16-bit channel", depth_array(bits=16), N.GS_MEM_ARRAY, UNSUPPORTED),
        ("unsigned 32-bit channel", depth_array(kind=KIND_UNSIGNED), N.GS_MEM_ARRAY, UNSUPPORTED),
        ("RGBA16F layer", layer_desc(ca.array(W, H, 2, np.float16), 0), N.GS_MEM_ARRAY_LAYER, UNSUPPORTED),
        ("wrong width", depth_array(W + 1), N.GS_MEM_ARRAY, INVALID),
        ("wrong height", depth_array(h=H - 1), N.GS_MEM_ARRAY, INVALID),
        ("wrong layered extent", layer_desc(depth_array(h=H + 1, layers=2), 0), N.GS_MEM_ARRAY_LAYER, INVALID),
        ("layered array as kind 2", ok3, N.GS_MEM_ARRAY, INVALID),
        ("2-D array as kind 4", layer_desc(ok2d, 0), N.GS_MEM_ARRAY_LAYER, INVALID),
        ("layer out of range", layer_desc(ok3, 3), N.GS_MEM_ARRAY_LAYER, INVALID),
        ("reserved not 0", layer_desc(ok3, 1, 1), N.GS_MEM_ARRAY_LAYER, INVALID),
        ("null array", layer_desc(0, 0), N.GS_MEM_ARRAY_LAYER, INVALID),
        ("no surface flag", depth_array(flags=0), N.GS_MEM_ARRAY, INVALID),
        ("no surface flag, layered", layer_desc(depth_array(layers=2, flags=LAYERED), 1), N.GS_MEM_ARRAY_LAYER, INVALID),
    ]
    rt = to_device(np.full((H, W, 4), SENTINEL, np.float16))
    from unitygaussiansplatting_b200.renderer import _image
    im = _image(rt, W, H)
    opt = N.GsRenderOptions()
    for x in rs:
        x.ResetOrder()
    orders = [x.readback_order() for x in rs]
    r.CalcViewData(cam)   # gs_render's precondition, so that only the depth buffer can refuse it

    def check_untouched(what):
        assert (to_host(ctx, rt) == np.float16(SENTINEL)).all(), what
        for x, o in zip(rs, orders):
            assert np.array_equal(x.readback_order(), o), what

    for what, d, kind, status in cases:
        assets, fps, do_sort, keep = frame_args(g, [(cam, x, None) for x in rs])
        for k in range(len(rs)):
            fps[k].scene_depth = C.addressof(d) if isinstance(d, N.GsArrayLayer) else d
            fps[k].scene_depth_on_device = kind
        n0 = launches(ctx)
        assert ctx._lib.gs_frame(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), 1, C.byref(im), None) == status, what
        assert ctx._lib.gs_render(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), C.byref(im)) == status, what
        assert ctx._lib.gs_frame_objects(ctx.handle, 2, assets, fps, do_sort, C.byref(opt), C.byref(im), None) == status, what
        counts = (C.c_uint32 * 2)(1, 1)
        ims = (C.POINTER(N.GsImage) * 2)(C.pointer(im), C.pointer(_image(to_device(np.zeros((H, W, 4), np.float16)), W, H)))
        no = (C.POINTER(N.GsImage) * 2)(C.POINTER(N.GsImage)(), C.POINTER(N.GsImage)())
        assert ctx._lib.gs_frame_cameras(ctx.handle, 2, counts, assets, fps, do_sort, C.byref(opt), ims, no) == status, what
        assert launches(ctx) == n0, what
        check_untouched(what)

    # a group call: the members share the frame parameters, and an array belongs to one device
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    grp = GaussianSplatGroup.create(r.m_Asset, [0, 0], emulate=True)
    rts = [np.full((H, W, 4), SENTINEL, np.float16) for _ in range(2)]
    for d in (g.CudaArrayDepth(ok2d, W, H), g.CudaArrayDepth(ok3, W, H, layer=1)):
        grp.sceneDepth = d
        with pytest.raises(N.GsError) as e:
            grp.SortAndRenderSplats(cam, rts=rts)
        assert e.value.code == INVALID
        for x in rts:
            assert (x == np.float16(SENTINEL)).all()
    check_untouched("group")
    for x in rs:
        x.Dispose()
