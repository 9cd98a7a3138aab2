"""The scene depth buffer in a CUDA array (GsFrameParams.scene_depth_on_device = GS_MEM_ARRAY) or in one layer of a layered one
(GS_MEM_ARRAY_LAYER): a camera depth copied into an imported R32 float texture, or one eye of an XR eye-depth array, read in place.

Every picture is compared byte for byte with the same call on a depth buffer in a device tensor holding the same texels; the
wall scene of test_gpu_parity.py::test_scene_depth_buffer is also checked against the oracle.  Layered depth arrays keep values
in their other layers that would change the picture (1.0 hides every splat), so a wrong layer shows."""
import ctypes as C

import numpy as np
import pytest

from cuda_arrays import H2D, KIND_FLOAT, KIND_UNSIGNED, LAYERED, SURFACE_LOAD_STORE, Cudart, _ChannelDesc, _Dim3, _Memcpy3DParms, _PitchedPtr
from util import camera

INVALID, UNSUPPORTED = -1, -4
SENTINEL = -3.25   # exact in half and float


@pytest.fixture
def ca(ctx):
    c = Cudart()
    yield c
    ctx.sync()
    c.free_all()


def depth_array(ca, w, h, layers=0, fill=None, bits=32, channels=1, kind=KIND_FLOAT, flags=None):
    """A (layers, h, w) array of `channels` channels of `bits` bits (layers 0: a 2-D array); fill: (h, w) or (layers, h, w)
    float32 texels of a one-channel float32 array.  flags None: cudaArraySurfaceLoadStore, and cudaArrayLayered when layered."""
    if flags is None:
        flags = SURFACE_LOAD_STORE | (LAYERED if layers else 0)
    ch = [bits if i < channels else 0 for i in range(4)]
    h_ = C.c_void_p()
    rc = ca.lib.cudaMalloc3DArray(C.byref(h_), C.byref(_ChannelDesc(*ch, kind)), _Dim3(w, h, layers), flags)
    assert rc == 0, "cudaMalloc3DArray failed with CUDA error %d" % rc
    ca.live.append(h_.value)
    if fill is not None:
        host = np.ascontiguousarray(fill, np.float32).reshape((-1, h, w))
        p = _Memcpy3DParms()
        p.srcPtr, p.dstArray = _PitchedPtr(host.ctypes.data, w * 4, w, h), h_.value
        p.extent, p.kind = _Dim3(w, h, host.shape[0]), H2D
        assert ca.lib.cudaMemcpy3D(C.byref(p)) == 0
    return h_.value


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint16) if a.dtype == np.float16 else a.view(np.uint32)


def _tensor(host):
    import torch
    return torch.from_numpy(np.ascontiguousarray(host)).cuda()


def _host(ctx, t):
    import torch
    ctx.sync()
    torch.cuda.synchronize()
    return t.cpu().numpy()


def wall_scene(g, W=400, H=300):
    """test_scene_depth_buffer's scene: 40 k clustered splats, a wall at view distance 6 over the left 60 %, plus NaN texels."""
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 40000, 0x5EED0095, "Medium")
    cam = camera(g, W, H)
    clip = cam.gpuProjectionMatrix(True).astype(np.float64) @ np.array([0.0, 0.0, -6.0, 1.0])
    depth = np.zeros((H, W), np.float32)
    depth[:, :int(W * 0.6)] = np.float32(clip[2] / clip[3])
    depth[::37, ::23] = np.nan
    return asset, cam, depth


class Depths:
    """One depth picture as a device tensor, a 2-D array, and layer k of a 3-layer array whose other layers hold 1.0."""

    def __init__(self, g, ca, depth, k=1):
        H, W = depth.shape
        self.tensor = _tensor(depth)
        self.a2d = depth_array(ca, W, H, 0, depth)
        layers = np.ones((3, H, W), np.float32)
        layers[k] = depth
        self.a3 = depth_array(ca, W, H, 3, layers)
        self.k = k
        self.g, self.W, self.H = g, W, H

    def kinds(self):
        g = self.g
        return {"array": g.CudaArrayDepth(self.a2d, self.W, self.H), "layer": g.CudaArrayDepth(self.a3, self.W, self.H, layer=self.k)}


class Target:
    """A render target of one kind, sentinel-filled: a device tensor, a 2-D array, or layer 1 of a 2-layer array."""

    def __init__(self, g, ca, kind, W, H, dtype):
        self.kind, self.dtype, self.W, self.H, self.ca = kind, np.dtype(dtype), W, H, ca
        if kind == "linear":
            self.t = _tensor(np.full((H, W, 4), SENTINEL, dtype))
            self.image = self.t
        else:
            layers = 0 if kind == "array" else 2
            self.handle = ca.array(W, H, layers, dtype, fill=SENTINEL)
            self.image = g.CudaArrayImage(self.handle, W, H, dtype, layer=None if kind == "array" else 1)

    def read(self, ctx):
        if self.kind == "linear":
            return _host(ctx, self.t)
        ctx.sync()
        if self.kind == "array":
            return self.ca.download(self.handle, (self.H, self.W, 4), self.dtype)
        both = self.ca.download(self.handle, (2, self.H, self.W, 4), self.dtype)
        assert (both[0] == self.dtype.type(SENTINEL)).all(), "layer 0 of the target was touched"
        return both[1]


def launches(ctx):
    return ctx.stage_times().kernel_launches


# ---- 1 + 2. one object: bit-identical with tensor depth, the oracle, and the right layer ------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,blend", [(np.float16, 0), (np.float16, 1), (np.float32, 0), (np.float32, 1)],
                         ids=["rgba16f-rop", "rgba16f-fp32", "rgba32f-rop", "rgba32f-fp32"])
def test_array_depth_equals_tensor_depth(g, O, ctx, ca, dtype, blend):
    asset, cam, depth = wall_scene(g)
    H, W = depth.shape
    n = asset.splatCount
    D = Depths(g, ca, depth)
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
            want = draw(D.tensor, Target(g, ca, "linear", W, H, dtype), staged)
            free = draw(None, Target(g, ca, "linear", W, H, dtype), staged)
            assert not np.array_equal(_bits(want), _bits(free)), "the wall hides nothing"
            if dtype == np.float16 and blend == 0 and selected is None and not staged:
                fp, _keep = g.make_frame_params(cam, splat_count=n, scene_depth=depth)
                assert np.array_equal(want.astype(np.float32), O.frame(asset, fp, threads=O.max_threads())["rt"])
            for dname, d in D.kinds().items():
                for tkind in ("linear", "array", "layer"):
                    got = draw(d, Target(g, ca, tkind, W, H, dtype), staged)
                    assert np.array_equal(_bits(got), _bits(want)), (dname, tkind, staged, selected is not None)
            # layer 0 of the 3-layer array holds 1.0: every splat is behind it
            hidden = draw(g.CudaArrayDepth(D.a3, W, H, layer=0), Target(g, ca, "linear", W, H, dtype), staged)
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
    t0, t1 = _tensor(d0), _tensor(d1)
    a3 = depth_array(ca, W, H, 3, np.stack([d0, d1, np.ones((H, W), np.float32)]))

    def frame(depths):
        for r, d in zip(rs, depths):
            r.sceneDepth = d
            r.ResetOrder()
        rt = _tensor(np.zeros((H, W, 4), np.float16))
        n0 = launches(ctx)
        active = g.SortAndRenderSplatsMulti(rs, cam, rt)
        n = launches(ctx) - n0
        return _host(ctx, rt), n, [r.readback_order() for r in active]

    def loop(depths):
        for r, d in zip(rs, depths):
            r.sceneDepth = d
            r.ResetOrder()
        rt = _tensor(np.zeros((H, W, 4), np.float16))
        active = g.GatherSplatsForCamera(rs, cam)
        for i, r in enumerate(active):
            r.load_rt = i > 0
            r.SortAndRenderSplats(cam, rt=rt)
            r.load_rt = False
        return _host(ctx, rt), [r.readback_order() for r in active]

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
        assert np.array_equal(_bits(want), _bits(ref)), name
        got, n_arr, got_orders = frame(arr)
        assert np.array_equal(_bits(got), _bits(want)), name
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
def _fps(g, pairs):
    """pairs: [(cam, renderer, depth)] -> GsFrameParams array, assets, do_sort, keep-alive."""
    from unitygaussiansplatting_b200 import _native as N
    fps = (N.GsFrameParams * len(pairs))()
    assets = (C.c_void_p * len(pairs))()
    do_sort = (C.c_int32 * len(pairs))(*([1] * len(pairs)))
    keep = []
    for i, (cam, r, d) in enumerate(pairs):
        fps[i], k = g.make_frame_params(cam, r.localToWorldMatrix, splat_count=r.splatCount, scene_depth=d)
        keep.append(k)
        assets[i] = C.cast(r._asset, C.c_void_p).value
    return fps, assets, do_sort, keep


def _frame_cameras(g, ctx, eyes, rs, rts):
    """eyes: [(cam, depth)]; every renderer drawn for every eye, in list order, into rts[eye]."""
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    fps, assets, do_sort, keep = _fps(g, [(cam, r, d) for cam, d in eyes for r in rs])
    counts = (C.c_uint32 * len(eyes))(*([len(rs)] * len(eyes)))
    ims = [_image(rt, cam.pixelWidth, cam.pixelHeight) for (cam, _), rt in zip(eyes, rts)]
    a = (C.POINTER(N.GsImage) * len(eyes))(*[C.pointer(x) for x in ims])
    b = (C.POINTER(N.GsImage) * len(eyes))(*([C.POINTER(N.GsImage)()] * len(eyes)))
    opt = N.GsRenderOptions()
    return ctx._lib.gs_frame_cameras(ctx.handle, len(eyes), counts, assets, fps, do_sort, C.byref(opt), a, b)


def _frame_objects(g, ctx, cam, d, rs, rt):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    fps, assets, do_sort, keep = _fps(g, [(cam, r, d) for r in rs])
    im = _image(rt, cam.pixelWidth, cam.pixelHeight)
    opt = N.GsRenderOptions()
    return ctx._lib.gs_frame_objects(ctx.handle, len(rs), assets, fps, do_sort, C.byref(opt), C.byref(im), None)


@pytest.mark.gpu
def test_stereo_pair_in_depth_layers(g, ctx, ca):
    W = H = 256
    rs = _renderers(g, ctx)[:2]
    cams = [camera(g, W, H, pos=(x, 0.5, -6.0)) for x in (-0.032, 0.032)]
    _, _, d0 = wall_scene(g, W, H)
    d1 = np.ascontiguousarray(d0[:, ::-1])
    da = depth_array(ca, W, H, 2, np.stack([d0, d1]))
    td = [_tensor(d0), _tensor(d1)]

    def reset():
        for r in rs:
            r.ResetOrder()

    # the reference: one gs_frame_objects call per eye on linear depth, and the pair through gs_frame_cameras on linear depth
    reset()
    want = []
    for e in range(2):
        rt = _tensor(np.zeros((H, W, 4), np.float16))
        assert _frame_objects(g, ctx, cams[e], td[e], rs, rt) == 0
        want.append(_host(ctx, rt))
    want_orders = [r.readback_order() for r in rs]
    reset()
    lin = [_tensor(np.zeros((H, W, 4), np.float16)) for _ in range(2)]
    n0 = launches(ctx)
    assert _frame_cameras(g, ctx, [(cams[0], td[0]), (cams[1], td[1])], rs, lin) == 0
    n_lin = launches(ctx) - n0
    for e in range(2):
        assert np.array_equal(_bits(_host(ctx, lin[e])), _bits(want[e]))

    # eye colour in layers 0 / 1 of an RGBA16F array, eye depth in layers 0 / 1 of a float32 array
    reset()
    colour = ca.array(W, H, 2, np.float16, fill=SENTINEL)
    rts = [g.CudaArrayImage(colour, W, H, np.float16, layer=e) for e in range(2)]
    n0 = launches(ctx)
    assert _frame_cameras(g, ctx, [(cams[e], g.CudaArrayDepth(da, W, H, layer=e)) for e in range(2)], rs, rts) == 0
    assert launches(ctx) - n0 == n_lin
    ctx.sync()
    got = ca.download(colour, (2, H, W, 4), np.float16)
    for e in range(2):
        assert np.array_equal(_bits(got[e]), _bits(want[e])), "eye %d" % e
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
    D = Depths(g, ca, depth)
    r = g.GaussianSplatRenderer(asset, ctx)
    r.sceneDepth = D.tensor
    r.ResetOrder()
    want = Target(g, ca, "linear", W, H, np.float16)
    r.SortAndRenderSplats(cam, rt=want.image)
    want = want.read(ctx)
    r.ResetOrder()
    layer = g.CudaArrayDepth(D.a3, W, H, layer=D.k)   # its GsArrayLayer must stay alive until the event has run
    fp, _keep = g.make_frame_params(cam, splat_count=asset.splatCount, scene_depth=layer)
    assert fp.scene_depth_on_device == N.GS_MEM_ARRAY_LAYER
    ev = N.GsUnityFrameEvent()
    ev.ctx, ev.asset = C.cast(ctx.handle, C.c_void_p).value, C.cast(r._asset, C.c_void_p).value
    C.memmove(C.byref(ev.params), C.byref(fp), C.sizeof(fp))
    ev.do_sort, ev.status, ev.has_rt, ev.has_camera_target = 1, -5, 1, 0
    t = Target(g, ca, "layer", W, H, np.float16)
    ev.rt = _image(t.image, W, H)
    fn = N.native().gs_unity_get_render_event_func()
    fn(N.GS_UNITY_EVENT_FRAME, C.addressof(ev))
    assert ev.status == 0
    fn(N.GS_UNITY_EVENT_SYNC, C.addressof(ev))
    assert ev.status == 0
    assert np.array_equal(_bits(t.read(ctx)), _bits(want))
    r.Dispose()


# ---- 6. refusals ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bad_depth_arrays_are_refused_before_any_work(g, ctx, ca):
    from unitygaussiansplatting_b200 import _native as N
    W, H = 200, 120
    cam = camera(g, W, H)
    rs = _renderers(g, ctx)[:2]
    r = rs[0]
    ok2d = depth_array(ca, W, H, 0, np.zeros((H, W), np.float32))
    ok3 = depth_array(ca, W, H, 3, np.zeros((3, H, W), np.float32))

    def layer_desc(array, layer, reserved=0):
        return N.GsArrayLayer(array, layer, reserved)

    cases = [   # (what, handle or descriptor, kind, status)
        ("RGBA float32 array", ca.array(W, H, 0, np.float32), N.GS_MEM_ARRAY, UNSUPPORTED),
        ("16-bit channel", depth_array(ca, W, H, 0, bits=16), N.GS_MEM_ARRAY, UNSUPPORTED),
        ("unsigned 32-bit channel", depth_array(ca, W, H, 0, kind=KIND_UNSIGNED), N.GS_MEM_ARRAY, UNSUPPORTED),
        ("RGBA16F layer", layer_desc(ca.array(W, H, 2, np.float16), 0), N.GS_MEM_ARRAY_LAYER, UNSUPPORTED),
        ("wrong width", depth_array(ca, W + 1, H), N.GS_MEM_ARRAY, INVALID),
        ("wrong height", depth_array(ca, W, H - 1), N.GS_MEM_ARRAY, INVALID),
        ("wrong layered extent", layer_desc(depth_array(ca, W, H + 1, 2), 0), N.GS_MEM_ARRAY_LAYER, INVALID),
        ("layered array as kind 2", ok3, N.GS_MEM_ARRAY, INVALID),
        ("2-D array as kind 4", layer_desc(ok2d, 0), N.GS_MEM_ARRAY_LAYER, INVALID),
        ("layer out of range", layer_desc(ok3, 3), N.GS_MEM_ARRAY_LAYER, INVALID),
        ("reserved not 0", layer_desc(ok3, 1, 1), N.GS_MEM_ARRAY_LAYER, INVALID),
        ("null array", layer_desc(0, 0), N.GS_MEM_ARRAY_LAYER, INVALID),
        ("no surface flag", depth_array(ca, W, H, 0, flags=0), N.GS_MEM_ARRAY, INVALID),
        ("no surface flag, layered", layer_desc(depth_array(ca, W, H, 2, flags=LAYERED), 1), N.GS_MEM_ARRAY_LAYER, INVALID),
    ]
    rt = _tensor(np.full((H, W, 4), SENTINEL, np.float16))
    from unitygaussiansplatting_b200.renderer import _image
    im = _image(rt, W, H)
    opt = N.GsRenderOptions()
    for x in rs:
        x.ResetOrder()
    orders = [x.readback_order() for x in rs]
    r.CalcViewData(cam)   # gs_render's precondition, so that only the depth buffer can refuse it

    def check_untouched(what):
        assert (_host(ctx, rt) == np.float16(SENTINEL)).all(), what
        for x, o in zip(rs, orders):
            assert np.array_equal(x.readback_order(), o), what

    for what, d, kind, status in cases:
        fps, assets, do_sort, keep = _fps(g, [(cam, x, None) for x in rs])
        for k in range(len(rs)):
            fps[k].scene_depth = C.addressof(d) if isinstance(d, N.GsArrayLayer) else d
            fps[k].scene_depth_on_device = kind
        n0 = launches(ctx)
        assert ctx._lib.gs_frame(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), 1, C.byref(im), None) == status, what
        assert ctx._lib.gs_render(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), C.byref(im)) == status, what
        assert ctx._lib.gs_frame_objects(ctx.handle, 2, assets, fps, do_sort, C.byref(opt), C.byref(im), None) == status, what
        counts = (C.c_uint32 * 2)(1, 1)
        ims = (C.POINTER(N.GsImage) * 2)(C.pointer(im), C.pointer(_image(_tensor(np.zeros((H, W, 4), np.float16)), W, H)))
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
