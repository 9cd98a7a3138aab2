"""A rectangle of a CUDA array as an image or a depth buffer (GS_MEM_ARRAY_RECT): an HDRP render target allocated larger than
the camera, whose camera draws into the rectangle at its origin, and the tiles of an atlas or a light-field quilt, one per
camera.  The library draws into, composites onto and depth-tests against the rectangle in place, and leaves every texel
outside it, and every other layer, as it was.

Arrays are made by cuda_arrays.Cudart, as test_gpu_layered_targets.py makes them.  Every result inside a rectangle is compared
byte for byte with the same call on linear device memory (or, for several cameras, with the camera loop it stands for), and
every texel outside the rectangles is checked to still hold its sentinel."""
import ctypes as C

import numpy as np
import pytest

from cuda_arrays import H2D, KIND_FLOAT, LAYERED, SURFACE_LOAD_STORE, Cudart, _ChannelDesc, _Dim3, _Memcpy3DParms, _PitchedPtr
from util import camera

INVALID, UNSUPPORTED = -1, -4
SENTINEL = -3.25   # exact in half and float
W, H = 200, 120    # a screen that is not a multiple of 16 on either axis
# (array width, array height, x, y): at the origin of a larger array, at an odd offset, flush with the far corner
PLACEMENTS = {"origin": (301, 157, 0, 0), "odd": (301, 157, 37, 19), "far-corner": (301, 157, 101, 37)}


@pytest.fixture
def ca(ctx):
    c = Cudart()
    yield c
    ctx.sync()
    c.free_all()


class Arr:
    """A (layers, h, w) RGBA array of `dtype` texels (layers 0: a 2-D array), every texel SENTINEL, and rectangles of it."""

    def __init__(self, g, ca, w, h, layers=0, dtype=np.float16):
        self.g, self.ca, self.w, self.h, self.layers, self.dtype = g, ca, w, h, layers, np.dtype(dtype)
        self.handle = ca.array(w, h, layers, dtype, fill=SENTINEL)

    def rect(self, x, y, w, h, layer=None):
        return self.g.CudaArrayImage(self.handle, w, h, self.dtype, layer=layer, origin=(x, y))

    def read(self):
        return self.ca.download(self.handle, (max(self.layers, 1), self.h, self.w, 4), self.dtype)

    def fill(self, layer, x, y, host):
        a = self.read()
        a[layer or 0, y:y + host.shape[0], x:x + host.shape[1]] = host
        self.ca.upload(self.handle, a)

    def check(self, ctx, regions, what):
        """regions: [(layer, x, y, want)]: each rectangle equals `want` bit for bit; every other texel holds the sentinel."""
        ctx.sync()
        got = self.read()
        outside = np.ones(got.shape[:3], bool)
        for layer, x, y, want in regions:
            h, w = want.shape[:2]
            assert np.array_equal(_bits(got[layer or 0, y:y + h, x:x + w]), _bits(want)), "%s: rectangle at (%d, %d) differs" % (what, x, y)
            outside[layer or 0, y:y + h, x:x + w] = False
        assert (got[outside] == self.dtype.type(SENTINEL)).all(), "%s: a texel outside the rectangles was touched" % what


def depth_array(ca, w, h, layers=0, fill=None, bits=32, channels=1, flags=None):
    """A (layers, h, w) array of `channels` float channels of `bits` bits (layers 0: a 2-D array); fill: (h, w) or (layers, h, w)
    float32 texels of a one-channel float32 array."""
    if flags is None:
        flags = SURFACE_LOAD_STORE | (LAYERED if layers else 0)
    h_ = C.c_void_p()
    rc = ca.lib.cudaMalloc3DArray(C.byref(h_), C.byref(_ChannelDesc(*[bits if i < channels else 0 for i in range(4)], KIND_FLOAT)),
                                  _Dim3(w, h, layers), flags)
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


def _background(h, w, dtype, seed):
    """A camera target's content: colours in [0, 1), alpha in [0, 0.5)."""
    bg = np.random.default_rng(seed).random((h, w, 4), np.float32)
    bg[..., 3] *= 0.5
    return bg.astype(np.float16).astype(dtype)


def launches(ctx):
    return ctx.stage_times().kernel_launches


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
    bg = _background(H, W, dtype, 5)
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
        t = _tensor(zeros); frame(t); want_f = _host(ctx, t)
        t = _tensor(zeros); frame(t, selected=sel); want_sel = _host(ctx, t)
        t = _tensor(want_f); load(t); want_load = _host(ctx, t)
        t, tg = _tensor(zeros), _tensor(bg); frame(t, tg); want_ftg = (_host(ctx, t), _host(ctx, tg))
        t, tg = _tensor(zeros), _tensor(bg); objects(t, tg); want_obj = (_host(ctx, t), _host(ctx, tg))
        assert want_f.any() and not np.array_equal(_bits(want_sel), _bits(want_f)) and not np.array_equal(_bits(want_load), _bits(want_f))
        whole = Arr(g, ca, W, H, 0, dtype)
        whole.fill(0, 0, 0, want_f)
        n_load_whole = counted(load, g.CudaArrayImage(whole.handle, W, H, dtype))
        whole_tg = Arr(g, ca, W, H, 0, dtype)
        whole_tg.fill(0, 0, 0, bg)
        n_obj_whole = counted(objects, g.CudaArrayImage(whole.handle, W, H, dtype), g.CudaArrayImage(whole_tg.handle, W, H, dtype))

        for pname, (aw, ah, x, y) in PLACEMENTS.items():
            for layers, k in ((0, None), (3, 1)):
                what = "%s, %s" % (pname, "layer %d" % k if layers else "2-D")
                A = Arr(g, ca, aw, ah, layers, dtype)
                frame(A.rect(x, y, W, H, k))
                A.check(ctx, [(k, x, y, want_f)], "gs_frame " + what)
                A = Arr(g, ca, aw, ah, layers, dtype)
                frame(A.rect(x, y, W, H, k), selected=sel)
                A.check(ctx, [(k, x, y, want_sel)], "gs_frame with a selection " + what)
                A = Arr(g, ca, aw, ah, layers, dtype)
                A.fill(k, x, y, want_f)
                assert counted(load, A.rect(x, y, W, H, k)) == n_load_whole, what
                A.check(ctx, [(k, x, y, want_load)], "GS_FLAG_LOAD_RT " + what)
                A, B = Arr(g, ca, aw, ah, layers, dtype), Arr(g, ca, aw, ah, layers, dtype)
                B.fill(k, x, y, bg)
                frame(A.rect(x, y, W, H, k), B.rect(x, y, W, H, k))
                A.check(ctx, [(k, x, y, want_ftg[0])], "gs_frame rt " + what)
                B.check(ctx, [(k, x, y, want_ftg[1])], "gs_frame camera target " + what)
                A, B = Arr(g, ca, aw, ah, layers, dtype), Arr(g, ca, aw, ah, layers, dtype)
                B.fill(k, x, y, bg)
                assert counted(objects, A.rect(x, y, W, H, k), B.rect(x, y, W, H, k)) == n_obj_whole, what
                A.check(ctx, [(k, x, y, want_obj[0])], "gs_frame_objects rt " + what)
                B.check(ctx, [(k, x, y, want_obj[1])], "gs_frame_objects camera target " + what)

        # staged gs_render, then gs_composite, with rt and camera target disjoint rectangles of one array
        t = _tensor(zeros)
        r.ResetOrder(); r.SortPoints(cam); r.CalcViewData(cam); r.DrawSplats(cam, t)
        want_r = _host(ctx, t)
        tg = _tensor(bg)
        r.Composite(t, tg)
        want_c = _host(ctx, tg)
        for layers, k in ((0, None), (3, 2)):
            A = Arr(g, ca, 420, 130, layers, dtype)
            A.fill(k, 211, 7, bg)
            rt_im, tg_im = A.rect(3, 5, W, H, k), A.rect(211, 7, W, H, k)
            r.ResetOrder(); r.SortPoints(cam); r.CalcViewData(cam); r.DrawSplats(cam, rt_im)
            r.Composite(rt_im, tg_im)
            A.check(ctx, [(k, 3, 5, want_r), (k, 211, 7, want_c)], "gs_render + gs_composite, %d layers" % layers)

        # the Unity render-thread event (gs_frame) with a GS_MEM_ARRAY_RECT render target
        fp, _keep = g.make_frame_params(cam, r.localToWorldMatrix, r.m_SplatScale, r.m_OpacityScale, r.m_SHOrder, r.m_SHOnly)
        A = Arr(g, ca, 301, 157, 0, dtype)
        rt_im = _image(A.rect(37, 19, W, H), W, H)   # points to the rectangle's descriptor, which rt_im keeps alive
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
    bgs = [_background(h, w, np.float16, 20 + i) for i, (_, _, w, h) in enumerate(TILES)]
    ctx.set_timing(True)
    try:
        # the definition: the camera loop, gs_frame_objects per camera into images of its own
        loop = _quilt_renderers(g, ctx, assets)
        rts = [_tensor(np.zeros((h, w, 4), np.float16)) for (_, _, w, h) in TILES]
        tgs = [_tensor(bg) for bg in bgs]
        n0 = launches(ctx)
        for c, cam in enumerate(cams):
            assert len(g.SortAndRenderSplatsMulti(loop, cam, rts[c], tgs[c])) == 2
        n_loop = launches(ctx) - n0
        want_rt, want_tg = [_host(ctx, t) for t in rts], [_host(ctx, t) for t in tgs]
        want_order = [r.readback_order() for r in loop]
        assert all(x.any() for x in want_rt)

        # the same cameras in one gs_frame_cameras call into separate arrays
        sep = _quilt_renderers(g, ctx, assets)
        sep_rt = [Arr(g, ca, w, h, 0) for (_, _, w, h) in TILES]
        sep_tg = [Arr(g, ca, w, h, 0) for (_, _, w, h) in TILES]
        for t, bg in zip(sep_tg, bgs):
            t.fill(0, 0, 0, bg)
        n0 = launches(ctx)
        actives = g.SortAndRenderCameras(sep, cams, [a.rect(0, 0, a.w, a.h) for a in sep_rt], [a.rect(0, 0, a.w, a.h) for a in sep_tg])
        n_sep = launches(ctx) - n0
        assert g.renderer.cameras_in_one_call(actives)

        # and into the tiles of one colour array, with the camera targets in the tiles of another
        call = _quilt_renderers(g, ctx, assets)
        A, B = Arr(g, ca, 400, 170, layers), Arr(g, ca, 400, 170, layers)
        for (x, y, _, _), bg in zip(TILES, bgs):
            B.fill(k, x, y, bg)
        n0 = launches(ctx)
        g.SortAndRenderCameras(call, cams, [A.rect(x, y, w, h, k) for (x, y, w, h) in TILES],
                               [B.rect(x, y, w, h, k) for (x, y, w, h) in TILES])
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
        ims = [A.rect(x, y, w, h) for (x, y, w, h) in tiles]
        if first == "whole":
            ims[0] = g.CudaArrayImage(A.handle, aw, ah)
        return ims

    ctx.set_timing(True)
    try:
        loop = _quilt_renderers(g, ctx, assets)
        L = Arr(g, ca, aw, ah)
        n0 = launches(ctx)
        for cam, im in zip(cams, images(L)):
            g.SortAndRenderSplatsMulti(loop, cam, im)
        n_loop = launches(ctx) - n0
        ctx.sync()
        want = L.read()
        call = _quilt_renderers(g, ctx, assets)
        A = Arr(g, ca, aw, ah)
        n0 = launches(ctx)
        g.SortAndRenderCameras(call, cams, images(A))
        n_call = launches(ctx) - n0
        ctx.sync()
        assert np.array_equal(_bits(A.read()), _bits(want))
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
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 40000, 0x5EED0095, "Medium")
    cam = camera(g, W, H)
    depth = _wall(g, cam, W, H)
    x, y = 37, 19
    # the rest of every depth array holds 1.0, which hides every splat: a wrong offset or layer shows
    flat = np.ones((157, 301), np.float32)
    flat[y:y + H, x:x + W] = depth
    layered = np.ones((3, 157, 301), np.float32)
    layered[2, y:y + H, x:x + W] = depth
    a2d, a3 = depth_array(ca, 301, 157, 0, flat), depth_array(ca, 301, 157, 3, layered)
    r = g.GaussianSplatRenderer(asset, ctx)

    def draw(d):
        r.sceneDepth = d
        r.ResetOrder()
        t = _tensor(np.zeros((H, W, 4), np.float16))
        r.SortAndRenderSplats(cam, rt=t)
        return _host(ctx, t)

    want = draw(_tensor(depth))
    assert not np.array_equal(_bits(want), _bits(draw(None))), "the wall hides nothing"
    for d in (g.CudaArrayDepth(a2d, W, H, origin=(x, y)), g.CudaArrayDepth(a3, W, H, layer=2, origin=(x, y))):
        assert np.array_equal(_bits(draw(d)), _bits(want))
    assert not draw(g.CudaArrayDepth(a3, W, H, layer=1, origin=(x, y))).any()

    # two cameras of one gs_frame_cameras call, each depth-tested against its tile of one depth array
    cams = [camera(g, W, H, pos=(s * 0.032, 0.5, -6.0)) for s in (-1, 1)]
    depths = [_wall(g, c, W, H) for c in cams]
    depths[1] = np.ascontiguousarray(depths[1][:, ::-1])
    tiles = [(0, 0), (210, 30)]
    atlas = np.ones((160, 420), np.float32)
    for (tx, ty), d in zip(tiles, depths):
        atlas[ty:ty + H, tx:tx + W] = d
    a_atlas = depth_array(ca, 420, 160, 0, atlas)

    def cameras(ds):
        fps = (N.GsFrameParams * 2)()
        keep = []
        for i, (c, d) in enumerate(zip(cams, ds)):
            fps[i], kp = g.make_frame_params(c, splat_count=asset.splatCount, scene_depth=d)
            keep.append(kp)
        assets = (C.c_void_p * 2)(*([C.cast(r._asset, C.c_void_p).value] * 2))
        do_sort = (C.c_int32 * 2)(1, 1)
        counts = (C.c_uint32 * 2)(1, 1)
        ts = [_tensor(np.zeros((H, W, 4), np.float16)) for _ in cams]
        ims = [_image(t, W, H) for t in ts]
        a = (C.POINTER(N.GsImage) * 2)(*[C.pointer(im) for im in ims])
        b = (C.POINTER(N.GsImage) * 2)(C.POINTER(N.GsImage)(), C.POINTER(N.GsImage)())
        r.ResetOrder()
        assert ctx._lib.gs_frame_cameras(ctx.handle, 2, counts, assets, fps, do_sort, C.byref(N.GsRenderOptions()), a, b) == 0
        return [_host(ctx, t) for t in ts]

    want = cameras([_tensor(d) for d in depths])
    got = cameras([g.CudaArrayDepth(a_atlas, W, H, origin=t) for t in tiles])
    for e in range(2):
        assert np.array_equal(_bits(got[e]), _bits(want[e])), "camera %d" % e
    r.Dispose()


# ---- 4. groups -------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_emulated_group_into_rects_equals_one_gpu(g, ctx, ca):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    assets = _assets(g)
    mats = [g.trs(position=(0.3, 0.0, 1.0)).astype(np.float32), g.trs(position=(-0.6, 0.1, 0.2)).astype(np.float32)]
    cam = camera(g, W, H)
    bg = _background(H, W, np.float16, 13)
    rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]
    for r, m in zip(rs, mats):
        r.localToWorldMatrix = m
    rt, tg = _tensor(np.zeros((H, W, 4), np.float16)), _tensor(bg)
    g.SortAndRenderSplatsMulti(rs, cam, rt, tg)
    want_rt, want_tg = _host(ctx, rt), _host(ctx, tg)
    for r in rs:
        r.Dispose()

    grp = GaussianSplatGroup.create(assets[0], [0, 0], emulate=True)
    objs = [grp, grp.add_object(assets[1])]
    for o, m in zip(objs, mats):
        o.localToWorldMatrix = m
    # member i draws into the rectangle at (37 i, 19) of layer i of its own array, and composites onto the rectangle at (11, 7 i)
    # of a 2-D array
    A = [Arr(g, ca, 301, 157, 2) for _ in range(2)]
    B = [Arr(g, ca, 260, 140, 0) for _ in range(2)]
    for i in range(2):
        B[i].fill(0, 11, 7 * i, bg)
    grp.SortAndRenderSplatsMulti(objs, cam, rts=[A[i].rect(37 * i, 19, W, H, i) for i in range(2)],
                                 camera_targets=[B[i].rect(11, 7 * i, W, H) for i in range(2)])
    grp.sync()
    for i in range(2):
        A[i].check(ctx, [(i, 37 * i, 19, want_rt)], "member %d rt" % i)
        B[i].check(ctx, [(0, 11, 7 * i, want_tg)], "member %d camera target" % i)
    # a depth rectangle is refused: the members share the frame parameters, and an array belongs to one device
    da = depth_array(ca, 301, 157, 0, np.zeros((157, 301), np.float32))
    grp.sceneDepth = g.CudaArrayDepth(da, W, H, origin=(3, 4))
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
        "good": (good, 0), "good3": (good3, 2),
        "3-D": (ca.array(200, 150, 2, flags=SURFACE_LOAD_STORE, fill=SENTINEL), 2),   # a 3-D array that is not layered
        "no surface": (ca.array(200, 150, 0, flags=0, fill=SENTINEL), 0),
        "wide": (ca.array(200, 150, 0, np.float32, fill=SENTINEL), 0),               # 4 x 32-bit for an RGBA16F image
    }
    image_cases = [   # (what, image, status, words of the message)
        ("null array", image(rect(0)), INVALID, "null"),
        ("reserved", image(rect(good, reserved=1)), INVALID, "reserved"),
        ("layer of a 2-D array", image(rect(good, layer=1)), INVALID, "layer"),
        ("layer out of range", image(rect(good3, layer=2)), INVALID, "layer"),
        ("layer 2^31", image(rect(good3, layer=1 << 31)), INVALID, "layer"),
        ("3-D array", image(rect(arrays["3-D"][0])), INVALID, "3-D"),
        ("no surface flag", image(rect(arrays["no surface"][0])), INVALID, "cudaArraySurfaceLoadStore"),
        ("past the right edge", image(rect(good, x=73)), INVALID, "inside"),
        ("past the bottom edge", image(rect(good3, y=55, layer=1)), INVALID, "inside"),
        ("origin that wraps", image(rect(good, x=2 ** 32 - 64)), INVALID, "inside"),
        ("row pitch", image(rect(good), pitch=w * 8), INVALID, "row_pitch_bytes"),
        ("channel format", image(rect(arrays["wide"][0])), UNSUPPORTED, "channel format"),
        ("memory kind 6", image(rect(good), memory=6), INVALID, "memory kind"),
    ]
    d2 = depth_array(ca, 200, 150, 0, np.zeros((150, 200), np.float32))
    d3 = depth_array(ca, 200, 150, 2, np.zeros((2, 150, 200), np.float32))
    depth_cases = [
        ("depth: null array", rect(0), INVALID),
        ("depth: reserved", rect(d2, reserved=1), INVALID),
        ("depth: layer of a 2-D array", rect(d2, layer=1), INVALID),
        ("depth: layer out of range", rect(d3, layer=2), INVALID),
        ("depth: 3-D array", rect(depth_array(ca, 200, 150, 2, flags=SURFACE_LOAD_STORE)), INVALID),
        ("depth: no surface flag", rect(depth_array(ca, 200, 150, 0, flags=0)), INVALID),
        ("depth: past the right edge", rect(d2, x=73), INVALID),
        ("depth: past the bottom edge", rect(d3, y=55, layer=1), INVALID),
        ("depth: origin that wraps", rect(d2, y=2 ** 32 - 8), INVALID),
        ("depth: RGBA16F array", rect(ca.array(200, 150, 0, np.float16)), UNSUPPORTED),
    ]
    rt_t = _tensor(np.full((h, w, 4), SENTINEL, np.float16))
    rt_lin = _image(rt_t, w, h)
    other = _image(_tensor(np.zeros((h, w, 4), np.float16)), w, h)
    opt = N.GsRenderOptions()
    no = (C.POINTER(N.GsImage) * 2)(C.POINTER(N.GsImage)(), C.POINTER(N.GsImage)())
    counts = (C.c_uint32 * 2)(1, 1)

    def params(depth=None):
        fps = (N.GsFrameParams * 2)()
        for i, x in enumerate(rs):
            fps[i] = x.frame_params(cam)
            if depth is not None:
                fps[i].scene_depth, fps[i].scene_depth_on_device = depth, N.GS_MEM_ARRAY_RECT
        assets = (C.c_void_p * 2)(*[C.cast(x._asset, C.c_void_p).value for x in rs])
        return fps, assets, (C.c_int32 * 2)(1, 1)

    def untouched(what):
        ctx.sync()
        assert (_host(ctx, rt_t) == np.float16(SENTINEL)).all(), what
        for name, (hd, layers) in arrays.items():
            dt = np.float32 if name == "wide" else np.float16
            assert (ca.download(hd, (max(layers, 1), 150, 200, 4), dt) == dt(SENTINEL)).all(), (what, name)
        for x, o in zip(rs, orders):
            assert np.array_equal(x.readback_order(), o), what

    ctx.set_timing(True)
    try:
        for what, im, status, words in image_cases:
            fps, assets, do_sort = params()
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
            fps, assets, do_sort = params(d)
            n0 = launches(ctx)
            assert lib.gs_frame(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), 1, C.byref(rt_lin), None) == status, what
            assert lib.gs_render(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), C.byref(rt_lin)) == status, what
            assert lib.gs_frame_objects(ctx.handle, 2, assets, fps, do_sort, C.byref(opt), C.byref(rt_lin), None) == status, what
            ims = (C.POINTER(N.GsImage) * 2)(C.pointer(rt_lin), C.pointer(other))
            assert lib.gs_frame_cameras(ctx.handle, 2, counts, assets, fps, do_sort, C.byref(opt), ims, no) == status, what
            assert launches(ctx) == n0, what
            untouched(what)
        # band-packed output and gs_unshuffle_bands output are linear memory only
        fps, assets, do_sort = params()
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
        A = Arr(g, ca, 200, 150)
        fps, assets, do_sort = params()
        im = _image(A.rect(72, 54, w, h), w, h)
        assert lib.gs_frame(ctx.handle, assets[0], C.byref(fps[0]), C.byref(opt), 1, C.byref(im), None) == 0
        ctx.sync()
        got = A.read()[0]
        inside = got[54:, 72:]
        assert not (inside == np.float16(SENTINEL)).all()
        got[54:, 72:] = np.float16(SENTINEL)
        assert (got == np.float16(SENTINEL)).all()
    finally:
        ctx.set_timing(False)
    for x in rs:
        x.Dispose()
