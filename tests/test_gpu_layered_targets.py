"""One layer of a layered CUDA array as an image (GS_MEM_ARRAY_LAYER): what an XR eye-texture array in single-pass-instanced
mode, or a cube map, looks like once it is imported into CUDA.  The library renders into and composites onto the layer in place,
through a layered surface, and leaves the array's other layers alone.

Arrays are made by images.Cudart, as every array test makes them.  Every result is compared byte for
byte with the same call on linear device memory (or, for the stereo run, with the camera loop it stands for), and every layer
the call does not name is checked to still hold its sentinel."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

from images import KIND_UNSIGNED, LAYERED, SENTINEL, SURFACE_LOAD_STORE, SharedArray, background, bits, ca, to_device, to_host  # noqa: F401
from util import camera

ROOT = Path(__file__).resolve().parents[1]

INVALID, UNSUPPORTED = -1, -4


def test_header_and_python_agree_on_gs_mem_array_layer():
    from unitygaussiansplatting_b200 import _native as N
    text = (ROOT / "include" / "gsplat_b200.h").read_text()
    m = re.search(r"#define GS_MEM_ARRAY_LAYER (\d+)u", text)
    assert m and int(m.group(1)) == N.GS_MEM_ARRAY_LAYER == 4
    m = re.search(r"typedef struct GsArrayLayer \{([^}]*)\} GsArrayLayer;", text)
    assert m and re.findall(r"(\w+);", m.group(1)) == ["array", "layer", "reserved"]
    assert [f[0] for f in N.GsArrayLayer._fields_] == ["array", "layer", "reserved"] and C.sizeof(N.GsArrayLayer) == 16


def test_cuda_array_image_layer_argument(g):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    im = _image(g.CudaArrayImage(0x1234, 8, 4, np.float32, layer=5), 8, 4)
    assert im.memory == N.GS_MEM_ARRAY_LAYER and im.row_pitch_bytes == 0 and im.format == N.GS_PIX_RGBA32F
    desc = N.GsArrayLayer.from_address(im.data)
    assert (desc.array, desc.layer, desc.reserved) == (0x1234, 5, 0)
    assert _image(g.CudaArrayImage(0x1234, 8, 4), 8, 4).memory == N.GS_MEM_ARRAY
    with pytest.raises(ValueError):
        g.CudaArrayImage(0x1234, 8, 4, layer=-1)


# ---- 1. byte identity of every entry point ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,blend", [(np.float16, 0), (np.float16, 1), (np.float32, 0), (np.float32, 1)],
                         ids=["rgba16f-rop", "rgba16f-fp32", "rgba32f-rop", "rgba32f-fp32"])
def test_layer_equals_linear_target(g, ctx, ca, dtype, blend):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    W, H = 272, 176
    depth, k = (3, 1) if dtype == np.float16 else (6, 4)
    a = g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED0C01, "Medium")
    b = g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0C02, "VeryHigh")
    cam = camera(g, W, H)
    bg = background(H, W, dtype, 5)
    zeros = np.zeros((H, W, 4), dtype)

    def renderer(asset, **kn):
        r = g.GaussianSplatRenderer(asset, ctx)
        r.blend_mode = blend
        for key, v in kn.items():
            setattr(r, key, v)
        return r

    def both(draw, rt_fill=None, tgt=False):
        """draw(rt, tgt) once on device tensors and once on layer k of two layered arrays; the results must agree."""
        rt_t = to_device(zeros if rt_fill is None else rt_fill)
        tg_t = to_device(bg) if tgt else None
        draw(rt_t, tg_t)
        want_rt, want_tg = to_host(ctx, rt_t), (to_host(ctx, tg_t) if tgt else None)
        A = SharedArray(g, ca, W, H, depth, dtype)
        if rt_fill is not None:
            A.fill(k, 0, 0, rt_fill)
        B = SharedArray(g, ca, W, H, depth, dtype) if tgt else None
        if tgt:
            B.fill(k, 0, 0, bg)
        draw(A.view(layer=k), B.view(layer=k) if tgt else None)
        return want_rt, want_tg, A, B

    # gs_frame, then gs_frame with GS_FLAG_LOAD_RT over what it drew, and gs_frame with a camera target
    r = renderer(a)
    want, _, A, _ = both(lambda rt, tg: (r.ResetOrder(), r.SortAndRenderSplats(cam, rt=rt)))
    assert want.any()
    A.check(ctx, [(k, 0, 0, want)], "gs_frame")
    r2 = renderer(b, localToWorldMatrix=g.trs(position=(-1.0, 0.2, 0.5)).astype(np.float32), load_rt=True)
    want2, _, A2, _ = both(lambda rt, tg: (r2.ResetOrder(), r2.SortAndRenderSplats(cam, rt=rt)), rt_fill=want)
    assert not np.array_equal(bits(want2), bits(want))
    A2.check(ctx, [(k, 0, 0, want2)], "gs_frame with GS_FLAG_LOAD_RT")
    r2.load_rt = False
    want, want_tg, A, B = both(lambda rt, tg: (r.ResetOrder(), r.SortAndRenderSplats(cam, rt=rt, camera_target=tg)), tgt=True)
    A.check(ctx, [(k, 0, 0, want)], "gs_frame rt")
    B.check(ctx, [(k, 0, 0, want_tg)], "gs_frame camera target")
    assert not np.array_equal(bits(want_tg), bits(bg))

    # gs_render (staged) and gs_composite
    want_r, _, A, _ = both(lambda rt, tg: (r.ResetOrder(), r.SortPoints(cam), r.CalcViewData(cam), r.DrawSplats(cam, rt)))
    A.check(ctx, [(k, 0, 0, want_r)], "gs_render")
    src = SharedArray(g, ca, W, H, depth, dtype)
    src.fill(depth - 1 - k, 0, 0, want)   # another layer index for the source: the two layers are read and written independently
    for source in (to_device(want), src.view(layer=depth - 1 - k)):
        _, want_c, _, B = both(lambda rt, tg: r.Composite(source, tg), tgt=True)
        B.check(ctx, [(k, 0, 0, want_c)], "gs_composite")

    # gs_frame_objects (two objects, one call), render target and camera target on layers
    ra, rb = renderer(a), renderer(b, localToWorldMatrix=g.trs(position=(1.5, 0.0, 3.0)).astype(np.float32))

    def multi(rt, tg):
        for x in (ra, rb):
            x.ResetOrder()
            x.m_FrameCounter = 0
        assert g.renderer.draws_in_one_call(g.GatherSplatsForCamera([ra, rb], cam))
        g.SortAndRenderSplatsMulti([ra, rb], cam, rt, tg)

    want, want_tg, A, B = both(multi, tgt=True)
    A.check(ctx, [(k, 0, 0, want)], "gs_frame_objects rt")
    B.check(ctx, [(k, 0, 0, want_tg)], "gs_frame_objects camera target")

    # the Unity render-thread event (gs_frame), render target and camera target on layers
    fp, _keep = g.make_frame_params(cam, r.localToWorldMatrix, r.m_SplatScale, r.m_OpacityScale, r.m_SHOrder, r.m_SHOnly)

    def event(rt, tg):
        ev = N.GsUnityFrameEvent()
        ev.ctx, ev.asset = C.cast(ctx.handle, C.c_void_p).value, C.cast(r._asset, C.c_void_p).value
        C.memmove(C.byref(ev.params), C.byref(fp), C.sizeof(fp))
        ev.options.blend_mode = blend
        ev.do_sort, ev.status, ev.has_rt, ev.has_camera_target = 1, -5, 1, 1
        ims = (_image(rt, W, H), _image(tg, W, H))   # the images point to the arrays' layer descriptors: rt / tg stay alive
        ev.rt, ev.camera_target = ims
        fn = N.native().gs_unity_get_render_event_func()
        fn(N.GS_UNITY_EVENT_FRAME, C.addressof(ev))
        assert ev.status == 0
        fn(N.GS_UNITY_EVENT_SYNC, C.addressof(ev))
        assert ev.status == 0

    r.ResetOrder()
    want, want_tg, A, B = both(lambda rt, tg: (r.ResetOrder(), event(rt, tg)), tgt=True)
    A.check(ctx, [(k, 0, 0, want)], "Unity event rt")
    B.check(ctx, [(k, 0, 0, want_tg)], "Unity event camera target")
    for x in (r, r2, ra, rb):
        x.Dispose()


# ---- 2. a stereo pair as one camera run ------------------------------------------------------------------------------------------
def _eyes(g, W, H, ipd=0.064):
    return [camera(g, W, H, pos=(s * ipd / 2, 0.5, -6.0)) for s in (-1.0, 1.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("same_layer", [False, True], ids=["eyes-on-two-layers", "eyes-on-one-layer"])
def test_stereo_pair_on_layers_is_the_camera_loop(g, ctx, ca, same_layer):
    W, H = 256, 192
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED0C11, "Medium"),
              g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0C12, "VeryHigh")]
    mats = [g.trs(position=(0.3, 0.0, 1.0)).astype(np.float32), g.trs(position=(-0.6, 0.1, 0.2)).astype(np.float32)]
    eyes = _eyes(g, W, H)
    bg = background(H, W, np.float16, 9)

    def renderers():
        rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]
        for r, m in zip(rs, mats):
            r.localToWorldMatrix = m
        return rs

    ctx.set_timing(True)
    try:
        # the definition: the camera loop, gs_frame_objects per eye into images of its own
        loop = renderers()
        rts = [to_device(np.zeros((H, W, 4), np.float16)) for _ in eyes]
        tgts = [to_device(bg) for _ in eyes]
        if same_layer:
            rts[1] = rts[0]
        n0 = ctx.stage_times().kernel_launches
        for e, cam in enumerate(eyes):
            active = g.SortAndRenderSplatsMulti(loop, cam, rts[e], tgts[e])
            assert len(active) == 2
        n_loop = ctx.stage_times().kernel_launches - n0
        want_rt = [to_host(ctx, t) for t in rts]
        want_tg = [to_host(ctx, t) for t in tgts]
        want_order = [r.readback_order() for r in loop]
        assert all(x.any() for x in want_rt) and (same_layer or not np.array_equal(want_rt[0], want_rt[1]))

        # the pair drawn by gs_frame_cameras into two separate 2-D arrays: the run it forms
        flat = renderers()
        flat_rts = [ca.array(W, H, 0, flags=SURFACE_LOAD_STORE, fill=0.0) for _ in eyes]
        n0 = ctx.stage_times().kernel_launches
        g.SortAndRenderCameras(flat, eyes, [g.CudaArrayImage(h, W, H) for h in flat_rts],
                               [to_device(bg) for _ in eyes])
        n_flat = ctx.stage_times().kernel_launches - n0

        # and into layers: rts on layers 0 and 1 of one array (or both on layer 0), camera targets on layers of another
        call = renderers()
        A, B = SharedArray(g, ca, W, H, 3), SharedArray(g, ca, W, H, 3)
        for e in range(2):
            B.fill(e, 0, 0, bg)
        rt_layers = [0, 0] if same_layer else [0, 1]
        n0 = ctx.stage_times().kernel_launches
        actives = g.SortAndRenderCameras(call, eyes, [A.view(layer=k) for k in rt_layers], [B.view(layer=0), B.view(layer=1)])
        n_call = ctx.stage_times().kernel_launches - n0
        assert all(len(a) == 2 for a in actives)
        assert g.renderer.cameras_in_one_call(actives)
        A.check(ctx, [(rt_layers[e], 0, 0, want_rt[e]) for e in range(2)], "render targets")
        B.check(ctx, [(e, 0, 0, want_tg[e]) for e in range(2)], "camera targets")
        for r, o in zip(call, want_order):
            assert np.array_equal(r.readback_order(), o), "draw order differs"
        if same_layer:   # one layer drawn twice: two runs, as the loop draws it
            assert n_call == n_loop
        else:            # two layers of one array: one run, as two separate arrays are
            assert n_call == n_flat < n_loop
        for r in loop + flat + call:
            r.Dispose()
    finally:
        ctx.set_timing(False)


# ---- 3. groups -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("members", [1, 2, 4])
def test_emulated_group_objects_into_layers_equal_one_gpu(g, ctx, ca, members):
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    W, H = 320, 240
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED0C21, "Medium"),
              g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0C22, "Medium")]
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
    assert want_rt.any()

    grp = GaussianSplatGroup.create(assets[0], [0] * members, emulate=True)
    objs = [grp, grp.add_object(assets[1])]
    for o, m in zip(objs, mats):
        o.localToWorldMatrix = m
    # member i draws into layer i % 3 of its own array A[i], and composites onto layer (i + 1) % 3 of B[i]
    A = [SharedArray(g, ca, W, H, 3) for _ in range(members)]
    B = [SharedArray(g, ca, W, H, 3) for _ in range(members)]
    for i in range(members):
        B[i].fill((i + 1) % 3, 0, 0, bg)
    grp.SortAndRenderSplatsMulti(objs, cam, rts=[A[i].view(layer=i % 3) for i in range(members)],
                                 camera_targets=[B[i].view(layer=(i + 1) % 3) for i in range(members)])
    grp.sync()
    for i in range(members):
        A[i].check(ctx, [(i % 3, 0, 0, want_rt)], "member %d rt" % i)
        B[i].check(ctx, [((i + 1) % 3, 0, 0, want_tg)], "member %d camera target" % i)
    grp.close()


# ---- 4. refusals -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_layer_refusals_write_nothing(g, ctx, ca):
    import torch
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0C31, "Medium")
    cam = camera(g, 128, 128)
    r = g.GaussianSplatRenderer(asset, ctx)
    fp = r.frame_params(cam)
    descs = []

    def image(handle, layer=0, memory=N.GS_MEM_ARRAY_LAYER, fmt=N.GS_PIX_RGBA16F, pitch=0, height=128, reserved=0):
        if memory == N.GS_MEM_ARRAY_LAYER and handle is not None:
            descs.append(N.GsArrayLayer(handle, layer, reserved))
            data = C.addressof(descs[-1])
        else:
            data = handle
        return N.GsImage(data, 128, height, pitch, fmt, memory)

    def frame(im, opt=None):
        return lib.gs_frame(ctx.handle, r._asset, C.byref(fp), C.byref(opt or r._options()), 1, C.byref(im), None)

    def unchanged(h, fill=SENTINEL):
        ctx.sync()
        got = ca.download(h)
        return np.array_equal(bits(got), bits(np.full_like(got, fill)))

    good = ca.array(128, 128, 2, fill=SENTINEL)
    flat = ca.array(128, 128, 0, flags=SURFACE_LOAD_STORE, fill=SENTINEL)             # a 2-D array
    no_surface = ca.array(128, 128, 2, flags=LAYERED, fill=SENTINEL)                  # no cudaArraySurfaceLoadStore
    wide = ca.array(128, 128, 2, np.float32, fill=SENTINEL)                           # 4 x 32-bit for an RGBA16F image
    bytes8 = ca.array(128, 128, 2, np.uint8, kind=KIND_UNSIGNED, fill=7)              # 4 x 8-bit
    cases = [
        (image(good, layer=2), INVALID, "layer"),                                     # layer == depth
        (image(good, layer=1 << 31), INVALID, "layer"),
        (image(flat), INVALID, "layered"),                                            # a 2-D array under kind 4
        (image(good, memory=N.GS_MEM_ARRAY), INVALID, "2-D array"),                   # a layered array under GS_MEM_ARRAY
        (image(no_surface), INVALID, "cudaArraySurfaceLoadStore"),
        (image(wide), UNSUPPORTED, "channel format"),
        (image(bytes8), UNSUPPORTED, "channel format"),
        (image(good, pitch=128 * 8), INVALID, "row_pitch_bytes"),
        (image(None), INVALID, "null"),                                               # a NULL descriptor
        (image(good, reserved=1), INVALID, "reserved"),
        (image(good, memory=3), INVALID, "memory kind"),                              # 3 stays undefined
    ]
    for im, code, words in cases:
        assert frame(im) == code, words
        assert words in lib.gs_last_error(ctx.handle).decode(), words
    opt = r._options()                                                          # band-packed output (one partition's rows)
    opt.partition_index, opt.partition_count, opt.band_rows, opt.band_packed = 0, 2, 1, 1
    assert frame(image(good, height=64), opt) == INVALID
    assert "band_packed" in lib.gs_last_error(ctx.handle).decode()
    gathered = torch.zeros((2, 64, 128, 4), dtype=torch.float16, device="cuda")   # gs_unshuffle_bands into a layer
    im = image(good)
    assert lib.gs_unshuffle_bands(ctx.handle, C.c_void_p(gathered.data_ptr()), 2, 1, 64, N.GS_PIX_RGBA16F, C.byref(im)) == INVALID
    # gs_composite refuses a bad layer on either side, before it writes anything
    src = to_device(np.full((128, 128, 4), 0.5, np.float16))
    dev = N.GsImage(src.data_ptr(), 128, 128, 0, N.GS_PIX_RGBA16F, N.GS_MEM_DEVICE)
    assert lib.gs_composite(ctx.handle, C.byref(dev), C.byref(image(good, layer=5))) == INVALID
    assert lib.gs_composite(ctx.handle, C.byref(image(good, layer=5)), C.byref(image(good, layer=0))) == INVALID
    assert unchanged(good) and unchanged(flat) and unchanged(no_surface) and unchanged(wide)
    assert unchanged(bytes8, 7)
    # and the same array, correctly described, is accepted: layer 1 drawn, layer 0 left as it was
    assert frame(image(good, layer=1)) == 0
    ctx.sync()
    got = bits(ca.download(good))
    sentinel = bits(np.full((128, 128, 4), SENTINEL, np.float16))
    assert np.array_equal(got[0], sentinel) and not np.array_equal(got[1], sentinel)
    r.Dispose()
