"""gs_frame_objects: several splat objects of one camera drawn by one call on one GPU, against the per-object loop it stands
for -- gs_frame per object (GS_FLAG_LOAD_RT from the second on), then gs_composite.  Every comparison is bit for bit, on the
render target, the camera target and every object's persistent draw order and sorted keys, over several orbit frames (so the
orders evolve and the objects' draw order changes).  The loop and the call each own a copy of every object, on the same
context (frame_loops.Twins)."""
import ctypes as C

import numpy as np
import pytest

from frame_loops import Twins, call_frame, compare_frame, frame_args, loop_frame, mixed_assets, next_sort, orbit
from images import ca  # noqa: F401
from util import CAP_ENTRIES, CAP_H, CAP_SPLATS, CAP_W, bin_row_splats, camera, pixels_per_unit, splat_records, world_at_pixel

pytestmark = pytest.mark.gpu

INVALID, OOM = -1, -3


# ---- 1. mixed scenes ------------------------------------------------------------------------------------------------------
RT_KINDS = ["host", "device", "array", None]
TGT_KINDS = [None, "host", "device", "array"]


@pytest.mark.parametrize("K", [2, 3, 5])
@pytest.mark.parametrize("blend", [0, 1])
@pytest.mark.parametrize("dtype", [np.float16, np.float32])
def test_mixed_scenes_equal_the_loop(g, ctx, ca, K, blend, dtype):
    assets = mixed_assets(g, K, 0x5EED0F00)

    def setup(i, r):
        s = -1.0 if i == 1 else 1.0    # object 1 is mirrored
        r.localToWorldMatrix = g.trs(position=(1.4 * i - 1.5, 0.2 * i, 0.8 * (i % 2)), scale=(0.8 * s, 0.8, 0.8)).astype(np.float32)
        r.m_SHOrder = (3, 1, 0, 2, 3)[i]
        r.m_SortNthFrame = (1, 2, 1, 3, 1)[i]
        if i == 0:
            r.m_Cutouts = [(np.diag([1 / 0.8, 1 / 0.8, 1 / 0.8, 1.0]).astype(np.float32), 1 | 0x100)]
        if i == 2:
            bits = np.random.default_rng(i).integers(0, 2 ** 32, (r.splatCount + 31) // 32, dtype=np.uint64).astype(np.uint32)
            r.m_DeletedBits = bits & np.uint32(0x11111111)

    tw = Twins(g, ctx, assets, setup)
    try:
        for f in range(4):
            rt_kind = RT_KINDS[f]
            tgt_kind = TGT_KINDS[(f + K) % 4] if rt_kind is not None else "device"
            compare_frame(g, ctx, ca, tw, orbit(g, f), blend, dtype, rt_kind, tgt_kind,
                           "frame %d (rt %s, target %s)" % (f, rt_kind, tgt_kind))
    finally:
        tw.dispose()


def test_async_readback_equals_the_loop(g, ctx):
    import torch
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, 8000, 0x5EED0F10 + i, "Medium") for i in range(3)]

    def setup(i, r):
        r.localToWorldMatrix = g.trs(position=(1.2 * i - 1.2, 0.0, 0.5 * i)).astype(np.float32)

    tw = Twins(g, ctx, assets, setup)
    try:
        cam = orbit(g, 1)
        W, H = cam.pixelWidth, cam.pixelHeight
        lo, hi = tw.ordered(g, cam)
        want = np.zeros((H, W, 4), np.float16)
        loop_frame(g, ctx, lo, cam, 0, want, None)
        pin = torch.zeros((H, W, 4), dtype=torch.float16).pin_memory()
        call_frame(g, ctx, hi, cam, 0, pin.numpy(), None, flags=1)
        ctx.sync()
        assert want.any() and np.array_equal(pin.numpy().view(np.uint16), want.view(np.uint16))
        tw.check_state()
    finally:
        tw.dispose()


# ---- 2. against the oracle ------------------------------------------------------------------------------------------------
def test_three_objects_against_the_oracle(g, O, ctx):
    """SortAndRenderSplatsMulti now draws in one call; the oracle draws the concatenated, per-object-sorted list."""
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, n, 0x5EED0F20 + i, q) for i, (n, q) in enumerate([(20000, "Medium"), (15000, "VeryHigh"), (10000, "Medium")])]
    rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]
    try:
        for i, r in enumerate(rs):
            r.localToWorldMatrix = g.trs(position=(1.3 * i - 1.3, 0.1 * i, 2.0 - 1.0 * i), scale=(0.7, 0.7, 0.7)).astype(np.float32)
        cam = camera(g, 400, 300)
        rt = np.zeros((300, 400, 4), np.float16)
        active = g.SortAndRenderSplatsMulti(rs, cam, rt)
        assert active == [rs[2], rs[1], rs[0]]
        views, orders, base = [], [], 0
        for r in active:
            fp, _keep = g.make_frame_params(cam, r.localToWorldMatrix)
            ref = O.frame(r.m_Asset, fp, threads=O.max_threads())
            assert np.array_equal(r.readback_order(), ref["order"])
            views.append(ref["view"]); orders.append(ref["order"] + np.uint32(base)); base += r.splatCount
        want = O.render(np.concatenate(views), np.concatenate(orders), 400, 300, 0, O.max_threads())
        assert rt.any() and np.array_equal(rt.astype(np.float32), want)
    finally:
        for r in rs:
            r.Dispose()


# ---- 3. selection and depth in one run ------------------------------------------------------------------------------------
@pytest.mark.parametrize("blend", [0, 1])
def test_selection_and_depth_in_one_run(g, ctx, ca, blend):
    import torch
    cam0 = orbit(g, 0)
    W, H = cam0.pixelWidth, cam0.pixelHeight
    depth = np.full((H, W), 0.02, np.float32)           # reversed Z: most splats are in front, some behind
    depth[:, W // 2:] = 0.2
    depth[H // 3:H // 2, :] = np.nan                    # NaN fails LEqual for the depth-tested object only
    depth_dev = torch.from_numpy(depth).cuda()
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, 9000, 0x5EED0F30 + i, "Medium") for i in range(3)]

    def setup(i, r):
        r.localToWorldMatrix = g.trs(position=(1.0 * i - 1.0, 0.0, 0.6 * i)).astype(np.float32)
        if i == 0:
            sel = np.zeros((r.splatCount + 31) // 32, np.uint32)
            sel[::3] = 0x0F0F0F0F
            r.m_SelectedBits = sel
        if i == 1:
            r.sceneDepth = depth_dev

    tw = Twins(g, ctx, assets, setup)
    try:
        for f in range(3):
            compare_frame(g, ctx, ca, tw, orbit(g, f), blend, np.float16, "device", "host", "frame %d" % f)
    finally:
        tw.dispose()


# ---- 4. rounding at an object boundary ------------------------------------------------------------------------------------
def test_fp32_blend_into_half_rounds_at_each_object(g, ctx, ca):
    """Object 0 (three splats of opacity 0.99) leaves alpha between 1 - 2^-12 and 1 over a disc: half 1.0, float < 1.  Object 1,
    behind it, is bright.  The loop stores object 0's result as half, so object 1 adds nothing there; without rounding at
    the boundary it would."""
    W, H = 128, 96
    cam = camera(g, W, H)
    ppu = pixels_per_unit(cam, 6.0)
    pos0 = world_at_pixel(cam, [64.0] * 3, [48.0] * 3, [6.0, 6.05, 6.1])
    rec0 = splat_records(pos0, np.array([[30.0, 30.0, 30.0]] * 3) / ppu, [0.99] * 3, [[0.4, 0.3, 0.2], [0.1, 0.2, 0.3], [0.2, 0.2, 0.2]])
    pos1 = world_at_pixel(cam, [64.0], [48.0], [7.0])
    rec1 = splat_records(pos1, np.array([[40.0, 40.0, 40.0]]) / pixels_per_unit(cam, 7.0), [0.9], [[300.0, 300.0, 300.0]])
    assets = [g.create_asset(rec0, "VeryHigh"), g.create_asset(rec1, "VeryHigh")]
    tw = Twins(g, ctx, assets, lambda i, r: None)
    try:
        half = compare_frame(g, ctx, ca, tw, cam, 1, np.float16, "host", None, "RGBA16F")
        full = compare_frame(g, ctx, ca, tw, cam, 1, np.float32, "host", None, "RGBA32F")
        differs = (full.astype(np.float16).view(np.uint16) != half.view(np.uint16)).any(-1)
        assert differs.sum() > 20, "the float result rounded once must differ where object 0's alpha rounds to 1"
        assert (half[..., 3] == 1.0).sum() > 20 and ((full[..., 3] < 1.0) & (half[..., 3] == 1.0)).any()
    finally:
        tw.dispose()


# ---- 5. saturation across objects -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("blend", [0, 1])
def test_saturated_pixels_ignore_an_inf_colour_in_a_later_object(g, ctx, ca, blend):
    W, H = 160, 128
    cam = camera(g, W, H)
    ppu = pixels_per_unit(cam, 6.0)
    opaque = splat_records(world_at_pixel(cam, [77.3], [61.8], [6.0]), np.array([[10.0, 9.0, 9.5]]) / ppu, [0.2], [[0.9, 0.4, 0.1]])
    depth = np.r_[np.linspace(6.1, 6.4, 40), 6.5]
    pos = world_at_pixel(cam, np.r_[np.full(40, 79.0), 80.6], np.r_[np.full(40, 63.0), 66.1], depth)
    sigma = np.r_[np.tile([[31.0, 27.0, 29.0]], (40, 1)), [[30.0, 26.0, 28.0]]]
    dc = np.r_[np.tile([[0.2, 0.3, 0.6]], (40, 1)), [[1e6, 1e6, 1e6]]]
    behind = splat_records(pos, sigma / ppu, np.r_[np.full(40, 0.0002), 0.6], dc)
    assets = [g.create_asset(opaque, "VeryHigh"), g.create_asset(behind, "VeryHigh")]

    def setup(i, r):
        r.m_OpacityScale = 100.0

    tw = Twins(g, ctx, assets, setup)
    try:
        got = compare_frame(g, ctx, ca, tw, cam, blend, np.float32 if blend else np.float16, "device", None, "saturation")
        got = got.astype(np.float32)
        assert (got[..., 3] == 1.0).sum() > 100 and np.isposinf(got[..., :3]).any() and not np.isnan(got).any()
    finally:
        tw.dispose()


# ---- 6. run splits --------------------------------------------------------------------------------------------------------
def test_eighteen_objects_two_runs(g, ctx, ca):
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, 1500, 0x5EED0F40 + i, "Medium") for i in range(18)]

    def setup(i, r):
        r.localToWorldMatrix = g.trs(position=(0.5 * (i % 6) - 1.25, 0.5 * (i // 6) - 0.5, 0.1 * i), scale=(0.3, 0.3, 0.3)).astype(np.float32)

    tw = Twins(g, ctx, assets, setup)
    try:
        for f in range(2):
            compare_frame(g, ctx, ca, tw, orbit(g, f), f, np.float16, "host", "device", "frame %d" % f)
    finally:
        tw.dispose()


def test_two_depth_buffers_empty_and_offscreen_objects(g, ctx, ca):
    import torch
    cam0 = orbit(g, 0)
    W, H = cam0.pixelWidth, cam0.pixelHeight
    da = np.full((H, W), 0.03, np.float32)
    db = np.full((H, W), 0.03, np.float32)
    db[:, : W // 3] = np.nan
    da_dev, db_host = torch.from_numpy(da).cuda(), db
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, 5000, 0x5EED0F50 + i, "Medium") for i in range(6)]

    def setup(i, r):
        r.localToWorldMatrix = g.trs(position=(0.8 * i - 2.0, 0.0, 0.3 * i), scale=(0.6, 0.6, 0.6)).astype(np.float32)
        r.sceneDepth = {0: da_dev, 2: db_host, 3: da_dev}.get(i)
        if i == 4:    # zero drawable splats
            r.m_DeletedBits = np.full((r.splatCount + 31) // 32, 0xFFFFFFFF, np.uint32)
        if i == 5:    # entirely off screen (behind the camera's far side)
            r.localToWorldMatrix = g.trs(position=(0.0, 500.0, 0.0)).astype(np.float32)

    tw = Twins(g, ctx, assets, setup)
    try:
        for f in range(3):
            compare_frame(g, ctx, ca, tw, orbit(g, f), f % 2, np.float16, "array", "host" if f else None, "frame %d" % f)
    finally:
        tw.dispose()


# ---- 7. capacity ----------------------------------------------------------------------------------------------------------
def test_summed_entries_over_capacity_and_recovery(g):
    """The construction of test_bin_list_exact_capacity_overflow_and_recovery split across two objects: 65,537 splats of 64
    entries each overflow the 4 Mi list by one splat; deleting one splat makes the next call fit exactly."""
    ctx = g.GaussianSplatContext(0)
    tw = None
    try:
        cam = camera(g, CAP_W, CAP_H)
        rec = bin_row_splats(cam, CAP_SPLATS + 1, 0xCA9)
        half = CAP_SPLATS // 2
        assets = [g.create_asset(rec[:half].copy(), "VeryHigh"), g.create_asset(rec[half:].copy(), "VeryHigh")]
        tw = Twins(g, ctx, assets, lambda i, r: None)
        lo, hi = tw.ordered(g, cam)
        rt = np.zeros((CAP_H, CAP_W, 4), np.float16)
        assert call_frame(g, ctx, hi, cam, 0, rt, None, check=False) == OOM
        from unitygaussiansplatting_b200 import _native as N
        assert "tile-list capacity exceeded" in N.native().gs_last_error(ctx.handle).decode()
        for r in tw.loop + tw.call:   # one splat of the second object deleted in both copies
            if r.m_Asset is assets[1]:
                bits = np.zeros((r.splatCount + 31) // 32, np.uint32)
                bits[0] = 1
                r.m_DeletedBits = bits
        want = np.zeros_like(rt)
        loop_frame(g, ctx, lo, cam, 0, want, None)
        got = np.zeros_like(rt)
        call_frame(g, ctx, hi, cam, 0, got, None)
        assert ctx.stage_times().tile_entries == CAP_ENTRIES
        assert got.any() and np.array_equal(got.view(np.uint16), want.view(np.uint16))
    finally:
        if tw:
            tw.dispose()
        ctx.close()


# ---- 8. rejections --------------------------------------------------------------------------------------------------------
def test_refused_inputs_write_nothing(g, ctx):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    lib = N.native()
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, 4000, 0x5EED0F60 + i, "Medium") for i in range(2)]
    rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]
    other = g.GaussianSplatContext(0)
    foreign = g.GaussianSplatRenderer(assets[0], other)
    try:
        cam = camera(g, 160, 120)
        rt = np.full((120, 160, 4), 3, np.float16)
        im = _image(rt, 160, 120)
        orders = [r.readback_order() for r in rs]
        fps = (N.GsFrameParams * 2)(rs[0].frame_params(cam), rs[1].frame_params(cam))
        ds = (C.c_int32 * 2)(1, 1)

        def call(assets_, fps_=fps, ds_=ds, k=2, opt=None, ctx_=ctx.handle, rt_=im):
            o = opt or N.GsRenderOptions()
            arr = (C.c_void_p * len(assets_))(*assets_) if assets_ is not None else None
            return lib.gs_frame_objects(ctx_, k, arr, fps_, ds_, C.byref(o), C.byref(rt_) if rt_ is not None else None, None)

        good = [rs[0]._asset.value, rs[1]._asset.value]
        cases = {"null ctx": dict(ctx_=None), "null assets": dict(assets_=None), "null fps": dict(fps_=None),
                 "null do_sort": dict(ds_=None), "no objects": dict(k=0), "null asset": dict(assets_=[good[0], None]),
                 "listed twice": dict(assets_=[good[0], good[0]]), "other context": dict(assets_=[good[0], foreign._asset.value]),
                 "no images": dict(rt_=None)}
        small = (N.GsFrameParams * 2)(rs[0].frame_params(cam), rs[1].frame_params(camera(g, 150, 120)))
        cases["screen sizes differ"] = dict(fps_=small)
        for name, flags in (("load_rt", dict(flags=N.GS_FLAG_LOAD_RT)), ("partition", dict(partition_count=2, band_rows=1)),
                            ("rows", dict(row_begin=0, row_end=2)), ("band_packed", dict(band_packed=1))):
            o = N.GsRenderOptions()
            for key, v in flags.items():
                setattr(o, key, v)
            cases[name] = dict(opt=o)
        for name, kw in cases.items():
            kw.setdefault("assets_", good)
            assert call(**kw) == INVALID, name
        ctx.sync()
        assert (rt == 3).all()
        for r, o in zip(rs, orders):
            assert np.array_equal(r.readback_order(), o)
    finally:
        foreign.Dispose()
        other.close()
        for r in rs:
            r.Dispose()


# ---- 9. one object --------------------------------------------------------------------------------------------------------
def test_one_object_is_gs_frame(g, ctx, ca):
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 12000, 0x5EED0F70, "Medium")
    tw = Twins(g, ctx, [asset], lambda i, r: None)
    try:
        cam = orbit(g, 2)
        W, H = cam.pixelWidth, cam.pixelHeight
        a, b = np.zeros((H, W, 4), np.float16), np.zeros((H, W, 4), np.float16)
        n0 = ctx.stage_times().kernel_launches
        loop_frame(g, ctx, tw.loop, cam, 0, a, None)
        n1 = ctx.stage_times().kernel_launches
        call_frame(g, ctx, tw.call, cam, 0, b, None)
        n2 = ctx.stage_times().kernel_launches
        assert a.any() and np.array_equal(a.view(np.uint16), b.view(np.uint16))
        assert n2 - n1 == n1 - n0
        tw.check_state()
    finally:
        tw.dispose()


# ---- 10. the Unity render-thread event -----------------------------------------------------------------------------------
def test_unity_frame_objects_event_equals_a_direct_call(g, ctx):
    from unitygaussiansplatting_b200 import _native as N
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, 7000, 0x5EED0F80 + i, "Medium") for i in range(3)]
    tw = Twins(g, ctx, assets, lambda i, r: setattr(r, "localToWorldMatrix", g.trs(position=(1.0 * i - 1.0, 0, 0.4 * i)).astype(np.float32)))
    try:
        cam = orbit(g, 1)
        W, H = cam.pixelWidth, cam.pixelHeight
        direct = np.zeros((H, W, 4), np.float16)
        call_frame(g, ctx, tw.loop, cam, 0, direct, None)
        k = len(tw.call)
        assets_arr, fps, ds, keep = frame_args(g, [(cam, r, r.sceneDepth) for r in tw.call], sort=next_sort)
        via = np.zeros_like(direct)
        ev = N.GsUnityFrameObjectsEvent()
        ev.ctx, ev.object_count = C.cast(ctx.handle, C.c_void_p).value, k
        ev.assets, ev.fps, ev.do_sort = C.addressof(assets_arr), C.addressof(fps), C.addressof(ds)
        ev.options.blend_mode = 0
        ev.status, ev.has_rt, ev.has_camera_target = -5, 1, 0
        ev.rt.data, ev.rt.width, ev.rt.height, ev.rt.format, ev.rt.memory = via.ctypes.data, W, H, 0, 0
        fn = N.native().gs_unity_get_render_event_func()
        fn(N.GS_UNITY_EVENT_FRAME_OBJECTS, C.addressof(ev))
        assert ev.status == 0
        ctx.sync()
        assert direct.any() and np.array_equal(via.view(np.uint16), direct.view(np.uint16))
        tw.check_state()
        ev.object_count = 0
        fn(N.GS_UNITY_EVENT_FRAME_OBJECTS, C.addressof(ev))
        assert ev.status == INVALID
    finally:
        tw.dispose()
