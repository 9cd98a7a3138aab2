"""Several splat objects per camera on a group (gs_group_frame_objects, GaussianSplatGroup.SortAndRenderSplatsMulti) against one
GPU drawing the same objects with SortAndRenderSplatsMulti (and gs_composite): every member's render target, camera target and
every object's draw order must be BIT-identical, frame after frame, while the camera flies through the scene and the objects'
draw order swaps.  Groups are emulated (GS_GROUP_EMULATE) so everything runs on one GPU; the real-device variant needs >= 2."""
import ctypes as C

import numpy as np
import pytest

from util import CAP_H, CAP_SPLATS, CAP_W, bin_row_splats, camera

pytestmark = pytest.mark.gpu


def _cams(g, w, h, k=5):
    # a fly-through that turns from right to left of the two front objects: their camera depths cross between frames 1 and 2
    heads = np.linspace(-0.16, 0.17, k)
    return [camera(g, w, h, pos=(0.1 * i - 0.2, 0.45 + 0.03 * i, -6.0 + 0.3 * i), forward=(np.sin(a), -0.02, np.cos(a)))
            for i, a in enumerate(heads)]


def _bits(n, every, seed):
    rng = np.random.default_rng(seed)
    bits = np.zeros((n + 31) // 32, np.uint32)
    ids = np.nonzero(rng.random(n) < 1.0 / every)[0]
    np.bitwise_or.at(bits, ids >> 5, np.uint32(1) << (ids & 31).astype(np.uint32))
    return bits


def _scene(g, w, h):
    """Three overlapping objects: clustered Medium (cutout + deleted bits), VeryHigh under a sheared, mirrored transform
    (selected bits + a scene depth buffer), VeryLow (Cluster4k SH + BC7 colour); every object its own m_RenderOrder and
    m_SortNthFrame."""
    a = g.synthetic_asset(g.SCENE_CLUSTERED, 60000, 0x5EED00A1, "Medium")
    b = g.synthetic_asset(g.SCENE_CLUSTERED, 40000, 0x5EED00A2, "VeryHigh")
    c = g.synthetic_asset(g.SCENE_CLUSTERED, 9000, 0x5EED00A3, "VeryLow")
    assert c.splatCount > 4096
    la = g.trs(position=(-0.7, 0.0, 1.5)).astype(np.float32)
    shear = np.eye(4)
    shear[0, 1], shear[2, 0] = 0.35, -0.2
    lb = (g.trs(position=(0.7, 0.15, 1.5)) @ shear @ np.diag([-0.8, 0.8, 0.8, 1.0])).astype(np.float32)
    lc = g.trs(position=(0.0, -0.4, 2.5), scale=(0.9, 0.9, 0.9)).astype(np.float32)
    ramp = np.broadcast_to(np.linspace(0.0, 0.08, w, dtype=np.float32), (h, w)).copy()
    knobs = [
        dict(localToWorldMatrix=la, m_RenderOrder=0, m_SortNthFrame=1, m_SplatScale=1.1,
             m_Cutouts=[(np.linalg.inv(g.trs(scale=(1.6, 1.6, 1.6))) @ la, 0)], m_DeletedBits=_bits(a.splatCount, 9, 1)),
        dict(localToWorldMatrix=lb, m_RenderOrder=0, m_SortNthFrame=2, m_OpacityScale=0.9, m_SHOrder=2,
             m_SelectedBits=_bits(b.splatCount, 11, 2), sceneDepth=ramp),
        dict(localToWorldMatrix=lc, m_RenderOrder=-1, m_SortNthFrame=3),
    ]
    return [a, b, c], knobs


def _single(g, ctx, assets, knobs, cams, fmt=np.float16, blend=None):
    rs = []
    for asset, kn in zip(assets, knobs):
        r = g.GaussianSplatRenderer(asset, ctx)
        for k, v in kn.items():
            setattr(r, k, v)
        if blend is not None:
            r.blend_mode = blend
        rs.append(r)
    frames = []
    for cam in cams:
        rt = np.zeros((cam.pixelHeight, cam.pixelWidth, 4), fmt)
        active = g.SortAndRenderSplatsMulti(rs, cam, rt)
        frames.append(([rs.index(r) for r in active], [r.readback_order() for r in rs], rt))
    for r in rs:
        r.Dispose()
    return frames


def _group(assets, knobs, gpus, blend=None):
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    grp = GaussianSplatGroup.create(assets[0], [0] * gpus, emulate=True) if isinstance(gpus, int) else GaussianSplatGroup.create(assets[0], gpus)
    objs = [grp] + [grp.add_object(a) for a in assets[1:]]
    for o, kn in zip(objs, knobs):
        for k, v in kn.items():
            setattr(o, k, v)
    if blend is not None:
        grp.blend_mode = blend
    return grp, objs


def _run_and_check(grp, objs, cams, want, make_rts, read_rt):
    swapped = set()
    for f, cam in enumerate(cams):
        rts = make_rts(cam)
        active = grp.SortAndRenderSplatsMulti(objs, cam, rts=rts)
        grp.sync()
        assert [objs.index(o) for o in active] == want[f][0], "frame %d: draw order of the objects differs" % f
        swapped.add(tuple(want[f][0]))
        for i in range(grp.local_count):
            got = read_rt(rts, i)
            assert got.any()
            assert np.array_equal(got.view(np.uint16), want[f][2].view(np.uint16)), "frame %d member %d: render target differs" % (f, i)
            for k, o in enumerate(objs):
                assert np.array_equal(o.readback_order(i), want[f][1][k]), "frame %d member %d object %d: draw order differs" % (f, i, k)
    return swapped


@pytest.mark.parametrize("gpus", [1, 2, 3, 4, 8])
def test_objects_equal_single_gpu(g, ctx, gpus):
    cams = _cams(g, 400, 256)
    assets, knobs = _scene(g, 400, 256)
    want = _single(g, ctx, assets, knobs, cams)
    grp, objs = _group(assets, knobs, gpus)
    swapped = _run_and_check(grp, objs, cams, want, lambda cam: [np.zeros((cam.pixelHeight, cam.pixelWidth, 4), np.float16) for _ in range(gpus)],
                             lambda rts, i: rts[i])
    assert len(swapped) == 2, "the fly-through must swap the objects' draw order"
    st = grp.stats()
    assert sum(st.slab_counts[:gpus]) > 0 and st.row_bounds[gpus] == (256 + 15) // 16
    grp.close()


def test_objects_overlap_on_screen(g, ctx):
    """The scene is a real multi-object test: the front objects cover common pixels, so each blends under another."""
    cam = _cams(g, 400, 256)[0]
    assets, knobs = _scene(g, 400, 256)
    cover = []
    for asset, kn in zip(assets, knobs):
        r = g.GaussianSplatRenderer(asset, ctx)
        for k, v in kn.items():
            setattr(r, k, v)
        rt = np.zeros((256, 400, 4), np.float16)
        r.SortAndRenderSplats(cam, rt=rt)
        cover.append(rt[..., 3] > 0.05)
        r.Dispose()
    assert (cover[0] & cover[1]).sum() > 500 and (cover[2] & (cover[0] | cover[1])).sum() > 500


def test_objects_rgba32f_fp32_blend(g, ctx):
    from unitygaussiansplatting_b200 import _native as N
    cams = _cams(g, 320, 200, 3)
    assets, knobs = _scene(g, 320, 200)
    want = _single(g, ctx, assets, knobs, cams, np.float32, N.GS_BLEND_FP32)
    grp, objs = _group(assets, knobs, 3, N.GS_BLEND_FP32)
    _run_and_check(grp, objs, cams, want, lambda cam: [np.zeros((cam.pixelHeight, cam.pixelWidth, 4), np.float32) for _ in range(3)],
                   lambda rts, i: rts[i])
    grp.close()


def test_objects_more_members_than_rows(g, ctx):
    """96 x 40: three 16-pixel rows for eight members."""
    cams = [camera(g, 96, 40, pos=(0.1 * i, 0.4, -6.0), forward=(0.05 * (i - 2), 0.0, 1.0)) for i in range(4)]
    assets, knobs = _scene(g, 96, 40)
    want = _single(g, ctx, assets, knobs, cams)
    grp, objs = _group(assets, knobs, 8)
    _run_and_check(grp, objs, cams, want, lambda cam: [np.zeros((40, 96, 4), np.float16) for _ in range(8)], lambda rts, i: rts[i])
    grp.close()


def test_objects_device_array_and_async_host_images(g, ctx):
    """Member images of every kind in one group: a device tensor, a CUDA array, and pinned host images filled asynchronously
    (GS_FLAG_ASYNC_READBACK, two in rotation, completed by sync())."""
    import torch
    from images import Cudart
    cams = _cams(g, 320, 200, 4)
    assets, knobs = _scene(g, 320, 200)
    want = _single(g, ctx, assets, knobs, cams)
    grp, objs = _group(assets, knobs, 3)
    grp.async_readback = True
    rt = Cudart()
    from unitygaussiansplatting_b200.renderer import CudaArrayImage
    arr = CudaArrayImage(rt.array(320, 200), 320, 200)
    dev = torch.zeros((200, 320, 4), dtype=torch.float16, device="cuda")
    pins = [torch.zeros((200, 320, 4), dtype=torch.float16).pin_memory() for _ in range(2)]
    try:
        for f, cam in enumerate(cams):
            grp.SortAndRenderSplatsMulti(objs, cam, rts=[dev, arr, pins[f & 1].numpy()])
            grp.sync()
            torch.cuda.synchronize()
            for got in (dev.cpu().numpy(), rt.download(arr.handle), pins[f & 1].numpy()):
                assert np.array_equal(got.view(np.uint16), want[f][2].view(np.uint16)), "frame %d" % f
    finally:
        grp.close()
        rt.free_all()


def test_objects_camera_targets(g, ctx):
    """Members with a camera target end with the bytes single-GPU gs_composite leaves on the same initial target (device,
    CUDA array and host targets); a member without one, and every member's render target, is as without targets."""
    import torch
    from images import Cudart
    from unitygaussiansplatting_b200.renderer import CudaArrayImage
    W, H = 320, 200
    cams = _cams(g, W, H, 3)
    assets, knobs = _scene(g, W, H)
    want = _single(g, ctx, assets, knobs, cams)
    rng = np.random.default_rng(9)
    grp, objs = _group(assets, knobs, 4)
    cu = Cudart()
    comp = g.GaussianSplatRenderer(assets[2], ctx)   # gs_composite on one GPU, through a renderer's context
    try:
        for f, cam in enumerate(cams):
            init = rng.random((H, W, 4)).astype(np.float16)
            expect = torch.from_numpy(init.copy()).cuda()
            comp.Composite(torch.from_numpy(want[f][2]).cuda(), expect)
            ctx.sync()
            expect = expect.cpu().numpy()
            assert not np.array_equal(expect, init)
            dev_t = torch.from_numpy(init.copy()).cuda()
            arr_t = CudaArrayImage(cu.array(W, H), W, H)
            cu.upload(arr_t.handle, init)
            host_t = init.copy()
            rts = [np.zeros((H, W, 4), np.float16) for _ in range(4)]
            grp.SortAndRenderSplatsMulti(objs, cam, rts=rts, camera_targets=[dev_t, None, arr_t, host_t])
            grp.sync()
            torch.cuda.synchronize()
            for i in range(4):
                assert np.array_equal(rts[i].view(np.uint16), want[f][2].view(np.uint16)), "frame %d member %d: render target" % (f, i)
            for name, got in (("device", dev_t.cpu().numpy()), ("array", cu.download(arr_t.handle)), ("host", host_t)):
                assert np.array_equal(got.view(np.uint16), expect.view(np.uint16)), "frame %d: %s camera target differs from gs_composite" % (f, name)
    finally:
        comp.Dispose()
        grp.close()
        cu.free_all()


def test_objects_rejections_write_nothing(g, ctx):
    """Every invalid call returns its status and leaves render targets, camera targets and draw orders byte-unchanged."""
    import torch
    from unitygaussiansplatting_b200 import _native as N
    W, H = 256, 160
    cam = _cams(g, W, H, 1)[0]
    assets, knobs = _scene(g, W, H)
    grp, objs = _group(assets[:2], knobs[:2], 2)
    other = grp.add_object(g.synthetic_asset(g.SCENE_CLUSTERED, 5000, 0x5EED00A4, "Medium"))   # a different splat count
    lib = N.native()
    rts = [torch.full((H, W, 4), 0.25, dtype=torch.float16, device="cuda"), np.full((H, W, 4), 0.5, np.float16)]
    cams = [torch.full((H, W, 4), 0.75, dtype=torch.float16, device="cuda"), None]
    before = [r.cpu().numpy().copy() if hasattr(r, "cpu") else r.copy() for r in rts + cams[:1]]
    orders = [o.readback_order(i) for o in objs for i in range(2)]

    def call(count=2, table=None, fps=None, flags=0, cam_img=None, rt_height=None):
        table = table if table is not None else [objs[0]._assets[0], objs[0]._assets[1], objs[1]._assets[0], objs[1]._assets[1]]
        arr = (C.c_void_p * len(table))(*table)
        if fps is None:
            fps = (N.GsFrameParams * 2)()
            fps[0], fps[1] = objs[0].frame_params(cam), objs[1].frame_params(cam)
        do_sort = (C.c_int32 * 2)(1, 1)
        opt = N.GsRenderOptions()
        opt.flags = flags
        keep = []
        rp = grp._images(rts, cam, keep)
        if rt_height is not None:
            rp[0].contents.height = rt_height
        cp = (C.POINTER(N.GsImage) * 2)()
        if cam_img is not None:
            keep.append(cam_img)
            cp[0] = C.pointer(cam_img)
        else:
            cp = grp._images(cams, cam, keep)
        return lib.gs_group_frame_objects(grp.handle, count, arr, fps, do_sort, C.byref(opt), rp, cp)

    from unitygaussiansplatting_b200.renderer import _image
    small = _image(torch.zeros((H // 2, W, 4), dtype=torch.float16, device="cuda"), W, H // 2)
    bad_fmt = _image(cams[0], W, H)
    bad_fmt.format = 7
    fps_size = (N.GsFrameParams * 2)()
    fps_size[0], fps_size[1] = objs[0].frame_params(cam), objs[1].frame_params(cam)
    fps_size[1].screen_w = W + 16
    a0, a1 = objs[0]._assets, objs[1]._assets
    cases = [
        ("object_count 0", dict(count=0), -1),
        ("null asset", dict(table=[a0[0], a0[1], a1[0], None]), -1),
        ("an asset listed twice", dict(table=[a0[0], a0[1], a0[0], a0[1]]), -1),
        ("different splat counts", dict(table=[a0[0], a0[1], a1[0], other._assets[1]]), -1),
        ("different screen sizes", dict(fps=fps_size), -1),
        ("GS_FLAG_LOAD_RT", dict(flags=N.GS_FLAG_LOAD_RT), -1),
        ("camera target of the wrong size", dict(cam_img=small), -1),
        ("render target of the wrong size", dict(rt_height=H - 16), -1),
        ("camera target of a bad format", dict(cam_img=bad_fmt), -4),
    ]
    for name, kw, status in cases:
        assert call(**kw) == status, name
        torch.cuda.synchronize()
        now = [r.cpu().numpy() if hasattr(r, "cpu") else r for r in rts + cams[:1]]
        for x, y in zip(before, now):
            assert np.array_equal(x.view(np.uint16), y.view(np.uint16)), "%s: an image was written" % name
        assert all(np.array_equal(o, o2) for o, o2 in zip(orders, [o.readback_order(i) for o in objs for i in range(2)])), "%s: an order moved" % name
    # and a valid call through the same helper does render
    assert call() == 0
    grp.sync()
    assert rts[1].any() and not np.array_equal(rts[1], before[1])
    grp.close()


def test_objects_real_devices(g, ctx):
    """gs_group_create over real devices (NCCL inside the library), the same comparison."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 CUDA devices")
    n = min(torch.cuda.device_count(), 4)
    cams = _cams(g, 400, 256)
    assets, knobs = _scene(g, 400, 256)
    want = _single(g, ctx, assets, knobs, cams)
    grp, objs = _group(assets, knobs, list(range(n)))
    _run_and_check(grp, objs, cams, want, lambda cam: [np.zeros((cam.pixelHeight, cam.pixelWidth, 4), np.float16) for _ in range(n)],
                   lambda rts, i: rts[i])
    grp.close()


def _bins(rt, edge=64):
    """64-pixel bins in which the image has any coverage"""
    h, w = rt.shape[:2]
    cov = rt[..., 3].astype(np.float32) > 0
    return np.add.reduceat(np.add.reduceat(cov, np.arange(0, h, edge), axis=0), np.arange(0, w, edge), axis=1) > 0


def test_objects_row_split_follows_the_summed_costs(g, ctx):
    """The row split of a call is gs_group_balance_rows of the row costs measured two calls earlier, and those are summed over
    the objects: on a group of one, the costs of a two-object call are the sum of each object's costs drawn alone (the objects
    cover disjoint 64-pixel bins, so neither changes the other's work); on a group of two, the bounds follow the summed costs,
    which split differently from the last-drawn object's alone."""
    from unitygaussiansplatting_b200.multigpu import balance_rows
    W, H = 400, 192
    rows = H // 16
    assets = [g.synthetic_asset(g.SCENE_LATTICE, 1000, 0x5EED00C1, "Medium"), g.synthetic_asset(g.SCENE_LATTICE, 1000, 0x5EED00C2, "Medium")]
    knobs = [dict(localToWorldMatrix=g.trs(position=(-2.2, 1.0, 0.0), scale=(0.6, 0.6, 0.6)).astype(np.float32)),
             dict(localToWorldMatrix=g.trs(position=(2.2, -1.0, 0.3), scale=(0.6, 0.6, 0.6)).astype(np.float32))]
    cam = camera(g, W, H, pos=(0.0, 0.0, -7.0))
    grp, objs = _group(assets, knobs, 1)
    alone, cover = [], []
    for o in objs:
        rt = np.zeros((H, W, 4), np.float16)
        assert grp.SortAndRenderSplatsMulti([o], cam, rts=[rt]) == [o]
        alone.append(grp.row_costs(rows))
        cover.append(_bins(rt))
    assert cover[0].any() and cover[1].any() and not (cover[0] & cover[1]).any()
    rt = np.zeros((H, W, 4), np.float16)
    assert grp.SortAndRenderSplatsMulti(objs, cam, rts=[rt]) == objs      # the second object is drawn last
    both = grp.row_costs(rows)
    assert np.array_equal(both, alone[0] + alone[1])
    grp.close()

    assert not np.array_equal(balance_rows(alone[0] + alone[1], 2), balance_rows(alone[1], 2))
    grp, objs = _group(assets, knobs, 2)
    costs = []
    for f in range(5):
        grp.SortAndRenderSplatsMulti(objs, cam)
        bounds = np.array(grp.stats().row_bounds[:3], np.uint32)
        if f >= 2:
            assert np.array_equal(bounds, balance_rows(costs[f - 2], 2)), "call %d" % f
            assert not np.array_equal(bounds, balance_rows(alone[1], 2)), "call %d: split on the last object's cost alone" % f
        costs.append(grp.row_costs(rows))
    grp.close()


def test_member_context_sync_with_a_pending_array_camera_target(g, ctx):
    """gs_sync on a member's own context right after the call, before gs_group_sync, waits for the composite onto a CUDA-array
    camera target (on the member's transfer stream) before it releases that target's surface; the target ends right."""
    import torch
    from images import Cudart
    from unitygaussiansplatting_b200.renderer import CudaArrayImage
    W, H = 320, 200
    cam = _cams(g, W, H, 1)[0]
    assets, knobs = _scene(g, W, H)
    want = _single(g, ctx, assets, knobs, [cam])[0][2]
    init = np.random.default_rng(11).random((H, W, 4)).astype(np.float16)
    expect = torch.from_numpy(init.copy()).cuda()
    comp = g.GaussianSplatRenderer(assets[2], ctx)
    comp.Composite(torch.from_numpy(want).cuda(), expect)
    ctx.sync()
    expect = expect.cpu().numpy()
    grp, objs = _group(assets, knobs, 2)
    cu = Cudart()
    try:
        targets = [CudaArrayImage(cu.array(W, H), W, H) for _ in range(2)]
        for t in targets:
            cu.upload(t.handle, init)
        grp.SortAndRenderSplatsMulti(objs, cam, camera_targets=targets)
        for c in grp.contexts:
            c.sync()
        grp.sync()
        torch.cuda.synchronize()
        for i, t in enumerate(targets):
            assert np.array_equal(cu.download(t.handle).view(np.uint16), expect.view(np.uint16)), "member %d" % i
    finally:
        comp.Dispose()
        grp.close()
        cu.free_all()


@pytest.mark.parametrize("image", ["host", "device"])
def test_truncated_list_of_an_earlier_object_is_reported(g, ctx, image):
    """A member draws the call's objects one after the other through one bin list.  On a fresh group (a 4 Mi entry list),
    object 0 is the construction of test_bin_list_exact_capacity_overflow_and_recovery, one splat over capacity, and object 1
    fits: the call still reports GS_ERR_OUT_OF_MEMORY, when it returns with a host image and at gs_group_sync with a device
    image.  Deleting the splat that no longer fits makes the next call succeed and equal the per-object gs_frame loop."""
    import torch
    from frame_loops import loop_frame
    W, H = CAP_W, CAP_H
    cam = camera(g, W, H)
    assets = [g.create_asset(bin_row_splats(cam, CAP_SPLATS + 1, 0xCA9), "VeryHigh"),
              g.create_asset(bin_row_splats(cam, 1000, 0xCAA), "VeryHigh")]
    grp, objs = _group(assets, [{}, {}], 1)
    rs = []
    try:
        def new_rt():
            return np.zeros((H, W, 4), np.float16) if image == "host" else torch.zeros((H, W, 4), dtype=torch.float16, device="cuda")

        rt = new_rt()
        if image == "host":
            with pytest.raises(g.GsError) as e:
                grp.SortAndRenderSplatsMulti(objs, cam, rts=[rt])
        else:
            assert grp.SortAndRenderSplatsMulti(objs, cam, rts=[rt]) == objs   # not checked when it is enqueued ...
            with pytest.raises(g.GsError) as e:
                grp.sync()                                                      # ... but at the next synchronising call
        assert e.value.code == -3 and "tile-list capacity exceeded" in str(e.value)

        last = int(grp.readback_order()[-1])
        bits = np.zeros((assets[0].splatCount + 31) // 32, np.uint32)
        bits[last >> 5] |= np.uint32(1 << (last & 31))
        objs[0].m_DeletedBits = bits
        rt = new_rt()
        assert grp.SortAndRenderSplatsMulti(objs, cam, rts=[rt]) == objs
        grp.sync()
        got = rt if image == "host" else rt.cpu().numpy()
        rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]
        rs[0].m_DeletedBits = bits
        want = np.zeros((H, W, 4), np.float16)
        loop_frame(g, ctx, rs, cam, 0, want, None)
        assert got.any() and np.array_equal(got.view(np.uint16), want.view(np.uint16))
        for o, r in zip(objs, rs):
            assert np.array_equal(o.readback_order(), r.readback_order())
    finally:
        for r in rs:
            r.Dispose()
        grp.close()


def test_python_multi_rejects_before_counting_and_draws_nothing_without_objects(g, ctx):
    """SortAndRenderSplatsMulti checks every object before any frame counter moves; with no objects it draws nothing."""
    W, H = 128, 96
    cam = _cams(g, W, H, 1)[0]
    assets, knobs = _scene(g, W, H)
    grp, objs = _group(assets[:2], knobs[:2], 2)
    other, other_objs = _group(assets[2:], knobs[2:], 1)
    before = [o.m_FrameCounter for o in objs]
    with pytest.raises(ValueError):
        grp.SortAndRenderSplatsMulti(objs + other_objs, cam)
    with pytest.raises(ValueError):
        grp.SortAndRenderSplatsMulti([objs[0], objs[1], objs[0]], cam)
    assert [o.m_FrameCounter for o in objs] == before
    rts = [np.full((H, W, 4), 0.5, np.float16) for _ in range(2)]
    assert grp.SortAndRenderSplatsMulti([], cam, rts=rts) == []
    grp.sync()
    assert all((r == np.float16(0.5)).all() for r in rts)
    assert [o.m_FrameCounter for o in objs] == before
    grp.close()
    other.close()
