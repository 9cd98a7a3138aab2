"""Screens up to 16384 x 16384 px, the largest render texture D3D12 makes: parity with the oracle bit for bit at the edges of
the bin-rectangle format (8-bit indices of 64-pixel bins), the two-pass 8-bit bin sort, the bin list growing on screens above
8160 px, the render and camera target kinds, several objects and groups, and the refusal above 16384.

Host memory: the oracle's float image of a 16384 x 16384 frame is 4 GiB; those tests need about 8 GiB free and say so when
it is not there."""
import numpy as np
import pytest

from util import camera, pixels_per_unit, splat_records, world_at_pixel

pytestmark = pytest.mark.gpu

GS_ERR_INVALID_ARGUMENT, GS_ERR_OUT_OF_MEMORY = -1, -3


def _need_host_gib(gib):
    try:
        with open("/proc/meminfo") as f:
            have = next(int(line.split()[1]) for line in f if line.startswith("MemAvailable:")) / 2**20
    except (OSError, StopIteration):
        return
    if have < gib:
        pytest.skip("needs %.0f GiB of free host memory, %.1f GiB available" % (gib, have))


def _grid_pairs():
    """Bin-list entries one pass of the persistent sort grid covers with one 8192-pair tile per CTA (2 CTAs per SM)."""
    import torch
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count * 8192


def _edge_scene(g, cam, n_base=20000, entries=0, seed=0x5EED0E00):
    """A small clustered scene, small splats along the last bin column and the last bin row (their footprints reach the last
    pixel column / row) and one in the bottom-right bin; with `entries`, wide flat splats across the screen on the bin-row
    boundaries (2 x binsX entries each) as many as give about that many entries."""
    W, H = cam.pixelWidth, cam.pixelHeight
    parts = [g.generate_input_splats(g.SCENE_CLUSTERED, n_base, seed)]
    t = np.linspace(0.04, 0.96, 9)
    xs = np.r_[np.full(9, W - 3.5), t * W, W - 20.5]
    ys = np.r_[t * H, np.full(9, H - 3.5), H - 18.3]
    depth = 6.0
    parts.append(splat_records(world_at_pixel(cam, xs, ys, depth), np.array([3.0, 2.0, 2.5]) / pixels_per_unit(cam, depth), 0.9,
                               (0.2, 0.9, 0.4)))
    if entries:
        parts.append(_flat_splats(cam, -(-entries // (2 * -(-W // 64))), W * H))
    return g.create_asset(np.ascontiguousarray(np.concatenate(parts)), "Medium")


def _flat_splats(cam, n, seed):
    """n splats as wide as the screen and about a pixel tall, centred on the boundaries between bin rows: each touches every
    bin of two bin rows."""
    W, H = cam.pixelWidth, cam.pixelHeight
    rng = np.random.default_rng(seed)
    depth = 5.0 + 3.0 * rng.random(n)
    cy = 64.0 * (1 + np.arange(n) % (-(-H // 64) - 1))
    scale = np.array([0.3 * W, 0.01, 0.01]) / pixels_per_unit(cam, depth)[:, None]
    return splat_records(world_at_pixel(cam, W / 2, cy, depth), scale, 0.1 + 0.3 * rng.random(n), rng.random((n, 3)))


def _equal_rows(got, want, rows=1024):
    """got (any float dtype) == want (float32), compared in bands of rows so that no 4 GiB temporaries are made."""
    return all(np.array_equal(got[y:y + rows].astype(np.float32), want[y:y + rows]) for y in range(0, got.shape[0], rows))


def _drawn_in_last_bins(rt, W, H):
    x0, y0 = (-(-W // 64) - 1) * 64, (-(-H // 64) - 1) * 64
    return rt[:, x0:, 3].max() > 0 and rt[y0:, :, 3].max() > 0 and rt[y0:, x0:, 3].max() > 0


# (width, height), bins, whether the scene gets enough entries that the persistent sort's CTAs take several tiles
SIZES = [
    ((8192, 4096), 8192, False),
    ((16384, 512), 2048, False),        # 256 bins across: bin x index 255
    ((512, 16384), 2048, False),
    ((16383, 577), 2560, False),        # partial last bin column (63 px) and last bin row (1 px)
    ((7232, 9280), 16385, True),        # 113 x 145: the first screen sorted in two 8-bit passes
    ((16384, 16384), 65536, True),      # the largest screen: bin (255, 255) included; RGBA16F only (4 GiB oracle image)
]


@pytest.mark.parametrize("size,bins,many", SIZES, ids=["%dx%d" % s[0] for s in SIZES])
def test_large_screen_frame_matches_oracle(g, O, ctx, size, bins, many):
    """Sorted keys and order, view data and the fp16-ROP render target equal the oracle's bit for bit, with splats drawn in
    the last bin column and the last bin row."""
    W, H = size
    assert -(-W // 64) * -(-H // 64) == bins
    if W * H > 8192 * 8192:
        _need_host_gib(8)
    cam = camera(g, W, H)
    asset = _edge_scene(g, cam, entries=7 * _grid_pairs() // 5 if many else 0)
    r = g.GaussianSplatRenderer(asset, ctx)
    rt = np.zeros((H, W, 4), np.float16)
    r.SortAndRenderSplats(cam, rt=rt)
    st = ctx.stage_times()
    if many:
        assert st.tile_entries > _grid_pairs(), "%d entries: one tile per CTA" % st.tile_entries
    fp, _keep = g.make_frame_params(cam)
    ref = O.frame(asset, fp, threads=O.max_threads())
    assert np.array_equal(r.readback_keys(), ref["keys"]), "sorted keys differ at %dx%d" % size
    assert np.array_equal(r.readback_order(), ref["order"]), "sorted splat indices differ at %dx%d" % size
    assert _drawn_in_last_bins(ref["rt"], W, H), "nothing draws in the last bin column / row"
    assert _equal_rows(rt, ref["rt"]), "render target differs at %dx%d" % size
    del rt, ref
    r.CalcViewData(cam)
    assert np.array_equal(r.readback_view(), O.calc_view(asset, fp, O.max_threads())), "SplatViewData differs at %dx%d" % size
    r.Dispose()


@pytest.mark.parametrize("blend", [0, 1], ids=["fp16rop", "fp32"])
@pytest.mark.parametrize("dtype", [np.float16, np.float32], ids=["rgba16f", "rgba32f"])
def test_wide_screen_blend_modes_and_formats(g, O, ctx, blend, dtype):
    W, H = 16384, 512
    cam = camera(g, W, H)
    asset = _edge_scene(g, cam)
    r = g.GaussianSplatRenderer(asset, ctx)
    r.blend_mode = blend
    rt = np.zeros((H, W, 4), dtype)
    r.SortAndRenderSplats(cam, rt=rt)
    fp, _keep = g.make_frame_params(cam)
    ref = O.frame(asset, fp, blend_mode=blend, threads=O.max_threads())["rt"]
    if dtype == np.float16 and blend == 1:
        ref = ref.astype(np.float16).astype(np.float32)   # blended in float, stored once as half
    assert ref[..., 3].max() > 0 and np.array_equal(rt.astype(np.float32), ref)
    r.Dispose()


def test_wide_screen_target_kinds_and_composite(g, O, ctx):
    """Host, device and CUDA-array render targets hold the oracle's frame; gs_composite of it onto host and CUDA-array camera
    targets leaves what the oracle's composite does."""
    import torch
    from images import Cudart
    W, H = 16384, 512
    cam = camera(g, W, H)
    asset = _edge_scene(g, cam)
    fp, _keep = g.make_frame_params(cam)
    ref = O.frame(asset, fp, threads=O.max_threads())["rt"]
    cu = Cudart()
    try:
        host = np.zeros((H, W, 4), np.float16)
        dev = torch.zeros((H, W, 4), dtype=torch.float16, device="cuda")
        torch.cuda.synchronize()   # filled on torch's stream: before the context's stream draws into it
        arr = g.CudaArrayImage(cu.array(W, H), W, H)
        got = {}
        for name, target in (("host", host), ("device", dev), ("array", arr)):
            r = g.GaussianSplatRenderer(asset, ctx)   # a fresh draw order each time: every frame sorts from the identity
            r.SortAndRenderSplats(cam, rt=target)
            ctx.sync()
            torch.cuda.synchronize()
            got[name] = host if name == "host" else dev.cpu().numpy() if name == "device" else cu.download(arr.handle)
            assert np.array_equal(got[name].astype(np.float32), ref), "%s render target differs from the oracle" % name
            r.Dispose()
        init = np.random.default_rng(11).random((H, W, 4)).astype(np.float16)
        want = O.composite(ref, init.astype(np.float32), target_fp16=True)
        comp = g.GaussianSplatRenderer(asset, ctx)
        host_t = init.copy()
        comp.Composite(host, host_t)
        arr_t = g.CudaArrayImage(cu.array(W, H), W, H)
        cu.upload(arr_t.handle, init)
        comp.Composite(dev, arr_t)
        ctx.sync()
        for name, t in (("host", host_t), ("array", cu.download(arr_t.handle))):
            assert not np.array_equal(t, init) and np.array_equal(t.astype(np.float32), want), "%s camera target differs" % name
        comp.Dispose()
    finally:
        ctx.sync()
        cu.free_all()


@pytest.mark.parametrize("edge,last_bin", [(16384, 255), (16320, 254)])
def test_splat_inside_the_last_bin_is_drawn(g, O, ctx, edge, last_bin):
    """A splat whose whole footprint lies in the bottom-right bin: at 16384 px that bin is (255, 255), whose one-bin rectangle
    packs to all ones, so the empty-rectangle sentinel must differ from it; 16320 px (last bin 254) is the control."""
    import torch
    _need_host_gib(5)
    W = H = edge
    cam = camera(g, W, H)
    c = last_bin * 64 + 32.0
    depth = 6.0
    asset = g.create_asset(splat_records(world_at_pixel(cam, [c], [c], depth), np.array([4.0, 3.0, 3.5]) / pixels_per_unit(cam, depth),
                                         0.9), "VeryHigh")
    r = g.GaussianSplatRenderer(asset, ctx)
    rt = torch.zeros((H, W, 4), dtype=torch.float16, device="cuda")
    # the zero fill runs on torch's stream and the frame on the context's own: the fill must land first (the splat's bin is
    # the last thing a 2 GiB fill writes, and the frame reaches it in well under a millisecond)
    torch.cuda.synchronize()
    r.SortAndRenderSplats(cam, rt=rt)
    ctx.sync()
    torch.cuda.synchronize()
    b0 = last_bin * 64
    assert rt[:b0].abs().max().item() == 0 and rt[:, :b0].abs().max().item() == 0, "the footprint must lie in the last bin"
    corner = rt[b0:, b0:].cpu().numpy()
    del rt
    torch.cuda.empty_cache()
    fp, _keep = g.make_frame_params(cam)
    ref = O.frame(asset, fp, threads=O.max_threads())["rt"]
    assert not ref[:b0].any() and not ref[:, :b0].any()
    assert ref[b0:, b0:, 3].max() > 0.5 and np.array_equal(corner.astype(np.float32), ref[b0:, b0:]), "the splat in bin %d is not drawn" % last_bin
    r.Dispose()


def test_bin_list_grows_on_a_large_screen(g, O, ctx):
    """Wide flat splats make far more than 8 entries per splat at 16384 x 4096, and more than the list's 4 Mi minimum: the frame
    still renders bit for bit, with every entry listed, and the same frame again bins once (the list has grown)."""
    ctx = g.GaussianSplatContext(0)   # a fresh context (not the session's): its bin list starts at the capacity rule's size
    W, H = 16384, 4096
    cam = camera(g, W, H)
    n = 12000
    asset = g.create_asset(np.ascontiguousarray(_flat_splats(cam, n, 7)), "Medium")
    r = g.GaussianSplatRenderer(asset, ctx)
    rt = np.zeros((H, W, 4), np.float16)
    before = ctx.stage_times().kernel_launches
    r.SortAndRenderSplats(cam, rt=rt)   # a host target: a truncated list would raise here
    st1 = ctx.stage_times()
    assert st1.tile_entries > max(8 * n, 4 << 20), "%d entries do not overflow the list's first size" % st1.tile_entries
    fp, _keep = g.make_frame_params(cam)
    ref = O.frame(asset, fp, threads=O.max_threads())
    assert np.array_equal(r.readback_order(), ref["order"])
    assert np.array_equal(rt.astype(np.float32), ref["rt"]), "the frame whose list grew differs from the oracle"
    first = st1.kernel_launches - before
    rt2 = np.zeros_like(rt)
    r.SortAndRenderSplats(cam, rt=rt2)
    st2 = ctx.stage_times()
    again = st2.kernel_launches - st1.kernel_launches
    assert st2.tile_entries == st1.tile_entries and np.array_equal(rt2, rt)
    assert first - again == 4, "the growing frame bins once more (bin_emit, look-back clear, two sort passes): %d vs %d" % (first, again)
    r.Dispose()
    ctx.close()


def test_bin_list_above_its_largest_size_reports_out_of_memory(g, O, ctx):
    """About 13,000 splats each covering all 65,536 bins of a 16384 x 16384 screen need ~852 M entries, more than 768 Mi: the
    frame reports GS_ERR_OUT_OF_MEMORY at gs_sync, and the next normal-sized frame on the same context is correct."""
    import torch
    from unitygaussiansplatting_b200._native import GsError
    ctx = g.GaussianSplatContext(0)   # a fresh context (not the session's), whose next frame is checked
    W = H = 16384
    cam = camera(g, W, H)
    n = 13000
    rng = np.random.default_rng(5)
    depth = 6.0 + rng.random(n)
    big = splat_records(world_at_pixel(cam, W / 2, H / 2, depth), np.full((n, 3), 1.2 * W) / pixels_per_unit(cam, depth)[:, None], 0.9,
                        rng.random((n, 3)))
    r = g.GaussianSplatRenderer(g.create_asset(big, "Medium"), ctx)
    rt = torch.zeros((H, W, 4), dtype=torch.float16, device="cuda")
    r.SortAndRenderSplats(cam, rt=rt)
    with pytest.raises(GsError) as e:
        ctx.sync()
    assert e.value.code == GS_ERR_OUT_OF_MEMORY
    r.Dispose()
    del rt
    torch.cuda.empty_cache()
    small = camera(g, 320, 200)
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0002, "Medium")
    r = g.GaussianSplatRenderer(asset, ctx)
    rt = np.zeros((200, 320, 4), np.float16)
    r.SortAndRenderSplats(small, rt=rt)
    ctx.sync()
    fp, _keep = g.make_frame_params(small)
    ref = O.frame(asset, fp, threads=O.max_threads())
    assert ref["rt"][..., 3].max() > 0 and np.array_equal(rt.astype(np.float32), ref["rt"])
    r.Dispose()
    ctx.close()


def _objects(g, cam):
    """Three objects of one camera; the first carries enough wide flat splats that a 16384 x 2048 list of all three grows."""
    a = _edge_scene(g, cam, n_base=15000, entries=5_200_000, seed=0x5EED0E01)
    b = g.synthetic_asset(g.SCENE_CLUSTERED, 12000, 0x5EED0E02, "VeryHigh")
    c = g.synthetic_asset(g.SCENE_CLUSTERED, 6000, 0x5EED0E03, "Medium")
    knobs = [dict(),
             dict(localToWorldMatrix=g.trs(position=(0.6, 0.1, 1.5)).astype(np.float32), m_RenderOrder=1),
             dict(localToWorldMatrix=g.trs(position=(-0.5, -0.3, 2.5)).astype(np.float32))]
    return [a, b, c], knobs


def _renderers(g, ctx, assets, knobs):
    rs = []
    for asset, kn in zip(assets, knobs):
        r = g.GaussianSplatRenderer(asset, ctx)
        for k, v in kn.items():
            setattr(r, k, v)
        rs.append(r)
    return rs


def test_frame_objects_on_a_large_screen(g, ctx):
    """gs_frame_objects with three objects at 16384 x 2048 equals gs_frame per object (GS_FLAG_LOAD_RT from the second) plus
    gs_composite, bit for bit: render target, camera target and every object's draw order."""
    from unitygaussiansplatting_b200.renderer import GatherSplatsForCamera
    W, H = 16384, 2048
    cam = camera(g, W, H)
    assets, knobs = _objects(g, cam)
    init = np.random.default_rng(4).random((H, W, 4)).astype(np.float16)
    one = _renderers(g, ctx, assets, knobs)
    rt1, tgt1 = np.zeros((H, W, 4), np.float16), init.copy()
    g.SortAndRenderSplatsMulti(one, cam, rt1, tgt1)   # host images: a truncated list would raise here
    assert ctx.stage_times().tile_entries > 4 << 20, "the run's list must outgrow the capacity rule's 4 Mi"
    each = _renderers(g, ctx, assets, knobs)
    rt2, tgt2 = np.zeros((H, W, 4), np.float16), init.copy()
    for i, r in enumerate(GatherSplatsForCamera(each, cam)):
        r.load_rt = i > 0
        r.SortAndRenderSplats(cam, rt=rt2)
    each[0].Composite(rt2, tgt2)
    assert rt1[..., 3].max() > 0 and np.array_equal(rt1.view(np.uint16), rt2.view(np.uint16)), "render targets differ"
    assert np.array_equal(tgt1.view(np.uint16), tgt2.view(np.uint16)), "camera targets differ"
    for a, b in zip(one, each):
        assert np.array_equal(a.readback_order(), b.readback_order())
    for r in one + each:
        r.Dispose()


@pytest.mark.parametrize("gpus", [2, 3])
def test_emulated_group_on_a_large_screen(g, ctx, gpus):
    """Emulated groups of 2 and 3 at 16384 x 2048 leave the render target and the camera target one GPU leaves."""
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    W, H = 16384, 2048
    cam = camera(g, W, H)
    assets, knobs = _objects(g, cam)
    init = np.random.default_rng(6).random((H, W, 4)).astype(np.float16)
    one = _renderers(g, ctx, assets, knobs)
    want_rt, want_tgt = np.zeros((H, W, 4), np.float16), init.copy()
    g.SortAndRenderSplatsMulti(one, cam, want_rt, want_tgt)
    grp = GaussianSplatGroup.create(assets[0], [0] * gpus, emulate=True)
    try:
        objs = [grp] + [grp.add_object(a) for a in assets[1:]]
        for o, kn in zip(objs, knobs):
            for k, v in kn.items():
                setattr(o, k, v)
        rts = [np.zeros((H, W, 4), np.float16) for _ in range(gpus)]
        tgts = [init.copy() for _ in range(gpus)]
        grp.SortAndRenderSplatsMulti(objs, cam, rts=rts, camera_targets=tgts)
        grp.sync()
        for i in range(gpus):
            assert np.array_equal(rts[i].view(np.uint16), want_rt.view(np.uint16)), "member %d: render target differs" % i
            assert np.array_equal(tgts[i].view(np.uint16), want_tgt.view(np.uint16)), "member %d: camera target differs" % i
            for k, o in enumerate(objs):
                assert np.array_equal(o.readback_order(i), one[k].readback_order()), "member %d object %d: draw order" % (i, k)
    finally:
        grp.close()
        for r in one:
            r.Dispose()


@pytest.mark.parametrize("size", [(16385, 64), (64, 16385)], ids=["wide", "tall"])
def test_screens_above_16384_are_refused(g, ctx, size):
    """16385 px on either axis: GS_ERR_INVALID_ARGUMENT from every entry point, with nothing enqueued or written."""
    import torch
    from unitygaussiansplatting_b200._native import GsError
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    W, H = size
    cam = camera(g, W, H)
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 4000, 0x5EED0E04, "Medium")
    r = g.GaussianSplatRenderer(asset, ctx)
    r2 = g.GaussianSplatRenderer(asset, ctx)
    rt = np.full((H, W, 4), 0.5, np.float16)
    dev = torch.full((H, W, 4), 0.5, dtype=torch.float16, device="cuda")
    before = ctx.stage_times().kernel_launches
    calls = [lambda: r.SortAndRenderSplats(cam, rt=rt), lambda: r.SortAndRenderSplats(cam, rt=dev, camera_target=rt),
             lambda: r.CalcViewData(cam), lambda: r.SortPoints(cam), lambda: g.SortAndRenderSplatsMulti([r, r2], cam, rt)]
    for call in calls:
        with pytest.raises(GsError) as e:
            call()
        assert e.value.code == GS_ERR_INVALID_ARGUMENT and "16384" in str(e.value)
    ctx.sync()
    assert ctx.stage_times().kernel_launches == before, "a refused call launched kernels"
    assert (rt == 0.5).all() and bool((dev == 0.5).all().item()), "a refused call wrote an image"
    grp = GaussianSplatGroup.create(asset, [0, 0], emulate=True)
    try:
        rts = [np.full((H, W, 4), 0.5, np.float16) for _ in range(2)]
        with pytest.raises(GsError) as e:
            grp.SortAndRenderSplatsMulti([grp], cam, rts=rts)
        assert e.value.code == GS_ERR_INVALID_ARGUMENT
        grp.sync()
        assert all((x == 0.5).all() for x in rts)
    finally:
        grp.close()
    r.Dispose()
    r2.Dispose()
