"""gs_frame_cameras: several cameras, each with its own objects, drawn by one call on one GPU, against the camera loop it
stands for -- gs_frame_objects per camera.  Every comparison is bit for bit, on every render target, every camera target and
every asset's persistent draw order and sorted keys.  The loop and the call each own a copy of every asset, on one context;
an asset appears in several cameras, so its draw order chains from camera to camera."""
import numpy as np
import pytest

from frame_loops import CAM_SIZES, Twins, call_cameras, compare, g_trs, loop_cameras, mixed_assets, mixed_setup, orbit
from images import ca  # noqa: F401
from util import camera, splat_records

pytestmark = pytest.mark.gpu

INVALID, OOM = -1, -3
KINDS = ["host", "device", "array", None]


# ---- 1. equal to the loop -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ncam", [2, 3, 5])
@pytest.mark.parametrize("blend", [0, 1])
@pytest.mark.parametrize("dtype", [np.float16, np.float32])
def test_cameras_equal_the_loop(g, ctx, ca, ncam, blend, dtype):
    tw = Twins(g, ctx, mixed_assets(g, 5), mixed_setup)
    try:
        for f in range(3):
            cams = [orbit(g, f, *CAM_SIZES[c], phase=0.9 * c) for c in range(ncam)]
            subsets = [[(c + j) % 5 for j in range(2 + (c + f) % 3)] for c in range(ncam)]   # different lists per camera
            idx = tw.gathered(g, subsets, cams)
            rk = [KINDS[(f + c) % 4] for c in range(ncam)]
            tk = [KINDS[(f + c + 1) % 4] if rk[c] is not None else "device" for c in range(ncam)]
            assert compare(g, ctx, ca, tw, idx, cams, blend, dtype, rk, tk, "frame %d" % f) > 0
    finally:
        tw.dispose()


def test_python_mirror_matches_the_loop(g, ctx):
    """SortAndRenderCameras takes the one call; its twin draws camera by camera with SortAndRenderSplatsMulti."""
    assets = mixed_assets(g, 4)
    a = [g.GaussianSplatRenderer(x, ctx) for x in assets]
    b = [g.GaussianSplatRenderer(x, ctx) for x in assets]
    try:
        for i in range(4):
            mixed_setup(i, a[i])
            mixed_setup(i, b[i])
        for f in range(3):
            cams = [orbit(g, f, *CAM_SIZES[c], phase=0.7 * c) for c in range(3)]
            ra = [np.zeros((c.pixelHeight, c.pixelWidth, 4), np.float16) for c in cams]
            rb = [x.copy() for x in ra]
            g.SortAndRenderCameras(a, cams, ra)
            for c, cam in enumerate(cams):
                g.SortAndRenderSplatsMulti(b, cam, rb[c])
            for x, y in zip(ra, rb):
                assert x.any() and np.array_equal(x.view(np.uint16), y.view(np.uint16))
            for p, q in zip(a, b):
                assert p.m_FrameCounter == q.m_FrameCounter == 3 * (f + 1)
                assert np.array_equal(p.readback_order(), q.readback_order())
    finally:
        for r in a + b:
            r.Dispose()


# ---- 2. order chaining ----------------------------------------------------------------------------------------------------
def _plane_asset(g):
    """Splats on planes parallel to camera A's image plane (A looks down +z): A's keys tie within a plane."""
    rng = np.random.default_rng(7)
    n = 24000
    z = rng.integers(0, 6, n).astype(np.float32) * 0.25
    xy = rng.uniform(-1.6, 1.6, (n, 2)).astype(np.float32)
    pos = np.c_[xy, z]
    dc = rng.uniform(0.1, 0.9, (n, 3)).astype(np.float32)
    rec = splat_records(pos, (0.05, 0.05, 0.02), 0.6, dc)
    return g.create_asset(rec, "VeryHigh")


def test_order_chaining(g, ctx, ca):
    """Cameras B, A, C in that order every frame, m_SortNthFrame = 2: A (looking straight at the planes) ties many keys and
    sorts on odd frames only, through the order C's sort left on the frame before; B and C see the planes at an angle.  A's
    independently sorted twin sorts at the same steps from its own history.  After each of A's sorts the keys agree and the
    orders differ: A's ties are broken by the order the previous camera left."""
    asset = _plane_asset(g)
    cam_a = camera(g, 256, 256, pos=(0.0, 0.0, -6.0), forward=(0.0, 0.0, 1.0))
    cams = [orbit(g, 2, 200, 160), cam_a, orbit(g, -2, 97, 61)]
    tw = Twins(g, ctx, [asset])
    alone = g.GaussianSplatRenderer(asset, ctx)   # camera A only: sorted independently, no chaining
    try:
        for r in tw.loop + tw.call + [alone]:
            r.m_SortNthFrame = 2
        rt = np.zeros((256, 256, 4), np.float16)
        for f in range(4):
            compare(g, ctx, ca, tw, [[0], [0], [0]], cams, 0, np.float16, ["device", "host", "array"], [None, None, "device"],
                    "frame %d" % f)
            alone.m_FrameCounter = 3 * f + 1    # A's place in the frame: it sorts exactly when the chained A does
            alone.SortAndRenderSplats(cam_a, rt=rt)
            if f % 2 == 1:   # A sorted last
                keys = alone.readback_keys()
                assert np.count_nonzero(np.diff(keys) == 0) > keys.size // 2, "camera A's keys should tie"
                assert np.array_equal(tw.call[0].readback_keys(), keys), "frame %d: the same keys" % f
                assert not np.array_equal(tw.call[0].readback_order(), alone.readback_order()), \
                    "frame %d: chained and independent orders agree, so the test has no teeth" % f
    finally:
        alone.Dispose()
        tw.dispose()


# ---- 3. run boundaries ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("counts", [[6, 6, 2, 2, 1], [4, 4, 4, 3, 2]])
def test_seventeen_pairs_make_two_runs(g, ctx, ca, counts):
    tw = Twins(g, ctx, mixed_assets(g, 6), mixed_setup)
    try:
        for f in range(2):
            cams = [orbit(g, f, *CAM_SIZES[c], phase=0.5 * c) for c in range(len(counts))]
            subsets = [[(c + j) % 6 for j in range(k)] for c, k in enumerate(counts)]
            idx = tw.gathered(g, subsets, cams)
            assert sum(len(i) for i in idx) == 17
            compare(g, ctx, ca, tw, idx, cams, f, np.float16, ["device", "host", "array", "device", None],
                    ["host", None, "device", None, "device"], "frame %d" % f)
    finally:
        tw.dispose()


@pytest.mark.parametrize("counts, dtypes", [
    ([8, 8, 4, 4], [np.float16] * 4),                                  # 16 pairs, then 8: two runs of two cameras
    ([2, 2, 2, 2], [np.float16, np.float16, np.float32, np.float32]),  # a new pixel format starts the second run
])
def test_two_camera_runs_in_one_call(g, ctx, ca, counts, dtypes):
    """The second run's first emit keeps the overflow flag of the first, the run scratch is laid out again, and each run's camera
    layout keeps its own tile-cost history over the frames."""
    tw = Twins(g, ctx, mixed_assets(g, 8), mixed_setup)
    try:
        for f in range(3):
            cams = [orbit(g, f, *CAM_SIZES[c], phase=0.5 * c) for c in range(len(counts))]
            subsets = [[(c + j) % 8 for j in range(k)] for c, k in enumerate(counts)]
            idx = tw.gathered(g, subsets, cams)
            compare(g, ctx, ca, tw, idx, cams, f % 2, dtypes, ["device", "host", "array", "device"], ["host", None, "device", "array"],
                    "frame %d" % f)
    finally:
        tw.dispose()


def test_large_camera_between_small_ones(g, ctx, ca):
    tw = Twins(g, ctx, mixed_assets(g, 3), mixed_setup)
    try:
        cams = [orbit(g, 1, 97, 61), orbit(g, 1, 8200, 64, phase=0.2), orbit(g, 1, 256, 256, phase=0.4)]
        idx = tw.gathered(g, [[0, 1], [1, 2], [2, 0]], cams)
        compare(g, ctx, ca, tw, idx, cams, 1, np.float32, ["device", "device", "host"], [None, "device", "array"], "large")
    finally:
        tw.dispose()


def test_camera_of_seventeen_objects_between_small_ones(g, ctx, ca):
    """The middle camera cannot join a run: it is drawn as two runs, the second loading the first's image, between two runs of
    one small camera each."""
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, 3000 + 250 * i, 0xCA3E1000 + i, ("Medium", "VeryHigh")[i % 2]) for i in range(17)]

    def setup(i, r):
        r.localToWorldMatrix = g_trs(position=(0.7 * (i % 6) - 1.75, 0.6 * (i // 6) - 0.6, 0.3 * (i % 2)), scale=(0.5, 0.5, 0.5))
        r.m_SortNthFrame = (1, 2)[i % 2]

    tw = Twins(g, ctx, assets, setup)
    try:
        for f, kind in enumerate(["host", "device", "array"]):
            cams = [orbit(g, f, 97, 61), orbit(g, f, 320, 200, phase=0.3), orbit(g, f, 256, 256, phase=0.6)]
            idx = tw.gathered(g, [[0, 1], list(range(17)), [2, 16]], cams)
            assert len(idx[1]) == 17
            assert compare(g, ctx, ca, tw, idx, cams, f % 2, np.float16, ["device", kind, "host"], [None, "device", None],
                           "frame %d" % f) > 0
    finally:
        tw.dispose()


def test_own_depth_buffer_per_camera(g, ctx, ca):
    import torch
    tw = Twins(g, ctx, mixed_assets(g, 3), mixed_setup)
    try:
        cams = [orbit(g, 0, 320, 200), orbit(g, 0, 256, 256, phase=0.6)]
        d0 = np.full((200, 320), 0.02, np.float32)
        d0[:, 160:] = 0.2
        d1 = np.full((256, 256), 0.05, np.float32)
        d1[100:150, :] = np.nan
        d1_dev = torch.from_numpy(d1).cuda()
        idx = tw.gathered(g, [[0, 1, 2], [2, 1]], cams)
        extras = [[{"scene_depth": d0} if k != 1 else {} for k in range(3)], [{"scene_depth": d1_dev}, {"scene_depth": d1_dev}]]
        for blend in (0, 1):
            compare(g, ctx, ca, tw, idx, cams, blend, np.float16, ["host", "device"], ["device", None], "depth", extras)
    finally:
        tw.dispose()


def test_selection_on_one_camera(g, ctx, ca):
    tw = Twins(g, ctx, mixed_assets(g, 2), mixed_setup)
    try:
        cams = [orbit(g, 2, 320, 200), orbit(g, 2, 97, 61, phase=0.3)]
        idx = tw.gathered(g, [[0, 1], [0, 1]], cams)
        sel = np.random.default_rng(3).integers(0, 2 ** 32, (tw.loop[idx[1][0]].splatCount + 31) // 32, dtype=np.uint64).astype(np.uint32)
        extras = [[{}, {}], [{"selected_bits": sel}, {}]]
        compare(g, ctx, ca, tw, idx, cams, 0, np.float16, ["device", "array"], [None, "host"], "selection", extras)
    finally:
        tw.dispose()


def test_camera_with_everything_off_screen(g, ctx, ca):
    tw = Twins(g, ctx, mixed_assets(g, 2), mixed_setup)
    try:
        away = camera(g, 128, 96, pos=(0.0, 0.5, -60.0), forward=(0.0, 0.0, -1.0))
        cams = [orbit(g, 0, 320, 200), away, orbit(g, 1, 97, 61)]
        idx = [[0, 1], [1, 0], [1]]
        drawn = compare(g, ctx, ca, tw, idx, cams, 1, np.float16, ["device", "host", "device"], [None, "device", None], "off screen")
        assert drawn == 2   # every camera but the one looking away drew something
    finally:
        tw.dispose()


# ---- 4. against the oracle ------------------------------------------------------------------------------------------------
def test_two_cameras_against_the_oracle(g, O, ctx, ca):
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, n, 0xCA3E0F20 + i, "Medium") for i, n in enumerate([12000, 8000])]
    tw = Twins(g, ctx, assets)
    try:
        for i, r in enumerate(tw.loop + tw.call):
            r.localToWorldMatrix = g_trs(position=(1.3 * (i % 2) - 0.6, 0.0, 1.0 * (i % 2)), scale=(0.7, 0.7, 0.7))
        cams = [orbit(g, 1, 200, 150), orbit(g, 1, 160, 120, phase=0.8)]
        idx = tw.gathered(g, [[0, 1], [0, 1]], cams)
        # camera 0's orders: what the loop's first camera leaves
        lo, hi = tw.pick(idx)
        rts = [np.zeros((c.pixelHeight, c.pixelWidth, 4), np.float16) for c in cams]
        loop_cameras(g, ctx, lo[:1], cams[:1], 0, rts[:1], [None])
        order0 = {i: tw.loop[i].readback_order() for i in idx[0]}
        call_cameras(g, ctx, hi, cams, 0, rts, [None, None])
        for c, cam in enumerate(cams):
            views, orders, base = [], [], 0
            for i in idx[c]:
                r = tw.call[i]
                fp, _keep = g.make_frame_params(cam, r.localToWorldMatrix)
                views.append(O.frame(r.m_Asset, fp, threads=O.max_threads())["view"])
                order = order0[i] if c == 0 else r.readback_order()
                orders.append(order + np.uint32(base))
                base += r.splatCount
            want = O.render(np.concatenate(views), np.concatenate(orders), cam.pixelWidth, cam.pixelHeight, 0, O.max_threads())
            assert rts[c].any() and np.array_equal(rts[c].astype(np.float32), want), "camera %d" % c
    finally:
        tw.dispose()


# ---- 5. overflow ----------------------------------------------------------------------------------------------------------
def test_overflow_reported_then_next_call_fits(g):
    import torch
    ctx = g.GaussianSplatContext(0)   # a fresh context: its bin list has the smallest capacity (4 Mi entries)
    rng = np.random.default_rng(11)
    n = 8500
    pos = np.c_[rng.uniform(-0.05, 0.05, (n, 2)), rng.uniform(-0.05, 0.05, n)].astype(np.float32)
    huge = g.create_asset(splat_records(pos, (20.0, 20.0, 20.0), 0.02), "VeryHigh")   # every splat covers every bin
    small = g.synthetic_asset(g.SCENE_CLUSTERED, 6000, 0xCA3E0F30, "Medium")
    rh, rs = g.GaussianSplatRenderer(huge, ctx), g.GaussianSplatRenderer(small, ctx)
    try:
        cams = [camera(g, 1024, 1024), camera(g, 1024, 1024, pos=(0.064, 0.5, -6.0))]
        rts = [torch.zeros((1024, 1024, 4), dtype=torch.float16, device="cuda") for _ in cams]
        # 2 x 8500 splats x 256 bins = 4.35 Mi entries > 4 Mi
        assert call_cameras(g, ctx, [[rh], [rh]], cams, 0, rts, [None, None], check=False) == 0
        assert ctx._lib.gs_sync(ctx.handle) == OOM
        host = [np.zeros((1024, 1024, 4), np.float16) for _ in cams]
        assert call_cameras(g, ctx, [[rh], [rh]], cams, 0, host, [None, None], check=False) == OOM
        assert call_cameras(g, ctx, [[rs], [rs]], cams, 0, host, [None, None], check=False) == 0
        assert all(h.any() for h in host)
        assert ctx._lib.gs_sync(ctx.handle) == 0
    finally:
        rh.Dispose()
        rs.Dispose()
        ctx.close()


@pytest.mark.parametrize("host", [False, True])
def test_overflow_kept_across_a_growing_camera(g, host):
    """A truncated run of two cameras, then a camera above 8160 px (129 bin rows, every splat in each) whose own list grows and
    fits: the call still reports the truncation, and the next call that fits reports none."""
    import torch
    ctx = g.GaussianSplatContext(0)   # a fresh context: its bin list has the smallest capacity (4 Mi entries)
    rng = np.random.default_rng(12)
    n = 40000   # 8 n < 4 Mi; on the tall camera n x 129 bins > 4 Mi
    pos = np.c_[rng.uniform(-0.05, 0.05, (n, 2)), rng.uniform(-0.05, 0.05, n)].astype(np.float32)
    huge = g.create_asset(splat_records(pos, (20.0, 20.0, 20.0), 0.02), "VeryHigh")   # every splat covers every bin
    small = g.synthetic_asset(g.SCENE_CLUSTERED, 6000, 0xCA3E0F31, "Medium")
    rh, rs = g.GaussianSplatRenderer(huge, ctx), g.GaussianSplatRenderer(small, ctx)
    try:
        cams = [camera(g, 1024, 1024), camera(g, 1024, 1024, pos=(0.064, 0.5, -6.0)), camera(g, 64, 8200)]
        if host:
            rts = [np.zeros((c.pixelHeight, c.pixelWidth, 4), np.float16) for c in cams]
        else:
            rts = [torch.zeros((c.pixelHeight, c.pixelWidth, 4), dtype=torch.float16, device="cuda") for c in cams]
        rc = call_cameras(g, ctx, [[rh], [rh], [rh]], cams, 0, rts, [None] * 3, check=False)
        if host:
            assert rc == OOM
        else:
            assert rc == 0 and ctx._lib.gs_sync(ctx.handle) == OOM
        assert call_cameras(g, ctx, [[rs], [rs], [rh]], cams, 0, rts, [None] * 3, check=False) == 0
        assert ctx._lib.gs_sync(ctx.handle) == 0
        if host:
            assert ctx.stage_times().tile_entries > 4 << 20, "the tall camera's list must outgrow 4 Mi entries"
            assert all(r.any() for r in rts)
    finally:
        rh.Dispose()
        rs.Dispose()
        ctx.close()


# ---- 6. refused inputs ----------------------------------------------------------------------------------------------------
def test_refused_inputs_write_nothing(g, ctx, ca):
    from unitygaussiansplatting_b200 import _native as N
    tw = Twins(g, ctx, mixed_assets(g, 2), mixed_setup)
    try:
        cams = [orbit(g, 0, 320, 200), orbit(g, 0, 97, 61, phase=0.5)]
        rs = tw.call
        orders = [r.readback_order() for r in rs]
        rts = [np.full((c.pixelHeight, c.pixelWidth, 4), 0.25, np.float16) for c in cams]
        before = [x.copy() for x in rts]
        counters = [r.m_FrameCounter for r in rs]

        def refused(**kw):
            for r, c0 in zip(rs, counters):
                r.m_FrameCounter = c0
            return call_cameras(g, ctx, kw.pop("per_cam", [[rs[0], rs[1]], [rs[1]]]), kw.pop("cams", cams), 0,
                                kw.pop("rts", rts), kw.pop("tgts", [None, None]), check=False, **kw)

        lib = N.native()
        assert lib.gs_frame_cameras(None, 0, None, None, None, None, None, None, None) == INVALID
        assert refused(counts=[2, 0]) == INVALID                                      # a camera without objects
        assert refused(per_cam=[[rs[0], rs[0]], [rs[1]]]) == INVALID                  # an asset twice in one camera
        assert refused(flags=N.GS_FLAG_ASYNC_READBACK) == INVALID
        assert refused(flags=N.GS_FLAG_LOAD_RT) == INVALID
        assert refused(rts=[rts[0], None]) == INVALID                                 # neither image for camera 1
        def shrink(ims):
            ims[1][0].width -= 1
        assert refused(patch=shrink) == INVALID                                       # an image of the wrong size
        assert refused(cams=[cams[0], orbit(g, 0, 16385, 1)], rts=[rts[0], np.zeros((1, 16385, 4), np.float16)]) == INVALID
        assert refused(per_cam=[[], []], cams=[], rts=[], tgts=[], counts=[]) == INVALID   # camera_count 0
        ctx.sync()
        for x, y in zip(rts, before):
            assert np.array_equal(x.view(np.uint16), y.view(np.uint16))
        for r, o in zip(rs, orders):
            assert np.array_equal(r.readback_order(), o)
    finally:
        tw.dispose()


# ---- 7. one camera --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nobj", [1, 3])
def test_one_camera_is_frame_objects(g, ctx, ca, nobj):
    tw = Twins(g, ctx, mixed_assets(g, 3), mixed_setup)
    try:
        ctx.set_timing(True)
        cam = orbit(g, 2, 320, 200)
        idx = tw.gathered(g, [list(range(nobj))], [cam])
        lo, hi = tw.pick(idx)
        a, b = np.zeros((200, 320, 4), np.float16), np.zeros((200, 320, 4), np.float16)
        n0 = ctx.stage_times().kernel_launches
        loop_cameras(g, ctx, lo, [cam], 0, [a], [None])
        n1 = ctx.stage_times().kernel_launches
        call_cameras(g, ctx, hi, [cam], 0, [b], [None])
        n2 = ctx.stage_times().kernel_launches
        assert a.any() and np.array_equal(a.view(np.uint16), b.view(np.uint16))
        assert n2 - n1 == n1 - n0
        tw.check_state()
    finally:
        ctx.set_timing(False)
        tw.dispose()
