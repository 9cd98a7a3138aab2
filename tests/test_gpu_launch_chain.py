"""The frame's launch chain (DESIGN §5 "Launch chain"): kernels placed while their predecessor drains, the view-calc run beside
the depth sort's last pass, the launch order computed beside the bin sort, and the per-frame clears done by kernels.  None of
it may change a bit.  Each case below is one where a kernel's early work could meet a buffer an earlier kernel still uses:
  * runs where an asset is binned and then sorted and view-calculated again (same call), every object sorted every frame;
  * back-to-back frames at two screen sizes (the tile-cost history is reset between them, and the launch order restarts);
  * a frame wider than 8160 px (the host waits for the binning and reads the bin list's total back before the raster);
  * an emulated group of 2 (view-calc on a second stream beside the slab sort)."""
import numpy as np
import pytest

from frame_loops import CAM_SIZES, Twins, compare, compare_frame, mixed_assets, mixed_setup, orbit
from images import ca  # noqa: F401
from util import camera

pytestmark = pytest.mark.gpu


def _sort_every_frame(i, r):
    mixed_setup(i, r)
    r.m_SortNthFrame = 1


@pytest.mark.parametrize("blend", [0, 1])
def test_camera_run_sorts_and_views_an_asset_it_has_binned(g, ctx, ca, blend):
    """Every camera draws the same two assets, so each later pair's sort and view-calc follows the bin emit of the same asset
    for an earlier camera; every pair is sorted, so every view-calc runs beside the sort's last pass."""
    tw = Twins(g, ctx, mixed_assets(g, 3), _sort_every_frame)
    try:
        for f in range(3):
            cams = [orbit(g, f, *CAM_SIZES[c], phase=0.7 * c) for c in range(3)]
            idx = tw.gathered(g, [[0, 1], [0, 1], [1, 0]], cams)
            assert compare(g, ctx, ca, tw, idx, cams, blend, np.float16, ["device"] * 3, [None] * 3, "frame %d" % f) > 0
    finally:
        tw.dispose()


@pytest.mark.parametrize("blend", [0, 1])
def test_object_run_sorted_every_frame_equals_the_loop(g, ctx, ca, blend):
    tw = Twins(g, ctx, mixed_assets(g, 4), _sort_every_frame)
    try:
        for f in range(3):
            cam = orbit(g, f)
            compare_frame(g, ctx, ca, tw, cam, blend, np.float16, "device", "device", "frame %d" % f)
    finally:
        tw.dispose()


def _frame(r, cam):
    rt = np.zeros((cam.pixelHeight, cam.pixelWidth, 4), np.float16)
    r.SortAndRenderSplats(cam, rt=rt)
    return rt, r.readback_order()


def test_two_screen_sizes_back_to_back(g, ctx):
    """One renderer alternates two screen sizes (tile history reset, launch order without history, then with it); another
    renders each size alone.  Pixels do not depend on the launch order, so both must agree bit for bit."""
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED0002, "Medium")
    sizes = [(320, 200), (256, 256)]
    alt = g.GaussianSplatRenderer(asset, ctx)
    alone = {s: g.GaussianSplatRenderer(asset, ctx) for s in sizes}
    try:
        for f in range(6):
            W, H = sizes[f % 2]
            cam = orbit(g, f, W, H)
            want_rt, want_order = _frame(alone[(W, H)], cam)
            rt, order = _frame(alt, cam)
            assert want_rt.any()
            assert np.array_equal(rt.view(np.uint16), want_rt.view(np.uint16)), "frame %d (%dx%d): render target" % (f, W, H)
            # the orders evolve from different histories after the first frames; the first frame of each size shares it
            if f == 0:
                assert np.array_equal(order, want_order)
    finally:
        alt.Dispose()
        for r in alone.values():
            r.Dispose()


def test_grown_bin_list_against_the_oracle(g, O, ctx):
    """A screen of more than 128 bins on an axis (> 8160 px): the host waits for the binning and reads the list's total back
    (growing the list and binning again when it overflowed) before the raster.  The frame must match the CPU oracle."""
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0002, "Medium")
    cam = camera(g, 8256, 96, pos=(0.0, 0.5, -6.0))
    r = g.GaussianSplatRenderer(asset, ctx)
    try:
        prev = r.readback_order()
        rt = np.zeros((cam.pixelHeight, cam.pixelWidth, 4), np.float16)
        r.SortAndRenderSplats(cam, rt=rt)
        fp, _keep = g.make_frame_params(cam)
        ref = O.frame(asset, fp, prev_order=prev, threads=O.max_threads())
        assert np.array_equal(r.readback_order(), ref["order"])
        assert rt.any()
        assert np.abs(rt.astype(np.float32) - ref["rt"]).max() <= 1e-3
    finally:
        r.Dispose()


def test_emulated_group_of_two_equals_one_gpu(g, ctx):
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 30000, 0x5EED0003, "Medium")
    r = g.GaussianSplatRenderer(asset, ctx)
    grp = GaussianSplatGroup.create(asset, [0, 0], emulate=True)
    try:
        for f in range(4):
            cam = orbit(g, f)
            rt, order = _frame(r, cam)
            rts = [np.zeros_like(rt) for _ in range(2)]
            grp.SortAndRenderSplats(cam, rts=rts)
            assert rt.any()
            for i in range(2):
                assert np.array_equal(grp.readback_order(i), order), "frame %d member %d: draw order" % (f, i)
                assert np.array_equal(rts[i].view(np.uint16), rt.view(np.uint16)), "frame %d member %d: render target" % (f, i)
    finally:
        grp.close()
        r.Dispose()
