"""The sorter's 8192-pair tiles and the bin sort's plans at their boundaries: sizes around one and two tiles, and screens at
both edges of every plan from 32 bins (one 5-bit pass) to 16384 bins (two 7-bit passes).  The two 8-bit passes above 16384
bins, up to 65536 on a 16384 x 16384 screen, are tested in test_gpu_large_screens.py and test_gpu_run_plans.py."""
import numpy as np
import pytest

from util import camera, splat_records, world_at_pixel, pixels_per_unit

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind", ["random", "equal"])
@pytest.mark.parametrize("n", [8191, 8192, 8193, 16383, 16385])
def test_sort_pairs_around_tile_edges(ctx, n, kind):
    rng = np.random.default_rng(n)
    keys = rng.integers(0, 2**32, n, dtype=np.uint32) if kind == "random" else np.full(n, 0x80000001, np.uint32)
    k, p = keys.copy(), np.arange(n, dtype=np.uint32)
    ctx.sort_pairs(k, p)
    order = np.argsort(keys, kind="stable").astype(np.uint32)
    assert np.array_equal(p, order), "payload order differs from a stable sort"
    assert np.array_equal(k, keys[order])


# (width, height): bins = ceil(W/64) * ceil(H/64); bin_sort_plan takes one pass up to 512 bins (5, 6, 7, 8, 9 bits at 32, 64,
# 128, 256, 512), else two passes of 5, 6, 7, 8 bits up to 1024, 4096, 16384, 65536 bins.  Each plan up to 7 bits at its upper
# edge and one past it.
PLAN_SCREENS = [
    ((512, 256), 32, 1, 5), ((704, 192), 33, 1, 6),
    ((512, 512), 64, 1, 6), ((832, 320), 65, 1, 7),
    ((1024, 512), 128, 1, 7), ((2752, 192), 129, 1, 8),
    ((1024, 1024), 256, 1, 8), ((2752, 384), 258, 1, 9),        # 257 bins is prime: it would need a 16448-pixel row
    ((1920, 1080), 510, 1, 9), ((2048, 1024), 512, 1, 9),
    ((2048, 1088), 544, 2, 5), ((1728, 1216), 513, 2, 5),
    ((2048, 2048), 1024, 2, 5), ((2624, 1600), 1025, 2, 6),
    ((4096, 4096), 4096, 2, 6), ((5248, 3200), 4100, 2, 7),
    ((8160, 8160), 16384, 2, 7),                                # also the largest camera a camera run takes
]
# the upper edge of each two-pass digit width sorts enough entries that the persistent grid's CTAs take several tiles
MULTI_TILE = {(2048, 2048), (4096, 4096), (8160, 8160)}


def _plan_scene(g, cam, entries):
    """The clustered scene, a few small splats in the bottom-right bin (where a digit one bit too narrow mis-sorts), and,
    when `entries` is set, wide flat splats across the whole screen on the bin-row boundaries: 2 x binsX entries each,
    as many as give about `entries`."""
    W, H = cam.pixelWidth, cam.pixelHeight
    base = g.generate_input_splats(g.SCENE_CLUSTERED, 60000, 0x5EED0002)
    ppu = pixels_per_unit(cam, 6.0)
    corner = splat_records(world_at_pixel(cam, [W - 20.5, W - 6.0, W - 40.2], [H - 18.3, H - 40.0, H - 5.5], 6.0),
                           np.array([3.0, 2.0, 2.5]) / ppu, 0.9, (0.2, 0.9, 0.4))
    parts = [base, corner]
    if entries:
        bins_x, bins_y = -(-W // 64), -(-H // 64)
        n = -(-entries // (2 * bins_x))
        rng = np.random.default_rng(W * H)
        depth = 5.0 + 3.0 * rng.random(n)
        cy = 64.0 * (1 + np.arange(n) % (bins_y - 1))
        scale = np.array([0.3 * W, 0.01, 0.01]) / pixels_per_unit(cam, depth)[:, None]
        parts.append(splat_records(world_at_pixel(cam, W / 2, cy, depth), scale, 0.1 + 0.3 * rng.random(n), rng.random((n, 3))))
    return g.create_asset(np.ascontiguousarray(np.concatenate(parts)), "Medium")


def test_bin_sort_plans_render_exactly(g, O, ctx):
    """Every bin-sort plan at both edges renders the oracle's frame bit for bit, bottom-right bin included; a one-pass plan
    launches exactly one kernel fewer than a two-pass plan; and the 5-, 6- and 7-bit persistent sorts each get more than
    one 8192-pair tile per CTA somewhere (2 CTAs per SM)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid_pairs = 2 * sms * 8192
    launches = {1: set(), 2: set()}
    for (w, h), bins, passes, bits in PLAN_SCREENS:
        assert -(-w // 64) * -(-h // 64) == bins
        cam = camera(g, w, h)
        # 1.4 x the grid's pairs: more than one tile per CTA, and with the scene still inside the list's 4 Mi minimum
        asset = _plan_scene(g, cam, 7 * grid_pairs // 5 if (w, h) in MULTI_TILE else 0)
        r = g.GaussianSplatRenderer(asset, ctx)
        rt = np.zeros((h, w, 4), np.float16)
        before = ctx.stage_times().kernel_launches
        r.SortAndRenderSplats(cam, rt=rt)
        st = ctx.stage_times()
        launches[passes].add(st.kernel_launches - before)
        if (w, h) in MULTI_TILE:
            assert st.tile_entries > grid_pairs, "%dx%d (%d-bit plan) sorts %d entries, one tile per CTA" % (w, h, bits, st.tile_entries)
        fp, _keep = g.make_frame_params(cam)
        ref = O.frame(asset, fp, threads=O.max_threads())
        assert ref["rt"][(bins // -(-w // 64) - 1) * 64:, (-(-w // 64) - 1) * 64:, 3].max() > 0, "nothing draws in the last bin"
        assert np.array_equal(r.readback_order(), ref["order"]), "sorted splat indices differ at %dx%d" % (w, h)
        assert np.array_equal(rt.astype(np.float32), ref["rt"]), "fp16-ROP render target differs at %dx%d" % (w, h)
        r.Dispose()
        del rt, ref
    assert len(launches[1]) == 1 and len(launches[2]) == 1, launches
    assert launches[1].pop() == launches[2].pop() - 1
