"""The sorter's 8192-pair tiles and the bin sort's plans at their boundaries: sizes around one and two tiles, and screens at
both edges of every plan from 32 bins (one 5-bit pass) to 16384 bins (two 7-bit passes).  The two 8-bit passes above 16384
bins, up to 65536 on a 16384 x 16384 screen, are tested in test_gpu_large_screens.py and test_gpu_run_plans.py."""
import numpy as np
import pytest

from util import PLAN_SCREENS, camera, plan_scene

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


# the upper edge of each two-pass digit width sorts enough entries that the persistent grid's CTAs take several tiles
MULTI_TILE = {(2048, 2048), (4096, 4096), (8160, 8160)}


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
        asset = plan_scene(g, cam, 7 * grid_pairs // 5 if (w, h) in MULTI_TILE else 0)
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
