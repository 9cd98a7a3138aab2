"""The sorter's 8192-pair tiles and the bin sort's plans at their boundaries: sizes around one and two tiles, and screens whose
bin count takes one 9-bit pass (510 and exactly 512 bins) or two passes (544 bins)."""
import numpy as np
import pytest

from util import camera

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


def test_bin_sort_plans_render_exactly(g, O, ctx):
    """30x17 = 510 and 32x16 = 512 bins sort in one 9-bit pass, 32x17 = 544 bins in two: one kernel launch more per frame."""
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 60000, 0x5EED0002, "Medium")
    r = g.GaussianSplatRenderer(asset, ctx)
    launches = {}
    for w, h in [(1920, 1080), (2048, 1024), (2048, 1088)]:
        cam = camera(g, w, h)
        rt = np.zeros((h, w, 4), np.float16)
        r.upload_order(np.arange(asset.splatCount, dtype=np.uint32))   # the oracle frame starts from the identity order
        before = ctx.stage_times().kernel_launches
        r.SortAndRenderSplats(cam, rt=rt)
        launches[w, h] = ctx.stage_times().kernel_launches - before
        fp, _keep = g.make_frame_params(cam)
        ref = O.frame(asset, fp, threads=O.max_threads())
        assert np.array_equal(r.readback_order(), ref["order"]), "sorted splat indices differ at %dx%d" % (w, h)
        assert np.array_equal(rt.astype(np.float32), ref["rt"]), "fp16-ROP render target differs at %dx%d" % (w, h)
    assert launches[1920, 1080] == launches[2048, 1024] == launches[2048, 1088] - 1
    r.Dispose()
