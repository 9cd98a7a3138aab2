"""Where the fused frame decides that something cannot produce a pixel and skips it: the culls at their edges
(fixture from tests/golden/make_cull_edges.py), the bin list at its capacity, and pixels that are saturated before a
splat with an inf colour reaches them.  The oracle has none of these shortcuts: it visits every splat's whole rectangle."""
import numpy as np
import pytest

from util import CAP_ENTRIES, CAP_H, CAP_SPLATS, CAP_W, bin_row_splats, camera, splat_records, world_at_pixel, pixels_per_unit, view_fields

pytestmark = pytest.mark.gpu


# ---- the bin list at its capacity ---------------------------------------------------------------------------------------
def _cap_frame(g, ctx, r, cam, rt=None):
    if rt is None:
        rt = np.zeros((CAP_H, CAP_W, 4), np.float16)
    r.SortAndRenderSplats(cam, rt=rt)
    return rt


def test_bin_list_exact_capacity_overflow_and_recovery(g, O):
    """Fresh context (the session one only grows its list).  65,536 splats of 64 entries fill the 4 Mi list exactly; one
    more overflows it by one splat, which emission (in draw order) drops as a whole: the last one drawn."""
    import torch
    ctx = g.GaussianSplatContext(0)
    renderers = []   # disposed before the context is closed, also when an assertion fails
    try:
        cam = camera(g, CAP_W, CAP_H)
        rec = bin_row_splats(cam, CAP_SPLATS + 1, 0xCA9)
        T = O.max_threads()

        # exact capacity
        full = g.create_asset(rec[:CAP_SPLATS].copy(), "VeryHigh")   # a copy: packing consumes its input
        r = g.GaussianSplatRenderer(full, ctx)
        renderers.append(r)
        rt = _cap_frame(g, ctx, r, cam)
        assert ctx.stage_times().tile_entries == CAP_ENTRIES, "precondition: every splat emits exactly 64 entries"
        fp, _k = g.make_frame_params(cam)
        ref = O.frame(full, fp, threads=T)
        assert np.array_equal(r.readback_order(), ref["order"])
        assert np.array_equal(rt.astype(np.float32), ref["rt"]), "render target at exact capacity differs from the oracle"

        # one splat more: the list is truncated, every synchronising call reports it
        over = g.create_asset(rec, "VeryHigh")
        r = g.GaussianSplatRenderer(over, ctx)
        renderers.append(r)
        fp, _k = g.make_frame_params(cam)
        ref = O.frame(over, fp, threads=T)
        rt = np.zeros((CAP_H, CAP_W, 4), np.float16)
        with pytest.raises(g.GsError) as e:
            _cap_frame(g, ctx, r, cam, rt)
        assert e.value.code == -3 and "tile-list capacity exceeded" in str(e.value)
        assert ctx.stage_times().tile_entries == CAP_ENTRIES
        assert np.array_equal(r.readback_order(), ref["order"])
        truncated = O.render(ref["view"], ref["order"][:-1], CAP_W, CAP_H, 0, T)
        assert not np.array_equal(truncated, ref["rt"]), "the last splat in draw order must be visible for this to test anything"
        assert np.array_equal(rt.astype(np.float32), truncated), "truncation must drop exactly the last splat in draw order"

        dev = torch.zeros((CAP_H, CAP_W, 4), dtype=torch.float16, device="cuda")
        r.SortAndRenderSplats(cam, rt=dev)                     # device target: not checked when enqueued ...
        with pytest.raises(g.GsError) as e:
            ctx.sync()                                         # ... but at the next synchronising call
        assert e.value.code == -3
        assert np.array_equal(dev.cpu().numpy().astype(np.float32), truncated)

        r.async_readback = True
        rt = np.zeros((CAP_H, CAP_W, 4), np.float16)
        r.SortAndRenderSplats(cam, rt=rt)
        with pytest.raises(g.GsError) as e:
            ctx.sync()
        assert e.value.code == -3
        assert np.array_equal(rt.astype(np.float32), truncated)
        r.async_readback = False

        # recovery: delete the splat that no longer fits; the same context renders the next frame exactly
        last = int(ref["order"][-1])
        bits = np.zeros((over.splatCount + 31) // 32, np.uint32)
        bits[last >> 5] |= np.uint32(1 << (last & 31))
        r.m_DeletedBits = bits
        rt = _cap_frame(g, ctx, r, cam)
        assert ctx.stage_times().tile_entries == CAP_ENTRIES
        fp, _k = g.make_frame_params(cam, deleted_bits=bits, splat_count=over.splatCount)
        ref2 = O.frame(over, fp, prev_order=ref["order"], threads=T)
        assert np.array_equal(r.readback_order(), ref2["order"])
        assert np.array_equal(rt.astype(np.float32), ref2["rt"])
    finally:
        for r in renderers:
            r.Dispose()
        ctx.close()


# ---- saturated pixels under a splat with an inf colour -----------------------------------------------------------------
@pytest.mark.parametrize("blend", [0, 1])
def test_saturated_pixels_ignore_an_inf_colour_behind(g, O, ctx, blend):
    """An opaque splat (opacity 0.2 x m_OpacityScale 100) saturates a disc of about 24 px radius whose edge cuts through
    some 8x4 warp blocks and covers others (and whole 16x16 tiles); 40 faint splats follow, so that the raster's warps
    reach a second 32-splat batch, where the last splat has f_dc = 1e6, a colour of half inf.  A pixel with dst.a == 1
    ignores every later splat, whatever its warp neighbours do; the others get +inf."""
    W, H = 160, 128
    cam = camera(g, W, H)
    ppu = pixels_per_unit(cam, 6.0)
    depth = np.r_[6.0, np.linspace(6.1, 6.4, 40), 6.5]
    pos = world_at_pixel(cam, np.r_[77.3, np.full(40, 79.0), 80.6], np.r_[61.8, np.full(40, 63.0), 66.1], depth)
    sigma = np.r_[[[10.0, 9.0, 9.5]], np.tile([[31.0, 27.0, 29.0]], (40, 1)), [[30.0, 26.0, 28.0]]]
    dc = np.r_[[[0.9, 0.4, 0.1]], np.tile([[0.2, 0.3, 0.6]], (40, 1)), [[1e6, 1e6, 1e6]]]
    rec = splat_records(pos, sigma / ppu, np.r_[0.2, np.full(40, 0.0002), 0.6], dc)
    asset = g.create_asset(rec, "VeryHigh")
    r = g.GaussianSplatRenderer(asset, ctx)
    r.m_OpacityScale = 100.0
    r.blend_mode = blend
    rt = np.zeros((H, W, 4), np.float32 if blend else np.float16)
    r.SortAndRenderSplats(cam, rt=rt)
    fp, _k = g.make_frame_params(cam, opacity_scale=100.0)
    ref = O.frame(asset, fp, blend_mode=blend, threads=O.max_threads())
    order, view = ref["order"], ref["view"]
    inf_id = int(np.nonzero(np.isinf(view_fields(view)["r"]))[0][0])
    assert order[-1] == inf_id, "the inf splat is drawn last"
    got = rt.astype(np.float32)
    assert np.array_equal(got, ref["rt"], equal_nan=False), "kernel and oracle differ (NaN: %d vs %d pixels)" % (
        np.isnan(got).any(-1).sum(), np.isnan(ref["rt"]).any(-1).sum())
    before = O.render(view, order[:-1], W, H, blend)
    sat = before[..., 3] == 1.0
    blocks = sat.reshape(H // 4, 4, W // 8, 8).transpose(0, 2, 1, 3).reshape(H // 4, W // 8, 32).sum(-1)
    assert (blocks == 32).sum() >= 8 and ((blocks > 0) & (blocks < 32)).sum() >= 8, "the disc must cover some warp blocks and cut others"
    assert np.array_equal(got[sat], before[sat]), "a saturated pixel changed under the splat behind it"
    drawn = O.render(view, order[-1:], W, H, blend)[..., 3] > 0
    open_px = drawn & ~sat
    assert open_px.sum() > 100 and np.isposinf(got[open_px][:, :3]).all(), "unsaturated pixels the inf splat covers are +inf"
    assert not np.isnan(got).any()
    r.Dispose()


# ---- culls at their edges ----------------------------------------------------------------------------------------------
def _fixture():
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).parent / "golden"))
    import make_cull_edges
    return make_cull_edges.load()


FIX = _fixture()
EXTRA_FAMILIES = ["internal", "discard", "discard_scaled"]


def _fp(fam):
    import ctypes as C
    from unitygaussiansplatting_b200 import _native as N
    fp = N.GsFrameParams()
    raw = np.ascontiguousarray(fam["fp"])
    C.memmove(C.addressof(fp), raw.ctypes.data, raw.size)
    return fp, int(fp.screen_w), int(fp.screen_h)


def _fused_staged_oracle(g, O, ctx, asset, fp, W, H, blend=0, rows=(0, 0)):
    """The fused frame, the staged path (gs_calc_view + gs_render, which culls nothing) and the oracle on one asset."""
    import ctypes as C
    from unitygaussiansplatting_b200 import _native as N
    r = g.GaussianSplatRenderer(asset, ctx)
    r.blend_mode = blend
    r.rows = rows
    dt = np.float32 if blend else np.float16
    rt = np.zeros((H, W, 4), dt)
    r.SortAndRenderSplats(camera(g, W, H), rt=rt, fp=fp)
    ref = O.frame(asset, fp, blend_mode=blend, threads=O.max_threads())
    assert np.array_equal(r.readback_order(), ref["order"]), "draw order differs from the oracle"
    lib = N.native()
    N.check(ctx.handle, lib.gs_calc_view(ctx.handle, r._asset, C.byref(fp)))
    staged = np.zeros_like(rt)
    opt = r._options()
    N.check(ctx.handle, lib.gs_render(ctx.handle, r._asset, C.byref(fp), C.byref(opt), C.byref(g.renderer._image(staged, W, H))))
    r.Dispose()
    return rt.astype(np.float32), staged.astype(np.float32), ref


@pytest.mark.parametrize("side", ["in", "out"])
@pytest.mark.parametrize("name", sorted(FIX))
def test_cull_edges_fused_frame_matches_oracle(g, O, ctx, name, side):
    """Splats bisected onto the edges where the fused frame culls (one pixel in, or none): the fused frame draws exactly
    the oracle's pixels and the staged path's, and every in-splat's witness pixel."""
    fam = FIX[name]
    fp, W, H = _fp(fam)
    asset = g.create_asset(np.array(fam[side], np.float32), fam["quality"].item())   # a copy: packing consumes it
    got, staged, ref = _fused_staged_oracle(g, O, ctx, asset, fp, W, H)
    assert np.array_equal(got, ref["rt"]), "%s/%s: fused frame differs from the oracle at %d pixels" % (
        name, side, (got != ref["rt"]).any(-1).sum())
    assert np.array_equal(staged, got), "%s/%s: staged path differs from the fused frame" % (name, side)
    if side == "in":
        w = fam["witness"]
        missing = w[got[w[:, 1], w[:, 0], 3] == 0]
        assert missing.size == 0, "%s: witness pixels not drawn by the kernel: %s" % (name, missing.tolist())
    t0, t1 = (int(v) for v in fam["rows"])
    if t1 > t0:
        part, part_staged, _ = _fused_staged_oracle(g, O, ctx, asset, fp, W, H, rows=(t0, t1))
        assert np.array_equal(part[16 * t0:16 * t1], got[16 * t0:16 * t1]), "%s/%s: rows [%d, %d) differ from the full frame" % (
            name, side, 16 * t0, 16 * t1)
        assert not part[:16 * t0].any() and not part[16 * t1:].any()
        assert np.array_equal(part_staged, part)


@pytest.mark.parametrize("extra", ["selected", "scene_depth", "fp32_blend"])
@pytest.mark.parametrize("side", ["in", "out"])
@pytest.mark.parametrize("name", EXTRA_FAMILIES)
def test_cull_edges_other_raster_paths(g, O, ctx, name, side, extra):
    """The same edge splats through the raster's other instantiations: every splat selected (opacity-1 footprint), a scene
    depth buffer bound, and float32 blending.  The witnesses were found under the default rule: only parity is asserted."""
    fam = FIX[name]
    fp, W, H = _fp(fam)
    asset = g.create_asset(np.array(fam[side], np.float32), fam["quality"].item())   # a copy: packing consumes it
    keep = None
    if extra == "selected":
        keep = np.full((asset.splatCount + 31) // 32, 0xFFFFFFFF, np.uint32)
        fp.selected_bits = keep.ctypes.data
    elif extra == "scene_depth":
        keep = np.random.default_rng(W * H).uniform(0.0, 0.1, (H, W)).astype(np.float32)   # the splats' z_ndc is about 0.05
        fp.scene_depth, fp.scene_depth_on_device = keep.ctypes.data, 0
    got, staged, ref = _fused_staged_oracle(g, O, ctx, asset, fp, W, H, blend=1 if extra == "fp32_blend" else 0)
    assert np.array_equal(got, ref["rt"]), "%s/%s/%s: fused frame differs from the oracle" % (name, side, extra)
    assert np.array_equal(staged, got), "%s/%s/%s: staged path differs from the fused frame" % (name, side, extra)
    del keep
