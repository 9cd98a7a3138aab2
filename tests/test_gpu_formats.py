"""The view, distance and export kernels against the CPU oracle on the asset format combinations no preset uses
(tests/util.py FORMAT_CASES): Float16 SH, BC7 colour beside unclustered SH, Norm6 and chunked Float32 positions, every
`other` record layout, Cluster64k / 32k palettes and palette indices past the end of the palette.

Every case is rendered under a sheared, rotated object transform with splat and opacity scale, an inverted cutout box,
deleted bits and SH order 3, on a 203 x 117 screen (a multiple of neither the 16-pixel tile nor the 64-pixel bin).  All
splat counts but one are odd, so the last 256-splat block of _SplatViewData ends in an odd-word tail; the inverted box
keeps the last (Morton-outermost) splats, so that tail holds a drawn splat."""
import numpy as np
import pytest

from util import FORMAT_CASES, camera, case_asset, format_case, palette_backed

pytestmark = pytest.mark.gpu

W, H = 203, 117
_ASSETS = {}


def _asset(g, name):
    if name not in _ASSETS:
        _ASSETS[name] = case_asset(g, format_case(name))
    return _ASSETS[name]


@pytest.fixture
def renderer(g, ctx):
    """A renderer on one of the format cases, disposed when the test ends even if it fails: a failed test's frames keep it
    alive, and a later garbage collection could otherwise finalise it after its context."""
    made = []

    def make(name):
        r = g.GaussianSplatRenderer(_asset(g, name), ctx)
        made.append(r)
        _set_knobs(r, r.splatCount)
        return r
    yield make
    for r in made:
        r.Dispose()


def _set_knobs(r, n):
    ang = 0.6
    rot = np.array([[np.cos(ang), -np.sin(ang), 0.0], [np.sin(ang), np.cos(ang), 0.0], [0.0, 0.0, 1.0]])
    shear = np.array([[1.0, 0.3, 0.0], [0.0, 1.0, 0.0], [0.2, 0.0, 1.0]])
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = (rot @ shear * 1.1).astype(np.float32)
    T[:3, 3] = (0.3, -0.1, 0.2)
    deleted = np.zeros((n + 31) // 32, np.uint32)
    deleted[3] = 0xF0F0F0F0
    deleted[-2] = 0x00FF00FF
    r.localToWorldMatrix = T
    r.m_SplatScale, r.m_OpacityScale, r.m_SHOrder = 0.9, 1.3, 3
    r.m_Cutouts = [(np.diag([1 / 3.0, 1 / 3.0, 1 / 3.0, 1.0]).astype(np.float32), 1 | 0x100)]   # cut what lies inside the box
    r.m_DeletedBits = deleted


def _frame_params(g, r, cam):
    return g.make_frame_params(cam, r.localToWorldMatrix, r.m_SplatScale, r.m_OpacityScale, r.m_SHOrder, r.m_SHOnly, r.m_Cutouts,
                               r.m_DeletedBits, r.splatCount)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", [c.name for c in FORMAT_CASES])
def test_fused_and_staged_frames_match_oracle(g, O, renderer, name):
    """The fused frame (k_calc_view<SH, CULL=true, BC7>) and the stand-alone view-calc (CULL=false) against O.frame."""
    r = renderer(name)
    asset, n = r.m_Asset, r.splatCount
    cam = camera(g, W, H)
    rt = np.zeros((H, W, 4), np.float16)
    r.SortAndRenderSplats(cam, rt=rt)
    fp, _keep = _frame_params(g, r, cam)
    ref = O.frame(palette_backed(asset), fp, threads=O.max_threads())
    assert (ref["rt"][..., 3] > 0).mean() > 0.2, "the case no longer draws much of the screen"
    assert np.array_equal(r.readback_keys(), ref["keys"]), "sorted distance keys differ"
    assert np.array_equal(r.readback_order(), ref["order"]), "sorted splat indices differ"
    differ = _bits(rt.astype(np.float32)) != _bits(ref["rt"])
    assert not differ.any(), "fused frame differs from the oracle at %d values, max err %g" % (
        differ.sum(), np.nanmax(np.abs(rt.astype(np.float32) - ref["rt"])))
    r.CalcViewData(cam)
    view = r.readback_view()
    bad = np.nonzero((view != ref["view"]).any(axis=1))[0]
    assert bad.size == 0, "SplatViewData differs for %d splats, first %s" % (bad.size, bad[:5])
    if n % 2:   # the last block holds an odd number of 10-word records: its last two words leave through the tail store
        assert ref["view"][-1, 3].view(np.float32) > 0 and ref["view"][-1, 8:10].all(), "the tail no longer holds a drawn splat"
    rt2 = np.zeros_like(rt)
    r.DrawSplats(cam, rt2)
    assert np.array_equal(rt2.view(np.uint16), rt.view(np.uint16)), "drawing the stand-alone view data differs from the fused frame"


@pytest.mark.parametrize("name", [c.name for c in FORMAT_CASES])
def test_export_matches_oracle(g, O, renderer, name):
    """k_export_data against CSExportData, under tests/test_zz_export_gpu.py's rule: bit-exact but for the log() columns."""
    r = renderer(name)
    asset, n = r.m_Asset, r.splatCount
    got = r.EditExportData()
    fp, _keep = _frame_params(g, r, camera(g, W, H))
    ref = O.export_data(palette_backed(asset), fp, threads=O.max_threads())
    exact = list(range(0, 54)) + list(range(58, 62))      # pos, nor, colour (IEEE sub + div), SH, rotation
    bad = np.nonzero((got[:, exact].view(np.uint32) != ref[:, exact].view(np.uint32)).any(axis=1))[0]
    assert bad.size == 0, "exported records differ for %d splats, first %s" % (bad.size, bad[:5])
    close = np.isclose(got[:, 54:58], ref[:, 54:58], rtol=2e-6, atol=2e-6)      # logf on the GPU, libm's log on the CPU
    assert close.all(), "opacity / log-scale columns differ for %d splats" % (~close).any(axis=1).sum()
    assert 0 < (got[:, 3] != 0).sum() < n


@pytest.mark.parametrize("name", ["norm6pos-f16sh", "f32pos-bc7-f16sh"])
def test_emulated_group_equals_one_gpu(g, renderer, name):
    """A group's key-range splitters are splats of last frame's order decoded through load_pos: an emulated group of 3 must
    give every member the one-GPU draw order and frame, bit for bit, over a short fly-through."""
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    r = renderer(name)
    cams = [camera(g, W, H, pos=(0.5 * i - 0.4, 0.5, -6.0 + 0.4 * i), forward=(0.15 * i, 0.0, 1.0)) for i in range(3)]
    grp = GaussianSplatGroup.create(r.m_Asset, [0, 0, 0], emulate=True)
    try:
        _set_knobs(grp, r.splatCount)
        for k, cam in enumerate(cams):
            rt = np.zeros((H, W, 4), np.float16)
            r.SortAndRenderSplats(cam, rt=rt)
            rts = [np.zeros_like(rt) for _ in range(3)]
            grp.SortAndRenderSplats(cam, rts=rts)
            assert rt.any()
            for i in range(3):
                assert np.array_equal(grp.readback_order(i), r.readback_order()), "frame %d member %d: draw order differs" % (k, i)
                assert np.array_equal(rts[i].view(np.uint16), rt.view(np.uint16)), "frame %d member %d: render target differs" % (k, i)
    finally:
        grp.close()
