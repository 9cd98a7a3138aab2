"""gs_asset_instance: a further renderer of an uploaded asset, sharing its five blobs in HBM and owning its draw order, keys, view
data and draw state.  Every instance is compared, bit for bit, with a separately uploaded copy of the same asset that gets
the same calls: render targets, camera targets, draw orders, sorted keys and _SplatViewData."""
import ctypes as C
import itertools

import numpy as np
import pytest

from frame_loops import call_cameras, call_frame, frame_args, mixed_setup, next_sort, opt, orbit
from golden.make_golden import CASES
from images import bits
from util import camera

pytestmark = pytest.mark.gpu

INVALID = -1
BLOBS = (3, 4, 5, 6, 7)   # gs_asset_device_ptr: pos, other, sh, color, chunks
OWN = (0, 1, 2)           # order, keys, view


# ---- fixtures -------------------------------------------------------------------------------------------------------------
def _golden_asset(g, name):
    kind, n, seed, quality, _w, _h, _pos, _sh = CASES[name]
    return g.synthetic_asset(kind, n, seed, quality)


ASSETS = {
    "lattice_1k_medium": lambda g: _golden_asset(g, "lattice_1k_medium"),
    "clustered_4k_medium_sh1": lambda g: _golden_asset(g, "clustered_4k_medium_sh1"),
    "clustered_4k_veryhigh": lambda g: _golden_asset(g, "clustered_4k_veryhigh"),
    # the bench scene's generator (bench.py: clustered, seed 0x5EED0002, Medium) at a reduced count
    "bench_200k_medium": lambda g: g.synthetic_asset(g.SCENE_CLUSTERED, 200_000, 0x5EED0002, "Medium"),
}
_cache = {}


def asset_of(g, name):
    if name not in _cache:
        _cache[name] = ASSETS[name](g)
    return _cache[name]


def ptr_of(handle, which):
    from unitygaussiansplatting_b200 import _native as N
    return N.native().gs_asset_device_ptr(handle, which)


def ptr(r, which):
    return ptr_of(r._asset, which)


def rt_of(cam, dtype=np.float16):
    return np.zeros((cam.pixelHeight, cam.pixelWidth, 4), dtype)


def frame(r, cam, dtype=np.float16):
    rt = rt_of(cam, dtype)
    r.SortAndRenderSplats(cam, rt=rt)
    return rt


def knobs(r, **kw):
    for k, v in kw.items():
        setattr(r, k, v)
    return r


def random_bits(n, every, seed):
    rng = np.random.default_rng(seed)
    b = np.zeros((n + 31) // 32, np.uint32)
    ids = np.nonzero(rng.random(n) < 1.0 / every)[0]
    np.bitwise_or.at(b, ids >> 5, np.uint32(1) << (ids & 31).astype(np.uint32))
    return b


def assert_same(a, b, what):
    """Draw order and sorted keys (every renderer of these tests sorts in its first frame)."""
    assert np.array_equal(a.readback_order(), b.readback_order()), what + ": draw order"
    assert np.array_equal(a.readback_keys(), b.readback_keys()), what + ": sorted keys"


# ---- 1. pixels and state over several frames ------------------------------------------------------------------------------
@pytest.mark.parametrize("sort_nth", [1, 2])
@pytest.mark.parametrize("name", list(ASSETS))
def test_frames_equal_a_separate_upload(g, ctx, name, sort_nth):
    """Source, instance and a second upload drawn with the same calls: every frame's pixels, the draw order and sorted keys,
    and _SplatViewData after gs_calc_view are identical across the three."""
    asset = asset_of(g, name)
    src = g.GaussianSplatRenderer(asset, ctx)
    inst = src.Instance()
    twin = g.GaussianSplatRenderer(asset, ctx)
    rs = [knobs(r, m_SortNthFrame=sort_nth) for r in (src, inst, twin)]
    try:
        for f in range(5):
            cam = orbit(g, f)
            want = frame(twin, cam)
            assert want[..., 3].any(), "frame %d draws nothing" % f
            for r, who in ((src, "source"), (inst, "instance")):
                assert np.array_equal(bits(frame(r, cam)), bits(want)), "%s frame %d: render target" % (who, f)
                assert_same(r, twin, "%s frame %d" % (who, f))
            if f % 2:
                for r in rs:
                    r.CalcViewData(cam)
                want_view = twin.readback_view()
                assert np.array_equal(src.readback_view(), want_view), "source frame %d: view data" % f
                assert np.array_equal(inst.readback_view(), want_view), "instance frame %d: view data" % f
    finally:
        for r in rs:
            r.Dispose()


# ---- 2. independence ------------------------------------------------------------------------------------------------------
def test_source_and_instance_keep_their_own_state(g, ctx):
    """Source and instance drawn with different transforms, cutouts, deleted / selected bits and sort cadences: each one's
    order and pixels equal its own separately uploaded twin's, and one's gs_calc_view leaves the other's view data alone."""
    asset = asset_of(g, "bench_200k_medium")
    n = asset.splatCount
    setups = [
        dict(localToWorldMatrix=g.trs(position=(-0.6, 0.0, 0.5)).astype(np.float32), m_SortNthFrame=1,
             m_Cutouts=[(np.linalg.inv(g.trs(scale=(1.8, 1.8, 1.8))), 0)], m_DeletedBits=random_bits(n, 7, 1)),
        dict(localToWorldMatrix=(g.trs(position=(0.7, 0.2, 1.0)) @ np.diag([-0.9, 0.9, 0.9, 1.0])).astype(np.float32),
             m_SortNthFrame=3, m_SHOrder=1, m_OpacityScale=0.8, m_SelectedBits=random_bits(n, 5, 2)),
    ]
    src = g.GaussianSplatRenderer(asset, ctx)
    inst = src.Instance()
    twins = [g.GaussianSplatRenderer(asset, ctx) for _ in range(2)]
    for r, t, kw in zip((src, inst), twins, setups):
        knobs(r, **kw)
        knobs(t, **kw)
    try:
        for f in range(5):
            cam = orbit(g, f)
            for k, (r, t) in enumerate(zip((src, inst), twins)):
                want = frame(t, cam)
                assert np.array_equal(bits(frame(r, cam)), bits(want)), "object %d frame %d: render target" % (k, f)
                assert_same(r, t, "object %d frame %d" % (k, f))
        assert not np.array_equal(src.readback_order(), inst.readback_order())
        cam_a, cam_b = orbit(g, 1), orbit(g, 7)
        inst.CalcViewData(cam_a)
        view = inst.readback_view()
        src.CalcViewData(cam_b)
        assert np.array_equal(inst.readback_view(), view), "the source's gs_calc_view changed the instance's view data"
        twins[0].CalcViewData(cam_b)
        assert np.array_equal(src.readback_view(), twins[0].readback_view())
        assert not np.array_equal(src.readback_view(), view)
        inst.CalcViewData(cam_b)   # and the other way round
        view = src.readback_view()
        inst.CalcViewData(cam_a)
        assert np.array_equal(src.readback_view(), view), "the instance's gs_calc_view changed the source's view data"
    finally:
        for r in [src, inst] + twins:
            r.Dispose()


# ---- 3. several objects and cameras ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("blend", [0, 1])
@pytest.mark.parametrize("depth", [False, True])
def test_frame_objects_over_instances_equal_three_uploads(g, ctx, blend, depth):
    """gs_frame_objects of a source and two of its instances in one camera against the same call over three uploads."""
    asset = asset_of(g, "bench_200k_medium")
    src = g.GaussianSplatRenderer(asset, ctx)
    shared = [src, src.Instance(), src.Instance()]
    uploads = [g.GaussianSplatRenderer(asset, ctx) for _ in range(3)]
    W, H = 320, 200
    ramp = np.broadcast_to(np.linspace(0.0, 0.1, W, dtype=np.float32), (H, W)).copy() if depth else None
    for i, (p, q) in enumerate(zip(shared, uploads)):
        mixed_setup(i, p)
        mixed_setup(i, q)
        p.sceneDepth = q.sceneDepth = ramp
    try:
        for f in range(4):
            cam = orbit(g, f, W, H)
            tgt0 = (np.random.default_rng(f).random((H, W, 4), np.float32) * 0.5).astype(np.float16)
            want_rt, want_tgt, got_rt, got_tgt = rt_of(cam), tgt0.copy(), rt_of(cam), tgt0.copy()
            call_frame(g, ctx, uploads, cam, blend, want_rt, want_tgt)
            call_frame(g, ctx, shared, cam, blend, got_rt, got_tgt)
            assert want_rt[..., 3].any()
            assert np.array_equal(bits(got_rt), bits(want_rt)), "frame %d: render target" % f
            assert np.array_equal(bits(got_tgt), bits(want_tgt)), "frame %d: camera target" % f
            for k, (p, q) in enumerate(zip(shared, uploads)):
                assert_same(p, q, "frame %d object %d" % (f, k))
    finally:
        for r in shared + uploads:
            r.Dispose()


@pytest.mark.parametrize("blend", [0, 1])
def test_frame_cameras_over_instances_equal_separate_uploads(g, ctx, blend):
    """gs_frame_cameras with two cameras, each drawing the source and an instance, against the same call over uploads."""
    asset = asset_of(g, "bench_200k_medium")
    src = g.GaussianSplatRenderer(asset, ctx)
    shared = [src, src.Instance()]
    uploads = [g.GaussianSplatRenderer(asset, ctx) for _ in range(2)]
    for i, (p, q) in enumerate(zip(shared, uploads)):
        mixed_setup(i, p)
        mixed_setup(i, q)
    try:
        for f in range(3):
            cams = [orbit(g, f, 320, 200), orbit(g, f, 256, 256, phase=1.3)]
            rts = [[rt_of(c) for c in cams] for _ in range(2)]
            tgts = [[np.full((c.pixelHeight, c.pixelWidth, 4), 0.25, np.float16) for c in cams] for _ in range(2)]
            call_cameras(g, ctx, [uploads, uploads], cams, blend, rts[0], tgts[0])
            call_cameras(g, ctx, [shared, shared], cams, blend, rts[1], tgts[1])
            for c in range(2):
                assert rts[0][c][..., 3].any()
                assert np.array_equal(bits(rts[1][c]), bits(rts[0][c])), "frame %d camera %d: render target" % (f, c)
                assert np.array_equal(bits(tgts[1][c]), bits(tgts[0][c])), "frame %d camera %d: camera target" % (f, c)
            for k, (p, q) in enumerate(zip(shared, uploads)):
                assert_same(p, q, "frame %d object %d" % (f, k))
    finally:
        for r in shared + uploads:
            r.Dispose()


# ---- 4. lifetime ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["clustered_4k_medium_sh1", "clustered_4k_veryhigh"])
def test_blobs_are_shared_and_outlive_the_source(g, ctx, name):
    """The blob pointers of a source, its instance and an instance of that instance are one set; their own buffers are not.
    With the source destroyed, and then the first instance, the rest keep drawing what a separate upload draws."""
    asset = asset_of(g, name)
    src = g.GaussianSplatRenderer(asset, ctx)
    a = src.Instance()
    b = a.Instance()
    twin = g.GaussianSplatRenderer(asset, ctx)
    try:
        for w in BLOBS:
            assert ptr(a, w) == ptr(src, w) == ptr(b, w), "blob %d is not shared" % w
            if w != 7:
                assert ptr(src, w) and ptr(src, w) != ptr(twin, w)
        assert (ptr(src, 7) is None) == (asset.chunkData is None), "chunk pointer"
        for w in OWN:
            assert len({ptr(src, w), ptr(a, w), ptr(b, w)}) == 3, "per-renderer buffer %d is shared" % w
        assert ptr(src, 8) is None and ptr(src, -1) is None
        for f in range(2):
            cam = orbit(g, f)
            want = frame(twin, cam)
            if f == 0:
                frame(src, cam)
                src.Dispose()
            for r in (a, b):
                assert np.array_equal(bits(frame(r, cam)), bits(want)), "frame %d after the source went" % f
                assert_same(r, twin, "frame %d" % f)
        a.Dispose()
        cam = orbit(g, 2)
        want = frame(twin, cam)
        assert np.array_equal(bits(frame(b, cam)), bits(want)), "the instance of an instance after both sources went"
        ctx.sync()
    finally:
        for r in (src, a, b, twin):
            r.Dispose()


def test_every_destruction_order_leaves_the_context_clean(g, ctx):
    asset = asset_of(g, "lattice_1k_medium")
    cam = orbit(g, 0)
    check = g.GaussianSplatRenderer(asset, ctx)
    want = frame(check, cam)
    try:
        for perm in itertools.permutations(range(3)):
            src = g.GaussianSplatRenderer(asset, ctx)
            rs = [src, src.Instance()]
            rs.append(rs[1].Instance())
            for r in rs:
                frame(r, cam)
            for i in perm:
                rs[i].Dispose()
            ctx.sync()
            check.ResetOrder()
            assert np.array_equal(bits(frame(check, cam)), bits(want)), "after destroying in order %s" % (perm,)
            ctx.sync()
    finally:
        check.Dispose()


# ---- 5. other entry points ------------------------------------------------------------------------------------------------
def test_packed_device_asset_as_source(g, ctx):
    """gs_pack_asset's asset_out as a source: its instance draws what an upload of the packed blobs draws."""
    from unitygaussiansplatting_b200.pack import pack_asset
    splats = g.generate_input_splats(g.SCENE_CLUSTERED, 30000, 0x5EED0A51)
    host, src = pack_asset(splats, "Medium", context=ctx, keep_on_device=True)
    inst = src.Instance()
    twin = g.GaussianSplatRenderer(host, ctx)
    try:
        for w in BLOBS:
            assert ptr(inst, w) == ptr(src, w)
        for f in range(3):
            cam = orbit(g, f)
            want = frame(twin, cam)
            assert want[..., 3].any()
            assert np.array_equal(bits(frame(inst, cam)), bits(want)), "frame %d" % f
            assert_same(inst, twin, "frame %d" % f)
    finally:
        for r in (src, inst, twin):
            r.Dispose()


def test_export_of_an_instance_equals_the_source(g, ctx):
    asset = asset_of(g, "clustered_4k_veryhigh")
    src = g.GaussianSplatRenderer(asset, ctx)
    inst = src.Instance()
    try:
        cut = [(np.linalg.inv(g.trs(scale=(1.5, 1.5, 1.5))), 0)]
        src.m_Cutouts = inst.m_Cutouts = cut
        want = src.EditExportData()
        assert (want[:, 3] == 1).any() and (want[:, 3] == 0).any()
        assert np.array_equal(inst.EditExportData().view(np.uint32), want.view(np.uint32))
    finally:
        inst.Dispose()
        src.Dispose()


def test_unity_frame_objects_event_over_instances_equals_the_direct_call(g, ctx):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    asset = asset_of(g, "bench_200k_medium")
    src = g.GaussianSplatRenderer(asset, ctx)
    ev_rs = [src, src.Instance(), src.Instance()]
    direct = [g.GaussianSplatRenderer(asset, ctx) for _ in range(3)]
    for i, (p, q) in enumerate(zip(ev_rs, direct)):
        mixed_setup(i, p)
        mixed_setup(i, q)
    try:
        for f in range(3):
            cam = orbit(g, f)
            want = rt_of(cam)
            call_frame(g, ctx, direct, cam, 0, want, None)
            got = rt_of(cam)
            assets, fps, ds, keep = frame_args(g, [(cam, r, None) for r in ev_rs], sort=next_sort)
            ev = N.GsUnityFrameObjectsEvent(ctx=ctx.handle.value, object_count=3, assets=C.addressof(assets), fps=C.addressof(fps),
                                            do_sort=C.addressof(ds), options=opt(N, 0), status=N.GS_ERR_NOT_READY, has_rt=1,
                                            rt=_image(got, cam.pixelWidth, cam.pixelHeight))
            assert N.unity_event(N.GS_UNITY_EVENT_FRAME_OBJECTS, ev) == 0
            assert want[..., 3].any()
            assert np.array_equal(bits(got), bits(want)), "frame %d" % f
            for k, (p, q) in enumerate(zip(ev_rs, direct)):
                assert_same(p, q, "frame %d object %d" % (f, k))
    finally:
        for r in ev_rs + direct:
            r.Dispose()


# ---- 6. group -------------------------------------------------------------------------------------------------------------
def test_group_member_asset_and_its_instance(g, ctx):
    """An emulated group of 2 draws two objects -- the group's asset and an instance of it -- exactly as the same group with
    two gs_group_asset_upload objects does."""
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    asset = asset_of(g, "bench_200k_medium")
    setups = [dict(localToWorldMatrix=g.trs(position=(-0.7, 0.0, 1.0)).astype(np.float32), m_SortNthFrame=1),
              dict(localToWorldMatrix=g.trs(position=(0.8, 0.1, 1.6)).astype(np.float32), m_SortNthFrame=2, m_SHOrder=2)]
    grps = [GaussianSplatGroup.create(asset, [0, 0], emulate=True) for _ in range(2)]
    shared = [grps[0], grps[0].add_instance(grps[0])]
    uploads = [grps[1], grps[1].add_object(asset)]
    for objs in (shared, uploads):
        for o, kw in zip(objs, setups):
            knobs(o, **kw)
    try:
        for i in range(2):
            for w in BLOBS:
                assert ptr_of(shared[1]._assets[i], w) == ptr_of(shared[0]._assets[i], w)
        for f in range(4):
            cam = camera(g, 320, 200, pos=(0.1 * f - 0.2, 0.5, -6.0 + 0.3 * f))
            out = []
            for grp, objs in zip(grps, (shared, uploads)):
                rts = [rt_of(cam) for _ in range(2)]
                grp.SortAndRenderSplatsMulti(objs, cam, rts=rts)
                grp.sync()
                out.append(rts)
            for i in range(2):
                assert out[1][i][..., 3].any()
                assert np.array_equal(bits(out[0][i]), bits(out[1][i])), "frame %d member %d" % (f, i)
                for k in range(2):
                    assert np.array_equal(shared[k].readback_order(i), uploads[k].readback_order(i)), "frame %d member %d object %d" % (f, i, k)
    finally:
        for grp in grps:
            grp.close()


# ---- 7. rejections --------------------------------------------------------------------------------------------------------
def test_null_arguments_are_rejected(g, ctx):
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    src = g.GaussianSplatRenderer(asset_of(g, "lattice_1k_medium"), ctx)
    try:
        h = C.c_void_p(1234)
        assert lib.gs_asset_instance(None, C.byref(h)) == INVALID
        assert not h.value, "*out must be NULL after a refused call"
        assert lib.gs_asset_instance(src._asset, None) == INVALID
        assert b"null" in lib.gs_last_error(ctx.handle)
        want = frame(src, orbit(g, 0))   # the context is still usable
        assert want[..., 3].any()
    finally:
        src.Dispose()
