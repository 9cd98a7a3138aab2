"""The fused frame at the camera poses XR and walk-through users render: cameras inside the splats, off-axis XR eye frusta,
roll, wide and narrow fields of view, portrait screens and one-bin strips, mirrored, oblique and orthographic projections,
and splats at the camera plane.

Nearly all of the fused frame's work skipping is derived from the camera (make_frame_consts' extentK, the chunk-box cull, the
far_off cull, the covariance cull, splat_footprint's cut-offs, a group member's row culls).  A bound that holds only for a
centred frustum, or only for a camera outside the scene, drops splats without notice.  The staged path (gs_calc_view +
gs_render) culls nothing, so at every pose the fused frame, the staged path and the oracle must agree bit for bit.  Each pose
also asserts what makes it the pose it claims to be (splats behind the camera, chunk boxes straddling the camera plane,
off-axis terms, roll, aspect), so a later change to the fixture cannot quietly turn it back into the default camera."""
import dataclasses

import numpy as np
import pytest

from images import SharedArray, bits, ca, to_device, to_host  # noqa: F401
from util import POSES, near_plane_camera, near_plane_scene, splat_records, xr_eye

pytestmark = pytest.mark.gpu

N, SEED = 40000, 0x5EED0E01
QUALITIES = ("Medium", "VeryHigh")     # chunked: the chunk-box cull decides first; unchunked: the per-splat culls alone


@pytest.fixture(scope="module")
def assets(g):
    return {q: g.synthetic_asset(g.SCENE_CLUSTERED, N, SEED, q) for q in QUALITIES}


def frame_vs_oracle(g, O, ctx, asset, cam, blend=0, selected=None, depth=None, localToWorld=None):
    """The fused frame, the staged path and the oracle at `cam`: keys, order, SplatViewData and the render target bit for bit.
    Returns (oracle frame, bin-list entries of the fused frame)."""
    r = g.GaussianSplatRenderer(asset, ctx)
    r.blend_mode = blend
    r.m_SelectedBits = selected
    r.sceneDepth = depth
    if localToWorld is not None:
        r.localToWorldMatrix = np.asarray(localToWorld, np.float32)
    try:
        return _compare(g, O, ctx, r, asset, cam, blend, selected, depth)
    finally:
        r.Dispose()   # also when a comparison fails: nothing is left for a finaliser


def _compare(g, O, ctx, r, asset, cam, blend, selected, depth):
    n = asset.splatCount
    rt = np.zeros((cam.pixelHeight, cam.pixelWidth, 4), np.float32 if blend == 1 else np.float16)
    ctx.set_timing(True)
    try:
        r.SortAndRenderSplats(cam, rt=rt)
        entries = int(ctx.stage_times().tile_entries)
    finally:
        ctx.set_timing(False)
    fp, _keep = g.make_frame_params(cam, r.localToWorldMatrix, splat_count=n, selected_bits=selected, scene_depth=depth)
    ref = O.frame(asset, fp, blend_mode=blend, threads=O.max_threads())
    assert np.array_equal(r.readback_keys(), ref["keys"]), "sorted distance keys differ"
    assert np.array_equal(r.readback_order(), ref["order"]), "sorted splat indices differ"
    bad = np.nonzero(rt.astype(np.float32).reshape(-1, 4) != ref["rt"].reshape(-1, 4))[0]
    assert bad.size == 0, "render target differs at %d pixels, first %s" % (bad.size, [divmod(int(i), cam.pixelWidth)[::-1] for i in bad[:4]])
    r.CalcViewData(cam)
    view = r.readback_view()
    # a splat whose view depth is 0 gets NaN screen axes on both sides: the device writes its canonical NaN, the host the
    # payload x86 propagates, and splat_footprint drops the splat either way.  Every other word is compared bit for bit.
    both_nan = np.zeros(view.shape, bool)
    both_nan[:, 4:8] = np.isnan(view[:, 4:8].view(np.float32)) & np.isnan(ref["view"][:, 4:8].view(np.float32))
    bad = np.nonzero(((view != ref["view"]) & ~both_nan).any(axis=1))[0]
    assert bad.size == 0, "SplatViewData differs for %d splats, first %s" % (bad.size, bad[:5])
    rt2 = np.zeros_like(rt)
    r.DrawSplats(cam, rt2)
    assert np.array_equal(bits(rt2), bits(rt)), "the staged draw differs from the fused frame"
    return ref, entries


# ---- what each pose is ---------------------------------------------------------------------------------------------------------
def chunk_boxes(asset):
    """(lo, hi) corners of every chunk's position box (SplatChunkInfo floats 4..9)."""
    ch = asset.chunkData.view(np.float32).reshape(-1, 16)
    return ch[:, [4, 6, 8]].astype(np.float64), ch[:, [5, 7, 9]].astype(np.float64)


def pose_stats(cam, asset, ref):
    """Numbers that say what a pose exercises, from the oracle's frame and the camera."""
    P = cam.gpuProjectionMatrix(True).astype(np.float64)
    V = cam.worldToCameraMatrix.astype(np.float64)
    w = ref["view"][:, 3].view(np.float32)
    s = {"behind": float((w <= 0).mean()), "p02": P[0, 2], "p12": P[1, 2], "p00": P[0, 0], "p11": P[1, 1],
         "drawn": float((ref["rt"][..., 3] > 0).mean())}
    if asset.chunkData is not None:
        lo, hi = chunk_boxes(asset)
        corners = np.stack([np.where([(k >> a) & 1 for a in range(3)], hi, lo) for k in range(8)], 1)
        tz = corners @ V[2, :3] + V[2, 3]
        s["straddle"] = int(((tz < 0).any(1) & (tz > 0).any(1)).sum())
        s["contain"] = int(((lo <= cam.position) & (cam.position <= hi)).all(1).sum())
    return s


def check_pose(g, name, cam, s):
    """The pose is what its name claims."""
    P, fwd = cam.gpuProjectionMatrix(True).astype(np.float64), np.asarray(cam.rotation)[:, 2]
    assert s["drawn"] > 0.3, "the frame draws (almost) nothing"
    if name.startswith("inside") or name.startswith("xr"):
        assert s["behind"] > 0.3, "a camera inside the cloud has a large share of splats behind it"
        if "contain" in s:
            assert s["contain"] >= 1 and s["straddle"] >= 20, "chunk boxes around and across the camera plane"
    if name == "inside-back":
        assert fwd[2] < -0.99
    if name.startswith("xr"):
        assert abs(P[0, 2]) > 0.2 and abs(P[1, 2]) > 0.02, "an XR eye's frustum is off-axis"
        assert cam.pixelWidth == cam.pixelHeight
        across = np.degrees(np.arctan((1 + abs(P[0, 2])) / P[0, 0]) + np.arctan((1 - abs(P[0, 2])) / P[0, 0]))
        assert 90 < across < 105
    else:
        assert P[0, 2] == 0 and P[1, 2] == 0
    if name.startswith("roll"):
        base = g.look_rotation(fwd)
        deg = float(name.split("-")[1])
        assert np.isclose(np.degrees(np.arctan2(base[:, 1] @ cam.rotation[:, 0], base[:, 0] @ cam.rotation[:, 0])), deg, atol=1e-6) or \
            deg == 180 and np.isclose(base[:, 0] @ cam.rotation[:, 0], -1.0)
    if name == "fov-110":
        assert np.isclose(np.degrees(2 * np.arctan(1 / abs(P[1, 1]))), 110.0, atol=1e-3)
    if name == "fov-3":
        assert cam.pixelWidth * P[0, 0] / 2 > 4000, "a narrow field of view has a large focal length (and extentK)"
    if name == "portrait":
        assert cam.pixelHeight > cam.pixelWidth
    if name.startswith("strip"):
        assert min(cam.pixelWidth, cam.pixelHeight) == 64 and max(cam.pixelWidth, cam.pixelHeight) == 1024   # one bin row / column
        assert abs(np.log2(abs(P[0, 0] / P[1, 1]))) == 4, "tanFovY == tanFovX is 16 times off the truth"
    if name == "mirrored":
        assert P[0, 0] < 0
    if name == "ortho-inside":
        # clip.w == 1: chunk boxes across the camera plane have every corner in front (w > 0), so the chunk cull's reach
        # must come from the view depth's sign change, not from the w ballot
        assert np.array_equal(P[3], [0, 0, 0, 1]) and s["behind"] == 0
        if "contain" in s:
            assert s["contain"] >= 1 and s["straddle"] >= 20
    if name == "oblique":
        sym = g.Camera(**{f.name: getattr(cam, f.name) for f in dataclasses.fields(g.Camera)}).gpuProjectionMatrix(True)
        assert not np.allclose(P[2], sym[2]) and np.array_equal(P[[0, 1, 3]], sym[[0, 1, 3]]), "only clip.z changes"


def wall(cam, dist, frac=0.6):
    """A depth buffer holding a wall at view distance `dist` over the left `frac` of the screen."""
    P = cam.gpuProjectionMatrix(True).astype(np.float64)
    clip = P @ np.array([0.0, 0.0, -dist, 1.0])
    depth = np.zeros((cam.pixelHeight, cam.pixelWidth), np.float32)
    depth[:, :int(cam.pixelWidth * frac)] = np.float32(clip[2] / clip[3])
    return depth


# ---- 1. every pose on a chunked and an unchunked asset -------------------------------------------------------------------------
@pytest.mark.parametrize("quality", QUALITIES)
@pytest.mark.parametrize("pose", list(POSES))
def test_pose_is_bit_exact(g, O, ctx, assets, pose, quality):
    cam = POSES[pose](g)
    asset = assets[quality]
    depth = wall(cam, 4.0) if pose == "oblique" else None     # an oblique near plane changes clip.z only: depth-test it
    ref, entries = frame_vs_oracle(g, O, ctx, asset, cam, depth=depth)
    s = pose_stats(cam, asset, ref)
    check_pose(g, pose, cam, s)
    assert entries > 0
    if depth is not None:
        fp, _keep = g.make_frame_params(cam, splat_count=asset.splatCount)
        assert not np.array_equal(O.frame(asset, fp, threads=O.max_threads())["rt"], ref["rt"]), "the depth buffer hides nothing"
    print("pose %-12s %-8s %4dx%-4d behind %.3f straddle %s contain %s P02 %+.3f P12 %+.3f p00 %+.3f entries %d drawn %.3f" % (
        pose, quality, cam.pixelWidth, cam.pixelHeight, s["behind"], s.get("straddle", "-"), s.get("contain", "-"), s["p02"],
        s["p12"], s["p00"], entries, s["drawn"]))


# ---- 2. XR eyes: a stereo camera run into two layers, and per-eye depth layers ------------------------------------------------
def test_xr_stereo_run_on_layers_is_the_eye_loop(g, ctx, assets, ca):
    W = H = 256
    eyes = [xr_eye(g, e, W, H) for e in range(2)]
    mats = [np.eye(4, dtype=np.float32), g.trs(position=(-0.6, 0.1, 0.4)).astype(np.float32)]

    def renderers():
        rs = [g.GaussianSplatRenderer(assets[q], ctx) for q in QUALITIES]
        for r, m in zip(rs, mats):
            r.localToWorldMatrix = m
        return rs

    loop = renderers()
    want = []
    for cam in eyes:
        rt = to_device(np.zeros((H, W, 4), np.float16))
        assert len(g.SortAndRenderSplatsMulti(loop, cam, rt)) == 2
        want.append(to_host(ctx, rt))
    want_orders = [r.readback_order() for r in loop]
    assert all(x.any() for x in want) and not np.array_equal(want[0], want[1])
    call = renderers()
    A = SharedArray(g, ca, W, H, 3)
    actives = g.SortAndRenderCameras(call, eyes, [A.view(layer=0), A.view(layer=1)])
    assert g.renderer.cameras_in_one_call(actives)
    A.check(ctx, [(e, 0, 0, want[e]) for e in range(2)], "eyes")
    for r, o in zip(call, want_orders):
        assert np.array_equal(r.readback_order(), o)
    for r in loop + call:
        r.Dispose()


def test_xr_eyes_with_depth_layers_equal_the_oracle(g, O, ctx, assets, ca):
    W = H = 256
    asset = assets["Medium"]
    eyes = [xr_eye(g, e, W, H) for e in range(2)]
    depths = [wall(eyes[0], 2.5), np.ascontiguousarray(wall(eyes[1], 2.5)[:, ::-1])]
    da = ca.array(W, H, 2, np.float32, 1, fill=np.stack(depths))
    for e, cam in enumerate(eyes):
        r = g.GaussianSplatRenderer(asset, ctx)
        r.sceneDepth = g.CudaArrayDepth(da, W, H, layer=e)
        rt = np.zeros((H, W, 4), np.float16)
        r.SortAndRenderSplats(cam, rt=rt)
        fp, _keep = g.make_frame_params(cam, splat_count=asset.splatCount, scene_depth=depths[e])
        ref = O.frame(asset, fp, threads=O.max_threads())
        free_fp, _k2 = g.make_frame_params(cam, splat_count=asset.splatCount)
        assert not np.array_equal(O.frame(asset, free_fp, threads=O.max_threads())["rt"], ref["rt"]), "the wall hides nothing"
        assert np.array_equal(rt.astype(np.float32), ref["rt"]), "eye %d differs from the oracle" % e
        assert np.array_equal(r.readback_order(), ref["order"])
        r.Dispose()


# ---- 3. fp32 blending and an edit selection; an emulated group --------------------------------------------------------------
@pytest.mark.parametrize("pose", ["xr-left", "inside-near"])
def test_fp32_blend_and_selection_at_pose(g, O, ctx, assets, pose):
    cam = POSES[pose](g)
    asset = assets["Medium"]
    sel = np.zeros((asset.splatCount + 31) // 32, np.uint32)
    sel[::3] = 0x33333333
    frame_vs_oracle(g, O, ctx, asset, cam, blend=1)
    frame_vs_oracle(g, O, ctx, asset, cam, selected=sel)


@pytest.mark.parametrize("pose", ["inside-z", "xr-right"])
def test_emulated_group_at_pose_equals_one_gpu(g, ctx, assets, pose):
    """Each member of a group of 3 culls splats against its own pixel rows with the splat's projected centre: off-axis and
    inside-the-scene centres must land on the same rows as on one GPU."""
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    cam = POSES[pose](g)
    for q in QUALITIES:
        r = g.GaussianSplatRenderer(assets[q], ctx)
        rt = np.zeros((cam.pixelHeight, cam.pixelWidth, 4), np.float16)
        r.SortAndRenderSplats(cam, rt=rt)
        r.Dispose()
        assert rt.any()
        grp = GaussianSplatGroup.create(assets[q], [0, 0, 0], emulate=True)
        try:
            rts = [np.zeros_like(rt) for _ in range(3)]
            grp.SortAndRenderSplats(cam, rts=rts)
            for i in range(3):
                assert np.array_equal(bits(rts[i]), bits(rt)), "%s member %d" % (q, i)
        finally:
            grp.close()


# ---- 4. splats at the camera plane ----------------------------------------------------------------------------------------------
def test_splats_at_the_camera_plane(g, O, ctx):
    cam = near_plane_camera(g)
    assert np.array_equal(cam.worldToCameraMatrix, np.diag([1.0, 1.0, -1.0, 1.0]).astype(np.float32)), "view depth is world z exactly"
    asset = near_plane_scene(g, cam)
    ref, _entries = frame_vs_oracle(g, O, ctx, asset, cam)
    w = ref["view"][:, 3].view(np.float32)
    pos = np.asarray(asset.posData).view(np.float32)[:3 * asset.splatCount].reshape(-1, 3)
    assert np.array_equal(w > 0, pos[:, 2] > 0) and (w == 0).sum() == (pos[:, 2] == 0).sum() > 0
    front = w > 0
    cx = np.abs((ref["view"][front, 0].view(np.float32) / w[front] * 0.5 + 0.5) * cam.pixelWidth)
    assert (cx > 1e7).any() and ((cx < 1e7) & (cx > 9e6)).any(), "centres on both sides of the 1e7 px cut-off"
    assert ref["rt"][..., 3].any(), "the splats just inside the screen draw"

    # w > 0 while the view depth the fused frame's culls use rounds to 0: an object far along z, its splats brought back
    # into view by positions of the opposite sign.  tz = (-1) pz + round(cz - T) = 0 exactly, while clip.w = round(pz + T) - cz
    # = 3: the far_off reach and the covariance divide by tz = 0
    T, cz = 100000008.0, 5.0
    cam2 = dataclasses.replace(cam, position=np.array([0.0, 0.0, cz]))
    rec = splat_records(np.array([[0.0, 0.0, -1e8], [2e-3, -1e-3, -1e8], [0.5, 0.2, 3.0 - T]], np.float32), (0.05, 0.02, 0.01), 0.8,
                        quat=(0.2, 0.1, 0.4, 0.9))
    one = g.create_asset(rec, "VeryHigh")
    ref, _ = frame_vs_oracle(g, O, ctx, one, cam2, localToWorld=g.trs((0.0, 0.0, T)))
    f32 = np.float32
    m11 = f32(f32(-f32(T)) + f32(cz))                            # make_frame_consts: (V o2w)[2][3], summed left to right
    tzq = f32(f32(-1.0) * f32(-1e8) + m11)
    w = ref["view"][:, 3].view(np.float32)
    assert tzq == 0.0 and (w == 3.0).sum() == 2
