#!/usr/bin/env python
"""What the reference's own shader code computes on the cases of tests/test_reference_hlsl.py and
tests/test_zz_reference_hlsl_gpu.py, stored as tests/golden/ref_hlsl_*.npz so that both compare with the reference wherever
they run.

The compiled reference is oracle/_ref/libref_hlsl.so, built from the reference's shader source by
oracle/refhlsl/build_ref_hlsl.py.  `reference(name)` returns its output for case `name`: computed on the spot when that
library is present, otherwise read from the fixture.  The scene-sized cases are stored for a fixed seeded sample of their
splats (the whole scenes would make fixtures of ~0.7 MB each); `idx` names the sampled splats (or sorted positions) and is
every one of them when the library computes the case.
Run from the repo root:  python tests/golden/make_ref_hlsl_golden.py [case ...]   (every case when none is named)
"""
import dataclasses
import hashlib
import sys
from pathlib import Path

import numpy as np

GOLD = Path(__file__).resolve().parent
ROOT = GOLD.parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from util import FORMAT_CASES  # noqa: E402

# ---- the GPU comparison: CSCalcViewData + CSCalcDistances with the renderer's defaults (ref_hlsl_<quality>.npz) ----------
QUALITIES = ("Medium", "VeryHigh")
N, SEED, WIDTH, HEIGHT = 20000, 0x5EED0091, 320, 240
SAMPLE, SAMPLE_SEED = 2048, 0x5EED0095

# ---- the oracle comparisons (ref_hlsl_<case>.npz) --------------------------------------------------------------------------
# "custom-<name>" is the format case <name> of tests/util.py FORMAT_CASES; BC7 colour is left out of the view cases because
# its block decode belongs to the texture unit, not to the reference's code (tests/golden/bc7_blocks.npz covers it)
VIEW_QUALITIES = ("Medium", "VeryHigh", "High", "Low", "custom-f16sh", "custom-norm6pos") + \
    tuple("custom-" + c.name for c in FORMAT_CASES if c.formats[2] != 3)
VIEW_SAMPLE = 512
KEY_QUALITIES = ("Medium", "VeryHigh", "custom-norm6pos-f16sh", "custom-f32pos-bc7-f16sh")   # + Norm6, chunked Float32 positions
KEY_N, KEY_SAMPLE = 30000, 4096
# "pose-<name>": the camera pose <name> of tests/util.py POSES (or "near", the near-plane scene) in place of the default camera
VIEW_POSES = ("pose-inside-back", "pose-xr-left", "pose-mirrored", "pose-near")
KEY_POSES = ("pose-inside-back",)
EXPORT_N, EXPORT_SAMPLE = 3000, 128
DRAW_W, DRAW_H = 200, 150


def asset_digest(asset):
    blobs = [asset.posData, asset.otherData, asset.colorData, asset.shData] + ([asset.chunkData] if asset.chunkData is not None else [])
    return np.frombuffer(hashlib.sha256(b"".join(b.tobytes() for b in blobs)).digest(), np.uint8)


def scene(quality):
    """(asset, camera, frame params, asset digest) of one GPU case; the renderer's defaults (identity transform, SH order 3)."""
    import unitygaussiansplatting_b200 as g
    from util import camera
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, N, SEED, quality)
    cam = camera(g, WIDTH, HEIGHT)
    fp, keep = g.make_frame_params(cam)
    return asset, cam, (fp, keep), asset_digest(asset)


def sample_ids(n=N, k=SAMPLE, seed=SAMPLE_SEED):
    return np.sort(np.random.default_rng(seed).choice(n, k, replace=False)).astype(np.uint32)


def pose_camera(g, pose):
    from util import POSES, near_plane_camera
    return near_plane_camera(g) if pose == "near" else POSES[pose](g)


def view_case(quality):
    """(asset, (fp, keep)): object transform, splat / opacity scale, a cutout box and deleted bits on a clustered scene.
    "pose-<name>": the Medium scene seen from that camera pose; "pose-near": the near-plane scene under an identity transform,
    so that its view depths stay the exact ones it was built with."""
    import unitygaussiansplatting_b200 as g
    from util import camera, case_asset, format_case, near_plane_scene, palette_backed
    cam = camera(g, 320, 240)
    if quality.startswith("pose-"):
        cam = pose_camera(g, quality[len("pose-"):])
    if quality == "pose-near":
        asset = near_plane_scene(g, cam)
    elif quality.startswith("pose-"):
        asset = g.synthetic_asset(g.SCENE_CLUSTERED, N, 0x5EED0091, "Medium")
    elif quality in ("custom-f16sh", "custom-norm6pos"):     # Float16 SH; Norm6 positions with Norm16 scale
        fmts = {"custom-f16sh": (g.VectorFormat.Norm16, g.VectorFormat.Norm6, g.ColorFormat.Float16x4, g.SHFormat.Float16),
                "custom-norm6pos": (g.VectorFormat.Norm6, g.VectorFormat.Norm16, g.ColorFormat.Float32x4, g.SHFormat.Norm11)}[quality]
        asset = g.create_asset(g.generate_input_splats(g.SCENE_CLUSTERED, N, 0x5EED0091), formats=fmts)
    elif quality.startswith("custom-"):
        # a clustered palette padded to the 65536 entries a u16 index can name, as the device backs it
        asset = palette_backed(case_asset(g, format_case(quality[len("custom-"):]), N, 0x5EED0091))
    else:
        asset = g.synthetic_asset(g.SCENE_CLUSTERED, N, 0x5EED0091, quality)
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = np.array([[0.8, -0.6, 0.0], [0.6, 0.8, 0.0], [0.0, 0.0, 1.0]], np.float32) * 1.1
    T[:3, 3] = (0.3, -0.1, 0.2)
    if quality == "pose-near":
        T = np.eye(4, dtype=np.float32)
    box = np.diag([1 / 9.0, 1 / 9.0, 1 / 9.0, 1.0]).astype(np.float32)
    deleted = np.zeros((N + 31) // 32, np.uint32)
    deleted[3] = 0xF0F0F0F0
    return asset, g.make_frame_params(cam, localToWorld=T, splat_scale=0.9, opacity_scale=1.3, sh_order=3,
                                      cutouts=[(box, 1)], deleted_bits=deleted, splat_count=asset.splatCount)


def key_case(quality):
    """(asset, (fp, keep), order): CSCalcDistances through a random permutation ("pose-<name>": the Medium scene from that pose)."""
    import unitygaussiansplatting_b200 as g
    from util import camera, case_asset, format_case
    if quality.startswith("pose-"):
        asset = g.synthetic_asset(g.SCENE_CLUSTERED, KEY_N, 0x5EED0092, "Medium")
        order = np.random.default_rng(1).permutation(KEY_N).astype(np.uint32)
        return asset, g.make_frame_params(pose_camera(g, quality[len("pose-"):])), order
    if quality.startswith("custom-"):
        asset = case_asset(g, format_case(quality[len("custom-"):]), KEY_N, 0x5EED0092)
    else:
        asset = g.synthetic_asset(g.SCENE_CLUSTERED, KEY_N, 0x5EED0092, quality)
    order = np.random.default_rng(1).permutation(KEY_N).astype(np.uint32)
    return asset, g.make_frame_params(camera(g, 320, 240)), order


def export_case():
    """(asset, plain (fp, keep), transformed (fp, keep), T, rotation, scale) of the CSExportData comparison."""
    import unitygaussiansplatting_b200 as g
    from unitygaussiansplatting_b200.renderer import decompose_trs
    from util import camera
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, EXPORT_N, 0x5EED0093, "VeryHigh")
    ang = np.radians(50.0)
    Rm = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]]) @ \
        np.array([[1, 0, 0], [0, np.cos(0.4), -np.sin(0.4)], [0, np.sin(0.4), np.cos(0.4)]])
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = (Rm * 1.25).astype(np.float32)
    T[:3, 3] = (0.5, 0.25, -0.75)
    q, s = decompose_trs(T)
    return asset, g.make_frame_params(camera(g, 64, 64)), g.make_frame_params(camera(g, 64, 64), localToWorld=T), T, q, s


def draw_case(selected):
    """(view, order, W, H): the oracle's SplatViewData of one rotated, anisotropic splat (+ 40 far-away ones when `selected`)."""
    import unitygaussiansplatting_b200 as g
    from oracle import gs_oracle_py as O
    from util import camera, one_splat
    cam = camera(g, DRAW_W, DRAW_H, fov=50.0, pos=(0.1, 0.0, -3.0))
    asset = one_splat(g, pos=(0.2, -0.1, 0.3), scale=(0.25, 0.08, 0.05), quat=(0.3, 0.5, -0.2, 0.78),
                      opacity=0.02 if selected else 0.65, dc0=(0.7, 0.5, 0.9), n_pad=40 if selected else 0)
    fp, _keep = g.make_frame_params(cam, sh_order=0)
    return O.calc_view(asset, fp), np.arange(asset.splatCount, dtype=np.uint32), DRAW_W, DRAW_H


def quad_map(clip, qpos, W, H):
    """(corner pixels, A) with [x y 1] @ A = quad coordinates: the rasteriser's affine interpolation over the quad."""
    px = np.stack([(clip[:, 0] / clip[:, 3] * 0.5 + 0.5) * W, (0.5 - 0.5 * clip[:, 1] / clip[:, 3]) * H], 1).astype(np.float64)
    return px, np.linalg.solve(np.column_stack([px[:3], np.ones(3)]), qpos[:3].astype(np.float64))


def rotation_quats():
    rng = np.random.default_rng(3)
    out = []
    for _ in range(300):
        q = rng.standard_normal(4).astype(np.float32)
        out.append(q / np.linalg.norm(q))
    return np.array(out, np.float32)


CASES = (["gpu_" + q.lower() for q in QUALITIES] + ["view_" + q.lower() for q in VIEW_QUALITIES + VIEW_POSES] +
         ["keys_" + q.lower() for q in KEY_QUALITIES + KEY_POSES] + ["export", "draw", "draw_selected", "rotation"])
_NAMES = {q.lower(): q for q in VIEW_QUALITIES + KEY_QUALITIES + VIEW_POSES + KEY_POSES}


def compute(name):
    """Case `name` computed by the compiled reference (which must be present): every splat, pixel or quaternion of it."""
    from oracle import gs_oracle_py as O
    kind, _, q = name.partition("_")
    if kind == "gpu":
        asset, _cam, (fp, _keep), digest = scene(_NAMES[q])
        return {"idx": np.arange(N, dtype=np.uint32), "view": O.ref_calc_view(asset, fp),
                "keys": O.ref_calc_distances(asset, fp, np.arange(N, dtype=np.uint32)), "asset_sha256": digest}
    if kind == "view":
        asset, (fp, _keep) = view_case(_NAMES[q])
        return {"idx": np.arange(asset.splatCount, dtype=np.uint32), "view": O.ref_calc_view(asset, fp), "asset_sha256": asset_digest(asset)}
    if kind == "keys":
        asset, (fp, _keep), order = key_case(_NAMES[q])
        # CSCalcDistances reads positions only, and the compiled reference refuses a BC7 asset as a whole: call it Norm8x4
        pos_only = dataclasses.replace(asset, colorFormat=2) if asset.colorFormat == 3 else asset
        return {"idx": np.arange(KEY_N, dtype=np.uint32), "keys": O.ref_calc_distances(pos_only, fp, order), "asset_sha256": asset_digest(asset)}
    if name == "export":
        asset, (fp, _k), (fpT, _k2), _T, rq, rs = export_case()
        return {"idx": np.arange(EXPORT_N, dtype=np.uint32), "plain": O.ref_export(asset, fp),
                "baked": O.ref_export(asset, fpT, bake=True, rotation=rq, scale=rs), "asset_sha256": asset_digest(asset)}
    if name in ("draw", "draw_selected"):
        view, order, W, H = draw_case(name == "draw_selected")
        clip, qpos, col = O.ref_vert(view, order, 0, W, H)
        out = {"view": view, "clip": clip, "qpos": qpos}
        if name == "draw_selected":
            bits = np.array([1, 0], np.uint32)                          # splat 0 selected, the padding splats not
            col = O.ref_vert_selected(view, order, 0, W, H, bits)
            out["col_other"] = O.ref_vert_selected(view, order, 1, W, H, bits)
        out["col"] = col
        # the pixel shader at every pixel centre near the quad
        _px, A = quad_map(clip, qpos, W, H)
        frag, disc = np.zeros((H, W, 4), np.float32), np.zeros((H, W), bool)
        for y in range(H):
            for x in range(W):
                qx, qy = np.array([x + 0.5, y + 0.5, 1.0]) @ A
                if abs(qx) <= 2.3 and abs(qy) <= 2.3:
                    frag[y, x], disc[y, x] = O.ref_frag(col, float(qx), float(qy))
        out["frag"], out["discarded"] = frag, disc
        return out
    if name == "rotation":
        L = O.ref_hlsl()
        quats = rotation_quats()
        packed, enc, back = np.zeros((len(quats), 4), np.float32), np.zeros(len(quats), np.uint32), np.zeros((len(quats), 4), np.float32)
        for i, qq in enumerate(quats):
            enc[i] = L.refhlsl_pack_rotation(np.ascontiguousarray(qq).ctypes.data, packed[i].ctypes.data)
            L.refhlsl_decode_rotation(int(enc[i]), back[i].ctypes.data)
        return {"packed": packed, "enc": enc, "decoded": back}
    raise KeyError(name)


def stored(name):
    """What the fixture keeps of a computed case: a seeded sample of the scene-sized arrays, everything else whole."""
    d = compute(name)
    kind = name.partition("_")[0]
    k = {"gpu": SAMPLE, "view": VIEW_SAMPLE, "keys": KEY_SAMPLE, "export": EXPORT_SAMPLE}.get(kind)
    if k is None or k >= len(d["idx"]):
        return d
    idx = sample_ids(len(d["idx"]), k, SAMPLE_SEED if kind == "gpu" else SAMPLE_SEED + 1)
    return {key: (v if key == "asset_sha256" else v[idx]) for key, v in d.items()}


def fixture(name):
    return GOLD / ("ref_hlsl_%s.npz" % (name[4:] if name.startswith("gpu_") else name))


def reference(name):
    """Case `name`: computed by the compiled reference when it is present, else read from its fixture."""
    from oracle import gs_oracle_py as O
    if O.ref_hlsl() is not None:
        return compute(name)
    with np.load(fixture(name)) as f:
        return {k: f[k] for k in f.files}


if __name__ == "__main__":
    from oracle import gs_oracle_py as O
    if O.ref_hlsl() is None:
        raise SystemExit("oracle/_ref/libref_hlsl.so is not built")
    unknown = sorted(set(sys.argv[1:]) - set(CASES))
    if unknown:
        raise SystemExit("unknown case(s) %s; the cases are %s" % (unknown, CASES))
    for name in sys.argv[1:] or CASES:
        data = stored(name)
        np.savez_compressed(fixture(name), **data)
        print(name, {k: v.shape for k, v in data.items()})
