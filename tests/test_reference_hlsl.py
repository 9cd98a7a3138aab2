"""The oracle against THE REFERENCE'S OWN SHADER CODE.

oracle/_ref/libref_hlsl.so is package/Shaders/{GaussianSplatting.hlsl, SplatUtilities.compute, SphericalHarmonics.hlsl,
RenderGaussianSplats.shader} themselves -- syntactically rewritten to C++ spelling and compiled with g++ against a shim of
HLSL's types and intrinsics (oracle/refhlsl/).  Expressions, constants, operation order and branches are the reference's;
scalar arithmetic is IEEE float32 without contraction.  Where that library is built the reference's outputs are computed
on the spot; elsewhere they are read from tests/golden/ref_hlsl_*.npz (tests/golden/make_ref_hlsl_golden.py), which keep a
fixed seeded sample of the splats of the scene-sized cases.  The oracle (and the CUDA path, bit-identical to it) evaluates
the same formulas under its own arithmetic contract (explicit fmaf chains, reciprocal constants), so the two agree to float
rounding, not to the bit: tolerances below are a few ulp, scaled by conditioning where a formula cancels."""
import sys
from pathlib import Path

import numpy as np
import pytest

from util import screen_cov, unsortable, view_fields

sys.path.insert(0, str(Path(__file__).parent / "golden"))
import make_ref_hlsl_golden as M  # noqa: E402


def _same_asset(asset, want):
    assert np.array_equal(M.asset_digest(asset), want["asset_sha256"]), "the scene is no longer the one the reference output is for"


@pytest.mark.parametrize("quality", M.VIEW_QUALITIES + M.VIEW_POSES)
def test_view_data_matches_the_reference_shader_code(O, quality):
    asset, (fp, _keep) = M.view_case(quality)
    want = M.reference("view_" + quality.lower())
    _same_asset(asset, want)
    idx = want["idx"]
    ref, ora = view_fields(want["view"]), view_fields(O.calc_view(asset, fp)[idx])
    # which splats are culled (w = 0: deleted / cut) or behind the camera is decided identically
    assert np.array_equal(ref["pos"][:, 3] <= 0, ora["pos"][:, 3] <= 0)
    assert ((ref["pos"][:, 3] == 0) & (ora["pos"][:, 3] == 0)).sum() > 100 * len(idx) / M.N   # > 100 of the whole scene
    assert (np.abs(ref["pos"] - ora["pos"]).max(1) <= 2e-6 * (1 + np.abs(ora["pos"]).max(1))).all()
    vis = ora["pos"][:, 3] > 0
    for ch in "rgb":                                         # half-precision results: at most one unit in the last place apart
        d = np.abs(ref[ch][vis] - ora[ch][vis])
        assert (d <= np.maximum(np.abs(ora[ch][vis]), 2.0 ** -14) * 2.0 ** -9).all(), ch     # <= 2 half ulps
        assert (d == 0).mean() > 0.9
    assert np.array_equal(ref["a"][vis], ora["a"][vis])
    # the two screen axes, through the covariance they encode (eigenvectors of near-circular footprints are ill-defined)
    cr, co = screen_cov(ref)[vis], screen_cov(ora)[vis]
    rel = np.abs(cr - co).reshape(-1, 4).max(1) / (co[:, 0, 0] + co[:, 1, 1])
    assert np.percentile(rel, 50) < 1e-6 and np.percentile(rel, 99) < 2e-5 and rel.max() < 2e-3


@pytest.mark.parametrize("quality", M.KEY_QUALITIES + M.KEY_POSES)
def test_sort_keys_match_the_reference_shader_code(O, quality):
    asset, (fp, _keep), order = M.key_case(quality)
    want = M.reference("keys_" + quality.lower())
    _same_asset(asset, want)
    kr, ko = want["keys"], O.calc_distances(asset, fp, order)[want["idx"]]
    zr, zo = unsortable(kr), unsortable(ko)
    assert np.abs(zr - zo).max() <= 4e-6 and (kr == ko).mean() > 0.5     # view-space depth of +-36: a couple of ulp
    assert np.array_equal(np.argsort(kr, kind="stable")[:100], np.argsort(ko, kind="stable")[:100]) or (kr == ko).mean() < 1.0


def test_export_and_baked_transform_match_the_reference_shader_code(O):
    """CSExportData incl. the _ExportTransformFlags branch: QuatMul, scale, and RotateSH (the closed form after sh-lib,
    S/SphericalHarmonics.hlsl) against the oracle's export and the product's gsa_bake_transform (least-squares band matrices)."""
    from unitygaussiansplatting_b200.renderer import bake_transform
    asset, (fp, _keep), _fpT, T, q, s = M.export_case()
    want = M.reference("export")
    _same_asset(asset, want)
    idx = want["idx"]
    plain_ref, plain_ora = want["plain"], O.export_data(asset, fp)[idx]
    assert np.allclose(plain_ref, plain_ora, rtol=2e-6, atol=2e-6)
    baked_ref = want["baked"]
    baked_ours = bake_transform(O.export_data(asset, fp), T, rotation=q, scale=s)[idx]
    assert np.allclose(baked_ref[:, 0:3], baked_ours[:, 0:3], atol=1e-5)                  # positions
    assert np.allclose(baked_ref[:, 55:58], baked_ours[:, 55:58], atol=1e-5)              # log scale
    same = np.abs(baked_ref[:, 58:62] - baked_ours[:, 58:62]).max(1)
    flip = np.abs(baked_ref[:, 58:62] + baked_ours[:, 58:62]).max(1)
    assert np.minimum(same, flip).max() < 1e-5                                            # rotation (q and -q are the same)
    assert np.array_equal(baked_ref[:, 6:9], baked_ours[:, 6:9])                          # band 0
    assert np.abs(baked_ref[:, 9:54] - plain_ref[:, 9:54]).max() > 0.05                   # the rotation does something ...
    assert np.abs(baked_ref[:, 9:54] - baked_ours[:, 9:54]).max() < 2e-5                  # ... and ours is the same rotation


def test_draw_stages_match_the_reference_shader_code(O):
    """vert + frag of RenderGaussianSplats.shader on one rotated, anisotropic splat: the quad the reference emits maps pixel
    centres to quad coordinates (the rasteriser's linear interpolation), frag gives the fragment; the oracle's render of that
    splat (fp32 blend, so the image IS the fragment) must be the same picture."""
    view, order, W, H = M.draw_case(False)
    want = M.reference("draw")
    assert np.array_equal(view, want["view"]), "the oracle's view data is no longer the reference's input"
    rt = O.render(view, order, W, H, blend_mode=1)
    clip, qpos, col = want["clip"], want["qpos"], want["col"]
    assert np.array_equal(np.abs(qpos), np.full((4, 2), 2.0, np.float32))                 # quad corners at +-2 (:54-55)
    # pixel position of each corner; interpolation inside a parallelogram is affine: solve quad coords from three corners
    px, A = M.quad_map(clip, qpos, W, H)
    assert np.allclose(np.array([*px[3], 1.0]) @ A, qpos[3], atol=1e-4)
    checked = drawn = 0
    for y in range(0, H):
        for x in range(0, W):
            qx, qy = np.array([x + 0.5, y + 0.5, 1.0]) @ A
            if abs(qx) > 2.3 or abs(qy) > 2.3:
                assert rt[y, x, 3] == 0
                continue
            edge = min(abs(abs(qx) - 2), abs(abs(qy) - 2)) < 2e-3
            out, discarded = want["frag"][y, x], bool(want["discarded"][y, x])
            inside = abs(qx) <= 2 and abs(qy) <= 2
            wanted = np.zeros(4, np.float32) if (discarded or not inside) else out
            if edge or abs(float(np.exp(-(qx * qx + qy * qy))) * col[3] - 1 / 255) < 2e-5:
                continue                                                                   # on the quad edge / discard threshold
            assert np.abs(rt[y, x] - wanted).max() < 3e-6, (x, y, rt[y, x], wanted)
            checked += 1
            drawn += int(wanted[3] > 0)
    assert checked > 700 and drawn > 400


def test_selected_splat_branch_matches_the_reference_shader_code(O):
    """With an edit selection bound the reference's vertex shader hands a selected splat to the pixel shader with col.a = -1
    (S/RenderGaussianSplats.shader:63-73) and the pixel shader takes its "selected" branch (:87-101: opacity from the gaussian
    alone, +0.3, a solid magenta ring where exp(power) is in (7/255, 10/255), magenta tint).  The oracle's draw with
    selected_bits must give the picture the compiled reference vert + frag give."""
    view, order, W, H = M.draw_case(True)
    want = M.reference("draw_selected")
    assert np.array_equal(view, want["view"]), "the oracle's view data is no longer the reference's input"
    bits = np.zeros(2, np.uint32)
    bits[0] = 1                                                                            # splat 0 selected, the padding splats not
    col = want["col"]
    assert col[3] == -1.0
    assert want["col_other"][3] >= 0.0
    plain = O.render(view, order[:1], W, H, blend_mode=1)
    rt = O.render(view, order[:1], W, H, blend_mode=1, selected_bits=bits)
    assert plain[..., 3].max() < 0.03 and rt[..., 3].max() == 1.0                          # opacity 0.02 alone is almost nothing
    _px, A = M.quad_map(want["clip"], want["qpos"], W, H)
    checked = ring = 0
    for y in range(H):
        for x in range(W):
            qx, qy = np.array([x + 0.5, y + 0.5, 1.0]) @ A
            if abs(qx) > 2.3 or abs(qy) > 2.3:
                assert rt[y, x, 3] == 0
                continue
            e = float(np.exp(-(qx * qx + qy * qy)))
            if min(abs(abs(qx) - 2), abs(abs(qy) - 2)) < 2e-3 or min(abs(e - 1 / 255), abs(e - 7 / 255), abs(e - 10 / 255)) < 3e-5:
                continue                                                                   # on the quad edge / one of the three thresholds
            out, discarded = want["frag"][y, x], bool(want["discarded"][y, x])
            inside = abs(qx) <= 2 and abs(qy) <= 2
            wanted = np.zeros(4, np.float32) if (discarded or not inside) else out
            assert np.abs(rt[y, x] - wanted).max() < 3e-6, (x, y, rt[y, x], wanted)
            checked += 1
            ring += int(wanted[3] == 1.0 and wanted[0] == 1.0 and wanted[1] == 0.0)
    assert checked > 700 and ring > 20


def test_rotation_packing_matches_the_reference_shader_code():
    """The importer packs rotations with C# twins of these HLSL functions; the packer (gsa_pack_smallest3 + its 10.10.10.2
    encoder, checked through a one-splat asset) must produce the same code words, and decoding must agree."""
    from unitygaussiansplatting_b200 import _native as N
    lib = N.asset_lib()
    want = M.reference("rotation")
    for i, q in enumerate(M.rotation_quats()):
        ours, ref = np.zeros(4, np.float32), want["packed"][i]
        lib.gsa_pack_smallest3(np.ascontiguousarray(q).ctypes.data, ours.ctypes.data)
        enc_ref = int(want["enc"][i])
        assert np.allclose(ours, ref, atol=1e-7)
        enc_ours = (int(ours[0] * 1023.5) | (int(ours[1] * 1023.5) << 10) | (int(ours[2] * 1023.5) << 20) | (int(ours[3] * 3.5) << 30)) & 0xFFFFFFFF
        assert enc_ours == enc_ref or np.abs(ours - ref).max() > 0      # same code word whenever the packed floats are identical
        back = want["decoded"][i]
        assert min(np.abs(back - q).max(), np.abs(back + q).max()) < 2.5e-3                # 10-bit components
