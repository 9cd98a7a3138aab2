"""The CUDA path against the reference's own shader code: the same comparisons as tests/test_reference_hlsl.py, with the
C-ABI library's output in place of the oracle's and the reference's output read from tests/golden/ref_hlsl_*.npz (written
by tests/golden/make_ref_hlsl_golden.py from oracle/_ref/libref_hlsl.so).  The fixture holds a fixed seeded sample of 2,048
of the scene's 20,000 splats, so view data and keys are compared on those splats and the keys' order among them; the whole
scene is still rendered and sorted.  Named test_zz_* so that it runs after the parity tests proper."""
import sys
from pathlib import Path

import numpy as np
import pytest

from util import screen_cov, unsortable, view_fields

GOLD = Path(__file__).parent / "golden"
sys.path.insert(0, str(GOLD))
import make_ref_hlsl_golden as M  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("quality", M.QUALITIES)
def test_cuda_view_data_and_keys_match_the_reference_shader_code(g, ctx, quality):
    want = np.load(GOLD / ("ref_hlsl_%s.npz" % quality.lower()))
    asset, cam, _fp, digest = M.scene(quality)
    assert np.array_equal(digest, want["asset_sha256"]), "the synthetic scene is no longer the one the fixture was computed on"
    idx = want["idx"]
    r = g.GaussianSplatRenderer(asset, ctx)
    r.SortPoints(cam)
    r.CalcViewData(cam)
    view, keys, order = r.readback_view(), r.readback_keys(), r.readback_order()
    got, ref = view_fields(view[idx]), view_fields(want["view"])
    assert np.array_equal(ref["pos"][:, 3] <= 0, got["pos"][:, 3] <= 0)
    assert (np.abs(ref["pos"] - got["pos"]).max(1) <= 2e-6 * (1 + np.abs(got["pos"]).max(1))).all()
    vis = got["pos"][:, 3] > 0
    for ch in "rgb":
        d = np.abs(ref[ch][vis] - got[ch][vis])
        assert (d <= np.maximum(np.abs(got[ch][vis]), 2.0 ** -14) * 2.0 ** -9).all(), ch
    assert np.array_equal(ref["a"][vis], got["a"][vis])
    cr, cg = screen_cov(ref)[vis], screen_cov(got)[vis]
    rel = np.abs(cr - cg).reshape(-1, 4).max(1) / (cg[:, 0, 0] + cg[:, 1, 1])
    assert np.percentile(rel, 50) < 1e-6 and np.percentile(rel, 99) < 2e-5 and rel.max() < 2e-3
    # sorted keys: the reference's key of the splat at each sorted position is the same depth to a couple of ulp, and the
    # reference's keys taken in the CUDA draw order ascend
    pos = np.empty(len(order), np.int64)
    pos[order] = np.arange(len(order))
    at = pos[idx]
    assert np.abs(unsortable(want["keys"]) - unsortable(keys[at])).max() <= 4e-6
    ranked = want["keys"][np.argsort(at)]
    assert (np.diff(unsortable(ranked).astype(np.float64)) >= -8e-6).all()
    r.Dispose()
