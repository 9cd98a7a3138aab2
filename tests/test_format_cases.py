"""tests/util.py FORMAT_CASES must keep reaching every decode path the GPU format tests (tests/test_gpu_formats.py) are there
to compare with the oracle, so that an edit of the list cannot drop coverage silently."""
import sys
from pathlib import Path

import numpy as np

from util import FORMAT_CASES, case_asset, palette_backed

sys.path.insert(0, str(Path(__file__).parent / "golden"))
import make_ref_hlsl_golden as M  # noqa: E402

SCALE_BYTES = (12, 6, 4, 2)


def _chunked(f):
    return any(f)      # the importer chunks every asset that is not Float32 throughout


def test_view_kernel_instantiations():
    """k_calc_view<SHFMT, CULL, BC7>: SHFMT is the SH format, all clustered formats sharing 4; CULL is both tests' business."""
    pairs = {(min(c.formats[3], 4), c.formats[2] == 3) for c in FORMAT_CASES}
    assert pairs == {(s, b) for s in range(5) for b in (False, True)}


def test_other_record_layouts():
    """4 + scale bytes (+ 2 for the palette index): the unclustered 16 / 10 / 8 / 6 and clustered 18 / 12 / 10 / 8 byte records,
    over k_calc_view's uint4, uint2 and 2-aligned load paths."""
    layouts = {(c.formats[1], c.formats[3] > 3) for c in FORMAT_CASES}
    assert layouts == {(s, cl) for s in range(4) for cl in (False, True)}


def test_formats_inside_chunked_assets():
    chunked = [c.formats for c in FORMAT_CASES if _chunked(c.formats)]
    assert {f[0] for f in chunked} == {0, 1, 2, 3}, "every position format, chunk-lerped"
    assert {f[2] for f in chunked} == {0, 1, 2, 3}, "every colour format, chunk-lerped"
    assert {f[3] for f in chunked} >= {0, 1, 2, 3}, "every unclustered SH format in a chunked asset (Float32 is not lerped)"


def test_every_sh_format():
    assert {c.formats[3] for c in FORMAT_CASES} == set(range(9))


def test_splat_counts_reach_the_tails():
    """_SplatViewData leaves a block of 256 records in 16-byte stores plus a tail of 4-byte words when the block holds an odd
    number of records; k_calc_distances reads 4 splats per thread and takes its generic path for a partial last quad."""
    n = [c.n for c in FORMAT_CASES]
    assert len(set(n)) == len(n)
    assert all(k % 4 for k in n)
    assert {k % 4 for k in n} == {1, 2, 3}
    assert sum(k % 2 == 0 for k in n) <= 1, "all counts but the one with n % 4 == 2 are odd: their last block has an odd tail"
    assert any(k % 256 == 1 for k in n), "a last block of one splat"


def test_palette_indices_past_the_palette(g):
    """Cluster64k, 32k and 16k are synthesised from a host-packed Cluster4k asset; their indices, and those of the
    out-of-palette Cluster4k case, cover 0..65535, and the oracle's copy of the palette has all 65536 entries."""
    rewritten = {c.formats[3] for c in FORMAT_CASES if c.indices}
    assert rewritten >= {4, 5, 6, 8}
    for c in FORMAT_CASES:
        if not c.indices:
            continue
        a = case_asset(g, c)
        pf, sf, cf, shf = c.formats
        assert (a.posFormat, a.scaleFormat, a.colorFormat, a.shFormat) == c.formats
        entries = 65536 >> (shf - 4)
        assert a.shData.nbytes == entries * 96
        stride = 4 + SCALE_BYTES[sf] + 2
        idx = a.otherData[:c.n * stride].reshape(c.n, stride)[:, stride - 2:].copy().view(np.uint16).ravel()
        assert (idx >= 32768).mean() >= 0.25
        if entries < 65536:
            assert (idx >= entries).mean() >= 0.25, "indices past the palette's end"
        if shf in (4, 5, 6):
            h = a.shData.view(np.float16).reshape(entries, 48)
            assert np.isfinite(h).all() and (h[:, 45:] == 0).all() and np.abs(h[:, :45]).max() > 0.5
        b = palette_backed(a)
        assert b.shData.nbytes == 65536 * 96 and np.array_equal(b.shData[:a.shData.nbytes], a.shData) and not b.shData[a.shData.nbytes:].any()


def test_reference_shader_cases_follow_the_list():
    """Every format case without BC7 colour is pinned to the reference's shader code, and the Norm6 and chunked Float32
    position cases to its CSCalcDistances."""
    assert {"custom-" + c.name for c in FORMAT_CASES if c.formats[2] != 3} <= set(M.VIEW_QUALITIES)
    keyed = [c.formats for c in FORMAT_CASES if "custom-" + c.name in M.KEY_QUALITIES]
    assert any(f[0] == 3 for f in keyed) and any(f[0] == 0 and _chunked(f) for f in keyed)
