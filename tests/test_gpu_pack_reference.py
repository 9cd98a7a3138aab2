"""gs_pack_asset on the device against THE REFERENCE IMPORTER'S OWN C# (oracle/_ref/libref_cs.so, or its fixtures
tests/golden/ref_cs_pack_*.npz): every case of tests/golden/make_ref_cs_golden.py, compared directly, not through the host
packer.  BC7 colour and the k-means palette and indices are left out, as in tests/test_reference_cs.py."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).parent / "golden"))
import make_ref_cs_golden as M  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(M.CASES))
def test_device_packer_matches_the_reference_importer(g, ctx, name):
    splats, formats = M.CASES[name]()
    ref = M.reference(name)
    assert np.array_equal(M.digest(splats), ref["input_sha256"]), "the scene is no longer the one the reference bytes are for"
    bad = []
    for f in formats:
        asset = g.pack_asset(splats, formats=M.packer_formats(f), context=ctx)
        bad += ["%s: %s" % (M.label(f), m) for m in M.differences(asset, ref, f)]
    assert not bad, "\n".join(bad)
