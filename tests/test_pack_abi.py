"""The GPU packer's C ABI without a GPU: ctypes layouts match include/gsplat_b200.h, the symbols are exported, and
gs_pack_sizes is gsa_calc_sizes' arithmetic."""
import ctypes as C

import pytest


def test_pack_structs_match_the_header():
    from unitygaussiansplatting_b200 import _native as N
    assert C.sizeof(N.GsPackDesc) == 8 + 6 * 4
    assert C.sizeof(N.GsPackedAsset) == 5 * 8 + 2 * 4 + 6 * 4
    assert C.sizeof(N.GsPackSizes) == C.sizeof(N.GsaSizes) == 5 * 8 + 2 * 4
    assert [f[0] for f in N.GsPackSizes._fields_] == [f[0] for f in N.GsaSizes._fields_]
    assert N.GsPackedAsset.bounds_min.offset == 48 and N.GsPackDesc.splat_count.offset == 8


def test_pack_symbols_are_exported(g):
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    for name in ("gs_pack_asset", "gs_pack_sizes", "gs_kmeans", "gs_debug_pack_stats"):
        assert hasattr(lib, name) and name in N.NATIVE_SYMBOLS


@pytest.mark.parametrize("n", [1, 255, 256, 2049, 4096, 4097, 16385, 70000])
def test_pack_sizes_equal_host_sizes(g, n):
    from unitygaussiansplatting_b200 import _native as N
    lib, alib = N.native(), N.asset_lib()
    for pf in range(5):
        for sf in (0, 3, 4):
            for cf in range(5):
                for shf in range(10):
                    a, b = N.GsPackSizes(), N.GsaSizes()
                    rc = lib.gs_pack_sizes(n, pf, sf, cf, shf, C.byref(a))
                    rh = alib.gsa_calc_sizes(n, pf, sf, cf, shf, C.byref(b))
                    assert (rc == 0) == (rh == 0)
                    if rc == 0:
                        assert bytes(a) == bytes(b)
                    else:
                        assert rc == -4 and lib.gs_last_error(None)   # GS_ERR_UNSUPPORTED_FORMAT


def test_pack_entry_points_validate_without_a_device(g):
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    assert lib.gs_pack_asset(None, None, None, None) == -1
    assert lib.gs_kmeans(None, 45, None, 10, 4, 1.0, None, 2, None) == -1
    assert lib.gs_debug_pack_stats(None, None) == -1
    assert lib.gs_pack_sizes(10, 0, 0, 0, 0, None) == -1
