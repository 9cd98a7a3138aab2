"""check_regions, the one check of what a call wrote into an array and what it left alone, fails on every difference a word
comparison can see: a flipped bit, another NaN payload, -0 for +0, a touched texel in another layer or beside a region."""
import numpy as np
import pytest

from images import SENTINEL, check_regions

NAN_WORDS = {np.float16: (0x7E00, 0x7E01, np.uint16), np.float32: (0x7FC00000, 0x7FC00001, np.uint32)}


def _words(a):
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


def _array(dtype, start=None):
    """(texels, start, regions): two layers of `start` texels with a region of random content at (x, y) = (2, 1) of layer 1."""
    if start is None:
        start = np.uint32(0xDEADBEEF) if dtype == np.uint32 else dtype(SENTINEL)
    got = np.full((2, 6, 8, 4), start, dtype)
    want = np.random.default_rng(1).integers(0, 1000, (3, 4, 4)).astype(dtype)
    got[1, 1:4, 2:6] = want
    return got, start, [(1, 2, 1, want)]


def _nan(dtype, word):
    return np.array(word, NAN_WORDS[dtype][2]).view(dtype)


@pytest.mark.parametrize("dtype", [np.float16, np.float32, np.uint32])
def test_exact_equality_passes(dtype):
    got, start, regions = _array(dtype)
    check_regions(got, start, regions, "equal")


@pytest.mark.parametrize("dtype", [np.float16, np.float32, np.uint32])
def test_one_flipped_bit_inside_a_region_fails(dtype):
    got, start, regions = _array(dtype)
    _words(got)[1, 2, 3, 1] ^= 1
    with pytest.raises(AssertionError, match="rectangle"):
        check_regions(got, start, regions, "flipped bit")


@pytest.mark.parametrize("dtype", [np.float16, np.float32], ids=["rgba16f", "rgba32f"])
def test_another_nan_payload_fails(dtype):
    a, b, _ = NAN_WORDS[dtype]
    got, start, regions = _array(dtype)
    _words(regions[0][3])[0, 0, 0] = a
    _words(got)[1, 1, 2, 0] = b
    assert np.isnan(regions[0][3][0, 0, 0]) and np.isnan(got[1, 1, 2, 0])
    with pytest.raises(AssertionError, match="rectangle"):
        check_regions(got, start, regions, "NaN payload inside")
    _words(got)[1, 1, 2, 0] = a
    check_regions(got, start, regions, "the same NaN")
    # outside the regions, against a NaN start
    got, start, regions = _array(dtype, _nan(dtype, a))
    check_regions(got, start, regions, "NaN start")
    _words(got)[0, 5, 7, 3] = b
    with pytest.raises(AssertionError, match="outside"):
        check_regions(got, start, regions, "NaN payload outside")


@pytest.mark.parametrize("dtype", [np.float16, np.float32])
def test_negative_zero_is_not_positive_zero(dtype):
    got, start, regions = _array(dtype)
    regions[0][3][2, 3, 2] = 0.0
    got[1, 3, 5, 2] = -0.0
    with pytest.raises(AssertionError, match="rectangle"):
        check_regions(got, start, regions, "-0 inside")
    got[1, 3, 5, 2] = 0.0
    check_regions(got, start, regions, "+0 inside")
    got, start, regions = _array(dtype, dtype(0.0))
    got[0, 0, 0, 0] = -0.0
    with pytest.raises(AssertionError, match="outside"):
        check_regions(got, start, regions, "-0 outside")


@pytest.mark.parametrize("dtype", [np.float16, np.float32, np.uint32])
@pytest.mark.parametrize("where", [(0, 3, 4), (1, 0, 0), (1, 4, 2), (1, 2, 6)],
                         ids=["other-layer", "same-layer-corner", "below-the-region", "beside-the-region"])
def test_one_touched_texel_outside_fails(dtype, where):
    got, start, regions = _array(dtype)
    _words(got)[where + (1,)] ^= 0x10
    with pytest.raises(AssertionError, match="1 texels outside"):
        check_regions(got, start, regions, "touched")


@pytest.mark.parametrize("dtype", [np.float16, np.float32], ids=["rgba16f", "rgba32f"])
def test_nan_sentinel_passes_on_exact_equality(dtype):
    got, start, regions = _array(dtype, _nan(dtype, 0x7D55 if dtype == np.float16 else 0x7FA5A5A5))
    check_regions(got, start, regions, "NaN sentinel")
