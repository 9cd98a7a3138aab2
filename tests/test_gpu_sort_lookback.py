"""The sort's pointer-jumping look-back: tile edges, one and several waves of tiles, and digits that never change."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TILE = 8192
WAVE = 264 * TILE   # 2 CTAs on each of an H100 SXM's 132 SMs


def _check(ctx, keys):
    payload = np.arange(keys.size, dtype=np.uint32)
    k, p = keys.copy(), payload.copy()
    ctx.sort_pairs(k, p)
    order = np.argsort(keys, kind="stable").astype(np.uint32)
    assert np.array_equal(p, order), "payload order differs from a stable sort"
    assert np.array_equal(k, keys[order])


@pytest.mark.parametrize("n", [TILE - 1, TILE, TILE + 1, WAVE - 1, WAVE + 1, 3 * WAVE + 4097])
def test_tile_and_wave_edges(ctx, n):
    _check(ctx, np.random.default_rng(n).integers(0, 2**32, n, dtype=np.uint32))


@pytest.mark.parametrize("kind", ["all_equal", "one_digit_value"])
def test_constant_digits(ctx, kind):
    n = 2 * WAVE + 123
    rng = np.random.default_rng(5)
    if kind == "all_equal":
        keys = np.full(n, 0x8000_0001, np.uint32)
    else:   # the second byte is the same everywhere: that pass sends every pair of a tile to one digit
        keys = (rng.integers(0, 2**32, n, dtype=np.uint32) & np.uint32(0xFFFF00FF)) | np.uint32(0x5A00)
    _check(ctx, keys)
