"""VeryLow / Low importer presets (SURVEY 8f N4): BC7 colour and clustered-SH palettes -- decode pinned against an
independent BC7 decoder, the packer's two lossy stages checked against small restatements, CPU only."""
import ctypes as C
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
GOLD = ROOT / "tests" / "golden" / "bc7_blocks.npz"


def test_oracle_bc7_decode_matches_independent_decoder(O):
    """tests/golden/bc7_blocks.npz: 512 random blocks of each of the 8 modes, pixels decoded by Pillow
    (tests/golden/make_bc7_golden.py).  Bit-exact."""
    d = np.load(GOLD)
    got = O.bc7_decode_blocks(d["blocks"])
    bad = np.nonzero((got != d["pixels"]).any(axis=(1, 2)))[0]
    assert bad.size == 0, "oracle BC7 decode differs for blocks %s" % bad[:8]
    modes = [int(np.log2(b & -b)) for b in d["blocks"][:, 0].astype(np.int32)]
    assert sorted(set(modes)) == list(range(8))


def test_product_bc7_texel_decode_matches_independent_decoder(tmp_path):
    """csrc/gs_bc7.cuh is plain C++: compile the very code k_calc_view runs with g++ and check all 16 texels of every
    golden block (the device build of the same header is covered by the GPU parity tests)."""
    so = tmp_path / "libbc7t.so"
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", str(ROOT / "tests" / "bc7_texel_test.cpp"), "-o", str(so)],
                   check=True)
    lib = C.CDLL(str(so))
    d = np.load(GOLD)
    blocks = np.ascontiguousarray(d["blocks"])
    out = np.zeros((len(blocks), 16, 4), np.uint8)
    lib.bc7_texels(blocks.ctypes.data, len(blocks), out.ctypes.data)
    assert np.array_equal(out, d["pixels"])
    zero = np.zeros((1, 16), np.uint8)   # reserved mode (first byte 0): all channels 0
    lib.bc7_texels(zero.ctypes.data, 1, out.ctypes.data)
    assert not out[0].any()


def test_bc7_encoder_round_trip(g, O):
    from unitygaussiansplatting_b200 import _native as N
    L = N.asset_lib()
    rng = np.random.default_rng(7)

    def enc(blk):
        blk = np.ascontiguousarray(blk, np.float32)
        out = np.zeros(16, np.uint8)
        L.gsa_bc7_encode_block(blk.ctypes.data, out.ctypes.data)
        return out

    for _ in range(200):
        const = np.tile(rng.random(4), (16, 1)).astype(np.float32)
        e = enc(const)
        assert e[0] & 0x7F == 0x40, "mode 6"
        dec = O.bc7_decode_blocks(e[None])[0].astype(np.float32) / 255.0
        assert np.abs(dec - const).max() <= 1.0 / 255.0 + 1e-6
        base, slope = 0.25 + 0.5 * rng.random(4), 0.5 * (rng.random(4) - 0.5)   # stays inside [0,1]: a straight segment
        ramp = (base[None, :] + np.linspace(0, 1, 16)[:, None] * slope[None, :]).astype(np.float32)
        dec = O.bc7_decode_blocks(enc(ramp)[None])[0].astype(np.float32) / 255.0
        assert np.abs(dec - ramp).max() <= 0.02, "points on a line in RGBA are what mode 6 represents well"
    # NaN / out-of-range input never produces an invalid block
    weird = np.full((16, 4), np.nan, np.float32)
    weird[3] = [2.0, -1.0, 0.5, 1.0]
    assert enc(weird)[0] & 0x7F == 0x40


def test_bc7_encoder_bytes_match_fixture(g):
    """tests/golden/bc7_encode_blocks.npz (tests/golden/make_bc7_encode_golden.py): 2,560 blocks -- random, noisy ramps,
    constant, two-colour, out of range, NaN / Inf -- and the 16 bytes the encoder wrote for each.  The GPU packer runs the
    same encoder (csrc/gs_asset_format.h), so this pins both."""
    from unitygaussiansplatting_b200 import _native as N
    L = N.asset_lib()
    d = np.load(ROOT / "tests" / "golden" / "bc7_encode_blocks.npz")
    rgba = np.ascontiguousarray(d["rgba"], np.float32)
    out = np.zeros((len(rgba), 16), np.uint8)
    for i in range(len(rgba)):
        L.gsa_bc7_encode_block(rgba[i].ctypes.data, out[i].ctypes.data)
    bad = np.nonzero((out != d["encoded"]).any(axis=1))[0]
    assert bad.size == 0, "BC7 encoder output differs for blocks %s" % bad[:8]


# ---- k-means: a scalar restatement of E/Utils/KMeansClustering.cs in numpy float32, for a case small enough for Python ----
F = np.float32


def _pcg_hash(x):
    state = (x * 747796405 + 2891336453) & 0xFFFFFFFF
    word = (((state >> ((state >> 28) + 4)) ^ state) * 277803737) & 0xFFFFFFFF
    return ((word >> 22) ^ word) & 0xFFFFFFFF


class _Rng:
    def __init__(self):
        self.s = 1

    def random(self):
        state = self.s
        self.s = (self.s * 747796405 + 2891336453) & 0xFFFFFFFF
        word = (((state >> ((state >> 28) + 4)) ^ state) * 277803737) & 0xFFFFFFFF
        return ((word >> 22) ^ word) & 0xFFFFFFFF


def _dist(a, b):
    d = F(0)
    dim = len(a)
    i = 0
    while i + 7 < dim:
        v = [(a[i + k] - b[i + k]) * (a[i + k] - b[i + k]) for k in range(8)]
        h = [v[0] + v[1], v[2] + v[3], v[4] + v[5], v[6] + v[7]]
        d = d + (((h[0] + h[1]) + h[2]) + h[3])
        i += 8
    while i < dim:
        t = a[i] - b[i]
        d = d + t * t
        i += 1
    return d


def _batch(data, rng, n):
    seed = rng.random()
    picked, out = set(), []
    while len(out) < n:
        idx = _pcg_hash(seed) % len(data)
        seed = (seed + 1) & 0xFFFFFFFF
        if idx not in picked:
            picked.add(idx)
            out.append(data[idx].copy())
    return np.array(out)


def _assign(data, means):
    labels, dists = [], []
    for p in data:
        best, bi = F(np.finfo(np.float32).max), 0
        for j, m in enumerate(means):
            d = _dist(p, m)
            if d < best:
                best, bi = d, j
        labels.append(bi)
        dists.append(best)
    return labels, dists


def _kmeans_ref(data, k, batch, passes):
    n, dim = data.shape
    batch = min(n, batch)
    rng = _Rng()
    init = min(10 * k, n)
    cb, vb = _batch(data, rng, init), _batch(data, rng, init)
    best_sum, means = F(np.finfo(np.float32).max), None
    mind = np.zeros(init, np.float32)
    for _ in range(3):
        taken = [False] * init
        cur = []
        p = rng.random() % init
        taken[p] = True
        cur.append(cb[p].copy())
        for i in range(init):
            if i != p:
                mind[i] = _dist(cb[i], cur[0])
        while len(cur) < k:
            nb = (init + 1023) // 1024
            partial, total = [], F(0)
            for b in range(nb):
                s = F(0)
                for i in range(b * 1024, min((b + 1) * 1024, init)):
                    if not taken[i]:
                        s = s + mind[i]
                total = total + s
                partial.append(total)
            val = _pcg_hash((rng.s + len(cur)) & 0xFFFFFFFF)
            f = np.array([0x3F800000 | (val >> 9)], np.uint32).view(np.float32)[0] - F(1)
            rval = f * total
            lo, hi = 0, nb
            while lo < hi:
                mid = (lo + hi) // 2
                if partial[mid] < rval:
                    lo = mid + 1
                else:
                    hi = mid
            acc = partial[lo - 1] if lo > 0 else F(0)
            pick = -1
            for i in range(lo * 1024, init):
                if taken[i]:
                    continue
                acc = acc + mind[i]
                if acc >= rval:
                    pick = i
                    break
            if pick < 0:
                pick = max(i for i in range(init) if not taken[i])
            taken[pick] = True
            cur.append(cb[pick].copy())
            if len(cur) < k:
                for i in range(init):
                    if not taken[i]:
                        mind[i] = min(mind[i], _dist(cb[i], cur[-1]))
        _, dists = _assign(vb, cur)
        s = F(0)
        for d in dists:
            s = s + d
        mind[:] = dists
        if s < best_sum:
            best_sum, means = s, [c.copy() for c in cur]
    counts = np.zeros(k, np.float32)
    done, limit = F(0), F(n) * F(passes)
    while done < limit:
        pts = _batch(data, rng, batch)
        labels, _ = _assign(pts, means)
        for i, c in enumerate(labels):
            counts[c] += F(1)
            alpha = F(1) / counts[c]
            means[c] = means[c] + alpha * (pts[i] - means[c])
        done = done + F(batch)
    labels, _ = _assign(data, means)
    return np.array(means), np.array(labels)


def test_kmeans_matches_scalar_restatement():
    from unitygaussiansplatting_b200 import _native as N
    rng = np.random.default_rng(11)
    n, k, dim = 260, 7, 45
    centres = rng.standard_normal((5, dim)).astype(np.float32)
    data = (centres[rng.integers(0, 5, n)] + 0.3 * rng.standard_normal((n, dim))).astype(np.float32)
    means = np.zeros((k, dim), np.float32)
    labels = np.zeros(n, np.int32)
    rc = N.asset_lib().gsa_kmeans(dim, data.ctypes.data, n, 64, 1.2, means.ctypes.data, k, labels.ctypes.data)
    assert rc == 0
    with np.errstate(over="ignore"):
        ref_means, ref_labels = _kmeans_ref(data, k, 64, 1.2)
    assert np.array_equal(labels, ref_labels)
    assert np.array_equal(means.view(np.uint32), ref_means.astype(np.float32).view(np.uint32)), "centres must match to the bit"
    # every label is the nearest centre, and the run is deterministic
    d2 = ((data[:, None, :].astype(np.float64) - means[None].astype(np.float64)) ** 2).sum(-1)
    assert np.allclose(d2[np.arange(n), labels], d2.min(1), rtol=1e-5)
    means2, labels2 = np.zeros_like(means), np.zeros_like(labels)
    N.asset_lib().gsa_kmeans(dim, data.ctypes.data, n, 64, 1.2, means2.ctypes.data, k, labels2.ctypes.data)
    assert np.array_equal(means, means2) and np.array_equal(labels, labels2)
    assert N.asset_lib().gsa_kmeans(dim, data.ctypes.data, 5, 64, 1.2, means.ctypes.data, k, labels.ctypes.data) != 0  # fewer points than clusters


@pytest.mark.parametrize("quality", ["VeryLow", "Low"])
def test_low_preset_asset_layout_and_decode(g, O, quality):
    n = 20000 if quality == "VeryLow" else 17000
    if quality == "Low":
        with pytest.raises(ValueError):      # 16k palette entries need more than 16k splats (the reference writes a broken asset)
            g.synthetic_asset(g.SCENE_CLUSTERED, 16000, 1, "Low")
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, n, 0x5EED0021, quality)
    ref = g.synthetic_asset(g.SCENE_CLUSTERED, n, 0x5EED0021, "VeryHigh")
    k = 4096 if quality == "VeryLow" else 16384
    assert asset.shData.nbytes == k * 96                               # palette of SHTableItemFloat16
    assert asset.otherData.nbytes == (n * (4 + 2 + 2) + 7) // 8 * 8     # rot + Norm6 scale + u16 palette index
    tex_h = (((n + 2047) // 2048) + 15) // 16 * 16
    assert asset.colorData.nbytes == 2048 * tex_h * (1 if quality == "VeryLow" else 4)
    idx = asset.otherData[:n * 8].reshape(n, 8)[:, 6:8].copy().view(np.uint16)[:, 0]
    assert idx.max() < k
    pal = asset.shData.view(np.float16).reshape(k, 48)[:, :45].astype(np.float32)
    for i in range(0, n, 613):
        lo, hi = O.load_splat(asset, i), O.load_splat(ref, i)
        assert np.array_equal(np.asarray(lo["sh"], np.float32).reshape(45), pal[idx[i]])          # SH = the palette entry, no chunk lerp
        d2 = ((pal - np.asarray(hi["sh"], np.float32).reshape(1, 45)) ** 2).sum(1)
        assert d2[idx[i]] <= d2.min() * 1.0001 + 1e-6                                  # ... and the nearest one (fp16-rounded palette)
        assert np.abs(np.asarray(lo["pos"]) - np.asarray(hi["pos"])).max() < 0.05
        if quality == "Low":
            assert np.abs(np.asarray(lo["col"]) - np.asarray(hi["col"])).max() < 0.01
    if quality == "VeryLow":
        # BC7 is lossy on uncorrelated colours (this scene's are random per splat); on average it must still track them
        err = [np.abs(np.asarray(O.load_splat(asset, i)["col"]) - np.asarray(O.load_splat(ref, i)["col"])).mean() for i in range(0, n, 97)]
        assert np.mean(err) < 0.2


def test_low_preset_oracle_frame_is_close_to_lossless(g, O):
    """End to end through the oracle: a Low-preset asset renders like the VeryHigh one up to its quantisation."""
    from util import camera
    n = 17000
    cam = camera(g, 160, 120)
    fp, _keep = g.make_frame_params(cam, sh_order=0)
    rts = {}
    for q in ("Low", "VeryHigh"):
        rts[q] = O.frame(g.synthetic_asset(g.SCENE_CLUSTERED, n, 0x5EED0022, q), fp, threads=O.max_threads())["rt"].astype(np.float32)
    assert np.abs(rts["Low"] - rts["VeryHigh"]).mean() < 0.02
