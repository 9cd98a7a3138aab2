#!/usr/bin/env python
"""Regenerates tests/golden/bc7_encode_blocks.npz: float RGBA 4x4 blocks and the 16 bytes gsa_bc7_encode_block writes
for each.  No other fixture pins the encoder's bytes (bc7_blocks.npz pins decode, the round-trip test bounds the error),
and the GPU packer's k_bc7 runs the same encoder, so this file is what holds its output still.  The blocks: uniform
random, noisy ramps (what a Morton-ordered colour image looks like), constant, two-colour, out of [0, 1], and NaN / Inf.
The recorded bytes are the encoder's at the time of writing: regenerate only for an intended change of the encoder.
Run: python tests/golden/make_bc7_encode_golden.py"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))


def blocks():
    rng = np.random.default_rng(0xBC7E)
    f = np.float32
    uniform = rng.random((1024, 16, 4), dtype=f)
    t = np.linspace(0, 1, 16, dtype=f)[None, :, None]
    base, slope = rng.random((1024, 1, 4), dtype=f), rng.random((1024, 1, 4), dtype=f) - f(0.5)
    ramps = base + t * slope + f(0.03) * (rng.random((1024, 16, 4), dtype=f) - f(0.5))
    ramps = np.round(ramps * 4096) / 4096   # exact in float32; keeps the file small
    const = np.repeat(rng.random((128, 1, 4), dtype=f), 16, axis=1)
    const[:4] = [[0, 0, 0, 0]], [[1, 1, 1, 1]], [[0.5, 0.5, 0.5, 0.5]], [[1 / 255, 254 / 255, 0.25, 0.75]]
    two = np.repeat(rng.random((128, 2, 4), dtype=f), 8, axis=1)
    two = np.take_along_axis(two, np.argsort(rng.random((128, 16, 1)), axis=1), axis=1)   # the two colours shuffled
    wide = f(4) * rng.random((128, 16, 4), dtype=f) - f(1.5)   # mostly outside [0, 1]
    wide[:8] = rng.choice(np.array([-1e30, -1, -0.0, 0, 1, 2, 1e30], f), (8, 16, 4))
    odd = rng.random((128, 16, 4), dtype=f)
    special = np.array([np.nan, np.inf, -np.inf], f)
    mask = rng.random((128, 16, 4)) < 0.25
    odd[mask] = rng.choice(special, int(mask.sum()))
    odd[0], odd[1], odd[2] = np.nan, np.inf, -np.inf
    return np.concatenate([uniform, ramps, const, two, wide, odd]).astype(f)


def main():
    from unitygaussiansplatting_b200 import _native as N
    lib = N.asset_lib()
    rgba = np.ascontiguousarray(blocks())
    out = np.zeros((len(rgba), 16), np.uint8)
    for i in range(len(rgba)):
        lib.gsa_bc7_encode_block(rgba[i].ctypes.data, out[i].ctypes.data)
    np.savez_compressed(Path(__file__).with_name("bc7_encode_blocks.npz"), rgba=rgba, encoded=out)
    print("wrote", len(rgba), "blocks")


if __name__ == "__main__":
    main()
