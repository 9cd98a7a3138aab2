#!/usr/bin/env python
"""Times the host packer (create_asset) against the GPU packer (gs_pack_asset) per quality preset on the clustered synthetic
scene, and prints one JSON line.

Per preset: host_s (create_asset, all usable cores), gpu_s (pack_asset from a host numpy array: input upload, packing and
the blobs' copy back), gpu_device_input_s (the same from a CUDA tensor, so without the input upload).  Every GPU result is
compared byte for byte with the host's where the host was timed.

usage: time_pack.py [--n N] [--presets VeryLow,Low,...] [--no-host P1,P2]   (default: 6131954 splats, all five presets)
"""
import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=6_131_954)
    ap.add_argument("--presets", default="VeryLow,Low,Medium,High,VeryHigh")
    ap.add_argument("--no-host", default="", help="presets whose host packer is not timed")
    ap.add_argument("--seed", type=lambda s: int(s, 0), default=0x5EED0002)
    a = ap.parse_args()
    import torch
    import unitygaussiansplatting_b200 as g
    from unitygaussiansplatting_b200.asset import QUALITY
    from unitygaussiansplatting_b200.renderer import GaussianSplatContext

    ctx = GaussianSplatContext(0)
    splats = g.generate_input_splats(g.SCENE_CLUSTERED, a.n, a.seed)
    g.pack_asset(splats[:5000].copy(), "VeryLow", context=ctx)   # warm-up: module load, every kernel once
    d_splats = torch.from_numpy(splats).cuda()
    torch.cuda.synchronize()
    skip = set(s for s in a.no_host.split(",") if s)
    res = {}
    for q in a.presets.split(","):
        assert q in QUALITY, q
        r = {}
        t0 = time.perf_counter()
        gpu = g.pack_asset(splats, q, context=ctx)
        r["gpu_s"] = round(time.perf_counter() - t0, 3)
        t0 = time.perf_counter()
        gpu2 = g.pack_asset(d_splats, q, context=ctx)
        r["gpu_device_input_s"] = round(time.perf_counter() - t0, 3)
        same = all(np.array_equal(getattr(gpu, b), getattr(gpu2, b)) for b in ("posData", "otherData", "colorData", "shData"))
        if q in skip:
            r["host_s"] = None
        else:
            t0 = time.perf_counter()
            host = g.create_asset(splats.copy(), q)
            r["host_s"] = round(time.perf_counter() - t0, 3)
            for b in ("posData", "otherData", "colorData", "shData", "chunkData"):
                x, y = getattr(gpu, b), getattr(host, b)
                same = same and ((x is None and y is None) or (x is not None and y is not None and np.array_equal(x, y)))
        r["identical"] = bool(same)
        res[q] = r
        print(q, r, file=sys.stderr, flush=True)
    name, power = gpu_info()
    threads = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else os.cpu_count()
    print(json.dumps({"tool": "time_pack", "n": a.n, "scene": "clustered", "gpu": name, "power_limit": power, "host_cpus": threads,
                      "presets": res}))


if __name__ == "__main__":
    main()
