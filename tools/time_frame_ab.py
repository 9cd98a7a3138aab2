#!/usr/bin/env python
"""gs_frame of this tree's library against another build of it (e.g. the parent commit's), loaded side by side in one process
and timed in alternating blocks.

Workload: a bench.py workload (default metric: 6,131,954 splats, Medium, 1920x1080, orbiting camera) into a device render
target, frames issued back to back as bench.py issues them.  Per library and block: device milliseconds per frame, from CUDA
events around the block on the library's stream; reported as the median and interquartile range over the blocks.  Also
whether both libraries leave the same pixels and draw order on the path's last frame.  The card's name and power limit are
read in the same run.  Each library follows the same camera path, so the two keep the same draw-order history.

    python tools/time_frame_ab.py --baseline-lib OTHER/libgsplat_b200.so [--blocks 10] [--frames 20] [--workload metric]
        [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from time_array_target import card, spread  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", required=True, help="libgsplat_b200.so of the build to compare against")
    ap.add_argument("--blocks", type=int, default=10, help="blocks per library (alternating)")
    ap.add_argument("--frames", type=int, default=20, help="timed frames per block")
    ap.add_argument("--warmup", type=int, default=5, help="untimed frames per library before the first block")
    ap.add_argument("--workload", default="metric")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import numpy as np
    import torch
    import bench
    import unitygaussiansplatting_b200 as g
    from unitygaussiansplatting_b200 import _native as N
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    n, quality, w, h, fov, seed, _ = bench.WORKLOADS[args.workload]
    asset = bench.get_asset(n, quality, seed)
    this = N.native()
    libs = {"baseline": N._bind(C.CDLL(str(Path(args.baseline_lib).resolve())), N.NATIVE_SYMBOLS), "this": this}
    stream = torch.cuda.Stream(priority=-1)   # as bench.py
    ctxs, rs, rts = {}, {}, {}
    for name, lib in libs.items():
        N._native = lib   # the context and renderer made now keep this library
        ctxs[name] = g.GaussianSplatContext(0, stream.cuda_stream)
        rs[name] = g.GaussianSplatRenderer(asset, ctxs[name])
        rts[name] = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")
    N._native = this
    k = {name: 0 for name in libs}   # each library follows the same camera path, so both keep the same draw-order history

    def frames(name, count):
        for _ in range(count):
            cam = bench.orbit_camera(k[name], w, h, fov)
            k[name] += 1
            rs[name].SortAndRenderSplats(cam, rt=rts[name])

    acc = {name: [] for name in libs}
    with torch.cuda.stream(stream):
        for name in libs:
            frames(name, args.warmup)
        torch.cuda.synchronize()
        for _b in range(args.blocks):
            for name in libs:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                frames(name, args.frames)
                e1.record(stream)
                torch.cuda.synchronize()
                acc[name].append(e0.elapsed_time(e1) / args.frames)
        for name in libs:
            frames(name, 1)
        torch.cuda.synchronize()
    same_rt = bool(torch.equal(rts["baseline"].view(torch.int16), rts["this"].view(torch.int16)))
    same_order = bool(np.array_equal(rs["baseline"].readback_order(), rs["this"].readback_order()))
    res = {"what": "gs_frame, one object: device ms per frame (CUDA events around each block), alternating blocks",
           "workload": "%s: %d splats, %s, %dx%d, bench.orbit_camera, device render target" % (args.workload, n, quality, w, h),
           "baseline_lib": str(args.baseline_lib), "blocks": args.blocks, "frames_per_block": args.frames, **card(),
           "same_pixels_on_a_common_frame": same_rt, "same_order_on_a_common_frame": same_order,
           "frame_ms": {name: spread(v) for name, v in acc.items()}}
    for name in libs:
        rs[name].Dispose()
        ctxs[name].close()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
