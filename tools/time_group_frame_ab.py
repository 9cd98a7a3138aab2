#!/usr/bin/env python
"""gs_group_frame with one object on a group of one: this tree's library against another build of it (e.g. the previous
commit's), loaded side by side in one process and timed in alternating blocks.

Workload: the bench.py metric scene (6,131,954 splats, Medium, 1920x1080, orbiting camera) into a device render target.  Per
library: host milliseconds per frame from the call to the end of gs_group_sync (median and interquartile range), and whether
both libraries leave the same pixels on a final common frame.  The card's name and power limit are read in the same run.

    python tools/time_group_frame_ab.py --baseline-lib OTHER/unitygaussiansplatting_b200/libgsplat_b200.so [--blocks 8] [--frames 20]
        [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from time_array_target import card, spread  # noqa: E402  (tools/ is this script's directory)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", required=True, help="libgsplat_b200.so of the build to compare against")
    ap.add_argument("--blocks", type=int, default=8, help="blocks per library (alternating)")
    ap.add_argument("--frames", type=int, default=20, help="timed frames per block")
    ap.add_argument("--warmup", type=int, default=5, help="untimed frames per library before the first block")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import torch
    import bench
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    baseline = C.CDLL(str(Path(args.baseline_lib).resolve()))
    # bind only what gs_group_frame needs and both builds export
    common = {k: v for k, v in N.NATIVE_SYMBOLS.items() if hasattr(baseline, k)}
    libs = {"baseline": N._bind(baseline, common), "this": N.native()}
    n, quality, w, h, fov, seed, _ = bench.WORKLOADS["metric"]
    asset = bench.get_asset(n, quality, seed)
    grps, rts = {}, {}
    for name, lib in libs.items():
        handle = C.c_void_p()
        N.check(None, lib.gs_group_create((C.c_int * 1)(0), 1, 0, C.byref(handle)))
        grps[name] = GaussianSplatGroup(handle, asset, lib)
        rts[name] = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")
    k = 0

    def frame(name, cam=None):
        nonlocal k
        if cam is None:
            cam = bench.orbit_camera(k, w, h, fov)
            k += 1
        t0 = time.perf_counter()
        grps[name].SortAndRenderSplats(cam, rts=[rts[name]])
        N.check(None, libs[name].gs_group_sync(grps[name].handle))
        return (time.perf_counter() - t0) * 1e3

    for name in libs:
        for _ in range(args.warmup):
            frame(name)
    acc = {name: [] for name in libs}
    for _b in range(args.blocks):
        for name in libs:
            for _ in range(args.frames):
                acc[name].append(frame(name))
    cam = bench.orbit_camera(k, w, h, fov)
    for name in libs:
        frame(name, cam)
    res = {"what": "gs_group_frame, one object, group of one: host ms per frame to gs_group_sync, alternating blocks",
           "workload": "%d splats, %s, %dx%d, bench.orbit_camera, device render target" % (n, quality, w, h),
           "baseline_lib": str(args.baseline_lib), "blocks": args.blocks, "frames_per_block": args.frames, **card(),
           "same_pixels_on_a_common_frame": bool(torch.equal(rts["baseline"], rts["this"])),
           "frame_ms": {name: spread(v) for name, v in acc.items()}}
    for grp in grps.values():
        grp.close()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
