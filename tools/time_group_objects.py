#!/usr/bin/env python
"""Two splat objects per camera: one GPU (SortAndRenderSplatsMulti, one gs_frame per object) against the group path
(gs_group_frame_objects, one call for both objects).

Workload: the bench.py metric scene (6,131,954 splats, Medium, 1920x1080, orbiting camera) plus a second object of about 2 M
VeryHigh splats beside it.  The arms run in alternating blocks of frames in one process:
  single   one context, GaussianSplatRenderer per object, SortAndRenderSplatsMulti into a device render target;
  group1   a group of one (gs_group_create) and its second object, GaussianSplatGroup.SortAndRenderSplatsMulti;
  group2 / group4   real groups over 2 / 4 devices, when the machine has them (otherwise "not measured").
Per arm: the frame total (host clock from the call to the end of a full synchronise, timing off) and the raster time (library
device events with timing on: gs_get_stage_times raster_ms summed over the two gs_frame calls; GsGroupStats raster_ms of the
group call), as median and interquartile range, plus the card's name and power limit read in the same run.

    python tools/time_group_objects.py [--blocks 6] [--frames 10] [--out profiles/h100_group_objects.json]
"""
import argparse
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from time_array_target import card, spread  # noqa: E402  (tools/ is this script's directory)

SECOND_N, SECOND_SEED = 2_000_000, 0x5EED00B2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=6, help="blocks per arm (alternating)")
    ap.add_argument("--frames", type=int, default=10, help="frames per block, each timed once with timing off and once with it on")
    ap.add_argument("--warmup", type=int, default=4, help="untimed frames per arm before the first block")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import numpy as np
    import torch
    import bench
    import unitygaussiansplatting_b200 as g
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    n, quality, w, h, fov, seed, _ = bench.WORKLOADS["metric"]
    first = bench.get_asset(n, quality, seed)
    second = g.synthetic_asset(g.SCENE_CLUSTERED, SECOND_N, SECOND_SEED, "VeryHigh")
    beside = g.trs(position=(2.6, 0.2, 0.8), scale=(0.6, 0.6, 0.6)).astype(np.float32)

    ctx = g.GaussianSplatContext(0)
    singles = [g.GaussianSplatRenderer(first, ctx), g.GaussianSplatRenderer(second, ctx)]
    singles[1].localToWorldMatrix = beside
    rt_single = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")

    ndev = torch.cuda.device_count()
    groups = {"group1": [0]}
    for size in (2, 4):
        if ndev >= size:
            groups["group%d" % size] = list(range(size))
    arms = {}
    for name, devs in groups.items():
        grp = GaussianSplatGroup.create(first, devs)
        obj = grp.add_object(second)
        obj.localToWorldMatrix = beside
        rts = [torch.zeros((h, w, 4), dtype=torch.float16, device="cuda:%d" % d) for d in devs]
        arms[name] = (grp, obj, rts)

    k = 0

    def frame(arm, timed):
        """One frame of `arm`; returns (host ms to a full synchronise, raster ms or None)."""
        nonlocal k
        cam = bench.orbit_camera(k, w, h, fov)
        k += 1
        t0 = time.perf_counter()
        raster = None
        if arm == "single":
            if timed:
                raster = 0.0
                for i, r in enumerate(g.GatherSplatsForCamera(singles, cam)):   # SortAndRenderSplatsMulti, reading each call's times
                    r.load_rt = i > 0
                    r.SortAndRenderSplats(cam, rt=rt_single)
                    raster += ctx.stage_times().raster_ms
                    r.load_rt = False
            else:
                g.SortAndRenderSplatsMulti(singles, cam, rt_single)
            ctx.sync()
        else:
            grp, obj, rts = arms[arm]
            grp.SortAndRenderSplatsMulti([grp, obj], cam, rts=rts)
            grp.sync()
            if timed:
                raster = grp.stats().raster_ms
        return (time.perf_counter() - t0) * 1e3, raster

    def set_timing(on):
        ctx.set_timing(on)
        for grp, _obj, _rts in arms.values():
            for c in grp.contexts:
                c.set_timing(on)

    names = ["single"] + list(arms)
    for arm in names:
        for _ in range(args.warmup):
            frame(arm, False)
    acc = {arm: {"frame_ms": [], "raster_ms": []} for arm in names}
    for _b in range(args.blocks):
        for arm in names:
            set_timing(False)
            for _ in range(args.frames):
                acc[arm]["frame_ms"].append(frame(arm, False)[0])
            set_timing(True)
            for _ in range(args.frames):
                acc[arm]["raster_ms"].append(frame(arm, True)[1])
    set_timing(False)
    res = {"what": "two splat objects per camera: single-GPU SortAndRenderSplatsMulti vs gs_group_frame_objects",
           "workload": "%d splats %s + %d splats VeryHigh beside it (trs (2.6, 0.2, 0.8), scale 0.6), %dx%d, bench.orbit_camera"
                       % (n, quality, SECOND_N, w, h),
           "blocks": args.blocks, "frames_per_block": args.frames, "devices": ndev, **card(),
           "fields": "frame_ms: host clock from the call to the end of a full synchronise, timing off; raster_ms: library device events",
           "arms": {arm: {f: spread(v) for f, v in fields.items()} for arm, fields in acc.items()}}
    for size in (2, 4):
        if "group%d" % size not in arms:
            res["arms"]["group%d" % size] = "not measured: this machine has %d device(s)" % ndev
    for grp, _obj, _rts in arms.values():
        grp.close()
    for r in singles:
        r.Dispose()
    ctx.close()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
