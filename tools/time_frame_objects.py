#!/usr/bin/env python
"""Several splat objects per camera on one GPU: the per-object loop (gs_frame per object, GS_FLAG_LOAD_RT from the second on,
then gs_composite) against one gs_frame_objects call (one bin list, one raster, one composite).

Workloads, both at 1920x1080 with bench.orbit_camera:
  beside    the bench.py metric scene (6,131,954 splats, Medium) plus about 2 M VeryHigh splats beside it (the
            time_group_objects.py scene);
  overlap   the metric scene plus three 1 M Medium objects that overlap it on screen.
Each arm owns its copy of every object on one context and draws into a device render target and a device camera target.
Before timing, both arms draw the same frame and their targets and draw orders are asserted bit-identical.  The arms then run
in alternating blocks of frames in one process.  Per arm: the frame total (host clock from the call to the end of a full
synchronise, timing off) and the bin and raster times (library device events, timing on; summed over the loop's gs_frame
calls), as median and interquartile range, plus the card's name and power limit read in the same run.

    python tools/time_frame_objects.py [--blocks 6] [--frames 10] [--out profiles/h100_frame_objects.json]
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
    ap.add_argument("--blocks", type=int, default=6, help="blocks per arm and workload (alternating)")
    ap.add_argument("--frames", type=int, default=10, help="frames per block, each timed once with timing off and once with it on")
    ap.add_argument("--warmup", type=int, default=4, help="untimed frames per arm before the first block")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import numpy as np
    import torch
    import bench
    import unitygaussiansplatting_b200 as g
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    n, quality, w, h, fov, seed, _ = bench.WORKLOADS["metric"]
    metric = bench.get_asset(n, quality, seed)
    workloads = {
        "beside": [(metric, None),
                   (g.synthetic_asset(g.SCENE_CLUSTERED, 2_000_000, 0x5EED00B2, "VeryHigh"),
                    g.trs(position=(2.6, 0.2, 0.8), scale=(0.6, 0.6, 0.6)))],
        "overlap": [(metric, None)] + [(g.synthetic_asset(g.SCENE_CLUSTERED, 1_000_000, 0x5EED00C0 + i, "Medium"),
                                        g.trs(position=p, scale=(0.5, 0.5, 0.5)))
                                       for i, p in enumerate([(0.4, 0.1, -0.5), (-0.5, 0.3, 0.2), (0.0, -0.3, 0.6)])],
    }
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    lib = N.native()
    ctx = g.GaussianSplatContext(0)
    rt = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")
    target = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")
    rt_im, tgt_im = _image(rt, w, h), _image(target, w, h)

    def next_sort(r):
        s = 1 if r.m_FrameCounter % max(1, int(r.m_SortNthFrame)) == 0 else 0
        r.m_FrameCounter += 1
        return s

    def draw(arm, rs, cam, timed):
        """One frame; returns (host ms to a full synchronise, bin ms, raster ms) -- the device times only when `timed`."""
        active = g.GatherSplatsForCamera(rs, cam)
        t0 = time.perf_counter()
        bin_ms = raster_ms = 0.0
        if arm == "loop":
            for i, r in enumerate(active):
                fp, opt = r.frame_params(cam), N.GsRenderOptions()
                opt.flags = N.GS_FLAG_LOAD_RT if i else 0
                N.check(ctx.handle, lib.gs_frame(ctx.handle, r._asset, fp, opt, next_sort(r), rt_im, None))
                if timed:
                    t = ctx.stage_times()
                    bin_ms += t.bin_ms
                    raster_ms += t.raster_ms
            N.check(ctx.handle, lib.gs_composite(ctx.handle, rt_im, tgt_im))
        else:
            k = len(active)
            fps, assets, ds = (N.GsFrameParams * k)(), (C.c_void_p * k)(), (C.c_int32 * k)()
            for i, r in enumerate(active):
                fps[i], assets[i], ds[i] = r.frame_params(cam), r._asset.value, next_sort(r)
            N.check(ctx.handle, lib.gs_frame_objects(ctx.handle, k, assets, fps, ds, N.GsRenderOptions(), rt_im, tgt_im))
            if timed:
                t = ctx.stage_times()
                bin_ms, raster_ms = t.bin_ms, t.raster_ms
        ctx.sync()
        return (time.perf_counter() - t0) * 1e3, bin_ms, raster_ms

    res = {"what": "several splat objects per camera on one GPU: per-object gs_frame + gs_composite vs one gs_frame_objects call",
           "screen": "%dx%d, bench.orbit_camera" % (w, h), "blocks": args.blocks, "frames_per_block": args.frames, **card(),
           "fields": "frame_ms: host clock from the call to the end of a full synchronise, timing off; bin_ms / raster_ms: library "
                     "device events (summed over the loop's calls)",
           "workloads": {}}
    for name, objs in workloads.items():
        arms = {}
        for arm in ("loop", "call"):
            rs = []
            for asset, m in objs:
                r = g.GaussianSplatRenderer(asset, ctx)
                if m is not None:
                    r.localToWorldMatrix = m.astype(np.float32)
                rs.append(r)
            arms[arm] = rs
        # the same frame from both arms: bit-identical targets and draw orders
        cam = bench.orbit_camera(0, w, h, fov)
        got = {}
        for arm in ("loop", "call"):
            target.zero_()
            draw(arm, arms[arm], cam, False)
            got[arm] = (rt.clone(), target.clone())
        assert torch.equal(got["loop"][0].view(torch.int16), got["call"][0].view(torch.int16)), name + ": render targets differ"
        assert torch.equal(got["loop"][1].view(torch.int16), got["call"][1].view(torch.int16)), name + ": camera targets differ"
        for a, b in zip(arms["loop"], arms["call"]):
            assert np.array_equal(a.readback_order(), b.readback_order()), name + ": draw orders differ"
        frame_no = 1
        for arm in arms:
            for _ in range(args.warmup):
                draw(arm, arms[arm], bench.orbit_camera(frame_no, w, h, fov), False)
                frame_no += 1
        acc = {arm: {"frame_ms": [], "bin_ms": [], "raster_ms": []} for arm in arms}
        for _b in range(args.blocks):
            for arm in arms:
                ctx.set_timing(False)
                for _ in range(args.frames):
                    acc[arm]["frame_ms"].append(draw(arm, arms[arm], bench.orbit_camera(frame_no, w, h, fov), False)[0])
                    frame_no += 1
                ctx.set_timing(True)
                for _ in range(args.frames):
                    _t, b, r = draw(arm, arms[arm], bench.orbit_camera(frame_no, w, h, fov), True)
                    acc[arm]["bin_ms"].append(b)
                    acc[arm]["raster_ms"].append(r)
                    frame_no += 1
        ctx.set_timing(False)
        res["workloads"][name] = {"objects": [a.splatCount for a, _m in objs], "bit_identical": True,
                                  "arms": {arm: {f: spread(v) for f, v in fields.items()} for arm, fields in acc.items()}}
        for rs in arms.values():
            for r in rs:
                r.Dispose()
    ctx.close()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
