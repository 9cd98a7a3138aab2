#!/usr/bin/env python
"""Several cameras on one GPU: the camera loop (gs_frame_objects per camera) against one gs_frame_cameras call (one bin list,
one bin sort and one raster pass per camera run).

Workloads, each with bench.orbit_camera as the centre of its rig:
  stereo    the bench.py metric scene (6,131,954 splats, Medium) seen by two 1920x1080 cameras 6.4 cm apart;
  quad      the metric scene plus a 2 M VeryHigh object beside it, seen by four 960x540 cameras on a 0.5 m square;
  eight     the metric scene seen by eight 480x270 cameras on a 0.5 m circle.
Each arm owns its copy of every object on one context and draws every camera into a device render target and a device camera
target.  Before timing, both arms draw the same frame and every target and draw order is asserted bit-identical.  The arms
then run in alternating blocks of frames in one process.  Per arm: the frame total (host clock from the first call to the end
of a full synchronise, timing off), and with timing on: the device time of the whole frame (CUDA events on the context stream
around all of the arm's calls; the library's own events stay off, since reading them waits for the device between the loop's
calls), and in separate frames the raster time from the library's events (timing on, summed over the loop's calls).  The device
time before the raster (sorts, view-calcs, bin emits and bin sort) is about the difference of the two.  A camera run emits each
object's bin entries right after its view-calc, between the sorts, so its binning cannot be timed apart from them.  Medians and interquartile ranges, with the card's name and power limit read in the same run.

    python tools/time_frame_cameras.py [--blocks 6] [--frames 10] [--out profiles/h100_frame_cameras.json]
"""
import argparse
import ctypes as C
import json
import sys
import time
from dataclasses import replace
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from time_array_target import card, spread  # noqa: E402  (tools/ is this script's directory)


def rig(cam, offsets):
    """Cameras at cam's position plus each (right, up) offset in metres, all looking where cam looks."""
    import numpy as np
    right, up = cam.rotation[:, 0], cam.rotation[:, 1]
    return [replace(cam, position=np.asarray(cam.position, np.float64) + dx * right + dy * up) for dx, dy in offsets]


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
    n, quality, _w, _h, fov, seed, _ = bench.WORKLOADS["metric"]
    metric = bench.get_asset(n, quality, seed)
    side = g.synthetic_asset(g.SCENE_CLUSTERED, 2_000_000, 0x5EED00B2, "VeryHigh")
    ring = [(0.25 * np.cos(2 * np.pi * k / 8), 0.25 * np.sin(2 * np.pi * k / 8)) for k in range(8)]
    workloads = {   # objects, camera size, camera offsets
        "stereo": ([(metric, None)], (1920, 1080), [(-0.032, 0.0), (0.032, 0.0)]),
        "quad": ([(metric, None), (side, g.trs(position=(2.6, 0.2, 0.8), scale=(0.6, 0.6, 0.6)))], (960, 540),
                 [(-0.25, -0.25), (0.25, -0.25), (-0.25, 0.25), (0.25, 0.25)]),
        "eight": ([(metric, None)], (480, 270), ring),
    }
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    lib = N.native()
    ctx = g.GaussianSplatContext(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def next_sort(r):
        s = 1 if r.m_FrameCounter % max(1, int(r.m_SortNthFrame)) == 0 else 0
        r.m_FrameCounter += 1
        return s

    def draw(arm, rs, cams, ims, timed):
        """One frame of every camera; returns (host ms to a full synchronise, device ms of the frame, raster ms).  timed:
        None, "events" (the frame's device time) or "library" (the library's raster events)."""
        actives = [g.GatherSplatsForCamera(rs, cam) for cam in cams]
        k = sum(len(a) for a in actives)
        fps, assets, ds = (N.GsFrameParams * k)(), (C.c_void_p * k)(), (C.c_int32 * k)()
        i = 0
        for active, cam in zip(actives, cams):
            for r in active:
                fps[i], assets[i], ds[i] = r.frame_params(cam), r._asset.value, next_sort(r)
                i += 1
        t0 = time.perf_counter()
        raster_ms = 0.0
        if timed == "events":
            ev0.record(stream)
        if arm == "loop":
            off = 0
            for c, active in enumerate(actives):
                m = len(active)
                N.check(ctx.handle, lib.gs_frame_objects(ctx.handle, m, C.cast(C.byref(assets, off * 8), C.POINTER(C.c_void_p)),
                                                         C.cast(C.byref(fps, off * C.sizeof(N.GsFrameParams)), C.POINTER(N.GsFrameParams)),
                                                         C.cast(C.byref(ds, off * 4), C.POINTER(C.c_int32)), N.GsRenderOptions(),
                                                         ims[c][0], ims[c][1]))
                off += m
                if timed == "library":
                    raster_ms += ctx.stage_times().raster_ms
        else:
            PI = C.POINTER(N.GsImage)
            a = (PI * len(cams))(*[C.pointer(x) for x, _ in ims])
            b = (PI * len(cams))(*[C.pointer(y) for _, y in ims])
            counts = (C.c_uint32 * len(cams))(*[len(x) for x in actives])
            N.check(ctx.handle, lib.gs_frame_cameras(ctx.handle, len(cams), counts, assets, fps, ds, N.GsRenderOptions(), a, b))
            if timed == "library":
                raster_ms = ctx.stage_times().raster_ms
        dev_ms = 0.0
        if timed == "events":
            ev1.record(stream)
        ctx.sync()
        if timed == "events":
            dev_ms = ev0.elapsed_time(ev1)
        return (time.perf_counter() - t0) * 1e3, dev_ms, raster_ms

    res = {"what": "several cameras on one GPU: gs_frame_objects per camera vs one gs_frame_cameras call",
           "blocks": args.blocks, "frames_per_block": args.frames, **card(),
           "fields": "frame_ms: host clock from the first call to the end of a full synchronise, timing off; device_frame_ms: CUDA "
                     "events on the context stream around the frame's calls, library timing off; raster_ms: the library's raster "
                     "events in separate frames, summed over the loop's calls",
           "workloads": {}}
    for name, (objs, (w, h), offsets) in workloads.items():
        arms, images = {}, {}
        for arm in ("loop", "call"):
            rs = []
            for asset, m in objs:
                r = g.GaussianSplatRenderer(asset, ctx)
                if m is not None:
                    r.localToWorldMatrix = m.astype(np.float32)
                rs.append(r)
            arms[arm] = rs
            tensors = [(torch.zeros((h, w, 4), dtype=torch.float16, device="cuda"), torch.zeros((h, w, 4), dtype=torch.float16, device="cuda"))
                       for _ in offsets]
            images[arm] = (tensors, [(_image(x, w, h), _image(y, w, h)) for x, y in tensors])

        def cams(f):
            return rig(bench.orbit_camera(f, w, h, fov), offsets)

        # the same frame from both arms: bit-identical targets and draw orders
        for arm in arms:
            draw(arm, arms[arm], cams(0), images[arm][1], None)
        for (x0, y0), (x1, y1) in zip(images["loop"][0], images["call"][0]):
            assert torch.equal(x0.view(torch.int16), x1.view(torch.int16)), name + ": render targets differ"
            assert torch.equal(y0.view(torch.int16), y1.view(torch.int16)), name + ": camera targets differ"
        for a, b in zip(arms["loop"], arms["call"]):
            assert np.array_equal(a.readback_order(), b.readback_order()), name + ": draw orders differ"
        frame_no = 1
        for arm in arms:
            for _ in range(args.warmup):
                draw(arm, arms[arm], cams(frame_no), images[arm][1], None)
                frame_no += 1
        acc = {arm: {"frame_ms": [], "device_frame_ms": [], "raster_ms": []} for arm in arms}
        for _b in range(args.blocks):
            for arm in arms:
                ctx.set_timing(False)
                for _ in range(args.frames):
                    acc[arm]["frame_ms"].append(draw(arm, arms[arm], cams(frame_no), images[arm][1], None)[0])
                    frame_no += 1
                for _ in range(args.frames):
                    acc[arm]["device_frame_ms"].append(draw(arm, arms[arm], cams(frame_no), images[arm][1], "events")[1])
                    frame_no += 1
                ctx.set_timing(True)
                for _ in range(args.frames):
                    acc[arm]["raster_ms"].append(draw(arm, arms[arm], cams(frame_no), images[arm][1], "library")[2])
                    frame_no += 1
        ctx.set_timing(False)
        res["workloads"][name] = {"objects": [a.splatCount for a, _m in objs], "cameras": len(offsets), "screen": "%dx%d" % (w, h),
                                  "bit_identical": True,
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
