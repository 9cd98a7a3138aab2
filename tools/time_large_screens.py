#!/usr/bin/env python
"""Large screens: the bench.py metric scene (6,131,954 splats, Medium, bench.orbit_camera) at 7680x4320, 8192x8192, 15360x8640
and 16384x16384, into a device RGBA16F render target.

Per size, on a context of its own (so that its bin list starts at the capacity rule's clamp(8 N, 4 Mi, 768 Mi) entries):
  - the first frame's bin-list entries (GsStageTimes.tile_entries), whether they outgrew the rule's capacity, and how many
    more kernels the first frame launched than a later one (4 when it binned twice: bin_emit, look-back clear, 2 sort passes);
  - the stage times of later frames (library device events, timing on), median and interquartile range, and the host-clock
    frame time (call to the end of a synchronise, timing off);
  - in a separate run under torch.profiler: the time of k_tile_order (the one-CTA raster launch order) against the raster
    kernel k_raster, per frame.
The card's name and power limit are read in the same run.

    python tools/time_large_screens.py [--frames 10] [--warmup 3] [--out profiles/h100_large_screens.json]
"""
import argparse
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from time_array_target import card, spread  # noqa: E402  (tools/ is this script's directory)

SIZES = [(7680, 4320), (8192, 8192), (15360, 8640), (16384, 16384)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10, help="timed frames per size (and as many with the host clock)")
    ap.add_argument("--warmup", type=int, default=3, help="untimed frames per size after the first")
    ap.add_argument("--profile-frames", type=int, default=3, help="frames per size under torch.profiler")
    ap.add_argument("--sizes", default=None, help="comma-separated WxH list instead of the default four")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import torch
    import bench
    import unitygaussiansplatting_b200 as g
    from torch.profiler import ProfilerActivity, profile
    from unitygaussiansplatting_b200._native import GsError
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    sizes = [tuple(int(v) for v in s.lower().split("x")) for s in args.sizes.split(",")] if args.sizes else SIZES
    n, quality, _w, _h, fov, seed, _ = bench.WORKLOADS["metric"]
    asset = bench.get_asset(n, quality, seed)
    rule = min(max(8 * n, 4 << 20), 768 << 20)
    res = {"what": "the metric scene on large screens: bin-list size and growth, stage times, k_tile_order's share of the raster",
           "scene": "%d splats, %s, bench.orbit_camera (fov %.5f)" % (n, quality, fov), "target": "device tensor, RGBA16F",
           "capacity_rule_entries": rule, **card(),
           "fields": "stages_ms: library device events (timing on); frame_ms: host clock from the call to the end of a synchronise "
                     "(timing off); profile: torch.profiler kernel times per frame",
           "sizes": {}}
    frame_no = 0
    for w, h in sizes:
        ctx = g.GaussianSplatContext(0)
        r = g.GaussianSplatRenderer(asset, ctx)
        rt = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")

        def frame():
            nonlocal frame_no
            r.SortAndRenderSplats(bench.orbit_camera(frame_no, w, h, fov), rt=rt)
            frame_no += 1

        l0 = ctx.stage_times().kernel_launches
        frame()
        try:
            ctx.sync()
        except GsError as e:   # more than 768 Mi entries: the frame is reported, nothing below is measured
            res["sizes"]["%dx%d" % (w, h)] = {"error": str(e), "tile_entries_first_frame": int(ctx.stage_times().tile_entries)}
            print(json.dumps(res["sizes"]["%dx%d" % (w, h)]), flush=True)
            r.Dispose()
            ctx.close()
            continue
        st = ctx.stage_times()
        first_launches, entries_first = st.kernel_launches - l0, int(st.tile_entries)
        for _ in range(args.warmup):
            frame()
        ctx.sync()
        l0 = ctx.stage_times().kernel_launches
        frame()
        ctx.sync()
        steady_launches = ctx.stage_times().kernel_launches - l0
        acc = {k: [] for k in ("distances_ms", "sort_ms", "view_ms", "bin_ms", "raster_ms", "total_ms")}
        entries, launches = [], []
        ctx.set_timing(True)
        for _ in range(args.frames):
            l0 = ctx.stage_times().kernel_launches
            frame()
            t = ctx.stage_times()
            for k in acc:
                acc[k].append(getattr(t, k))
            entries.append(int(t.tile_entries))
            launches.append(t.kernel_launches - l0)
        ctx.set_timing(False)
        host = []
        for _ in range(args.frames):
            t0 = time.perf_counter()
            frame()
            ctx.sync()
            host.append((time.perf_counter() - t0) * 1e3)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_frames):
                frame()
            ctx.sync()
            torch.cuda.synchronize()
        kern = {"k_tile_order": [0.0, 0], "k_raster": [0.0, 0]}
        for item in prof.key_averages():   # kernels launched by the library have no torch op above them: they are keys of their own
            for name in kern:
                if name in item.key:
                    kern[name][0] += item.device_time_total / 1e3
                    kern[name][1] += item.count
        tile_order_ms = kern["k_tile_order"][0] / args.profile_frames
        raster_ms = kern["k_raster"][0] / args.profile_frames
        rtiles = -(-w // 16) * -(-h // 64) * 4
        res["sizes"]["%dx%d" % (w, h)] = {
            "bins": -(-w // 64) * -(-h // 64), "raster_tiles": rtiles,
            "tile_entries_first_frame": entries_first, "entries_per_splat": entries_first / n,
            "list_grew": entries_first > rule, "extra_launches_first_frame": first_launches - steady_launches,
            "tile_entries_timed": spread(entries), "timed_frames_binned_twice": sum(1 for x in launches if x > min(launches + [steady_launches])),
            "stages_ms": {k: spread(v) for k, v in acc.items()}, "frame_ms": spread(host),
            "profile": {"frames": args.profile_frames, "k_tile_order_ms": tile_order_ms, "k_raster_ms": raster_ms,
                        "kernels_seen": {k: v[1] for k, v in kern.items()},
                        "k_tile_order_share_of_raster": tile_order_ms / (tile_order_ms + raster_ms) if raster_ms else None},
        }
        print(json.dumps({"%dx%d" % (w, h): res["sizes"]["%dx%d" % (w, h)]}), flush=True)
        r.Dispose()
        ctx.close()
        del rt
        torch.cuda.empty_cache()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
