#!/usr/bin/env python
"""Where a frame's time goes between its kernels: a torch.profiler trace (CUDA activities only) of orbit frames of the bench.py
metric workload (6,131,954 splats, Medium, 1920x1080, device render target), run back to back as bench.py runs them.

Per node of the trace (kernel, memset, copy): its name, start (us from the frame's first node) and duration.  Per frame:
  span_us            first node's start to last node's end
  busy_us            time some node of the frame runs (union of the nodes' intervals)
  idle_us            time between consecutive nodes where none runs (span - busy)
  gap_before_us      from the previous frame's last node to this frame's first
  memset_us          time in memset nodes, and their count
  tile_order_us      k_tile_order
  view_pass3_overlap_us  how long k_calc_view runs beside the depth sort's last pass (the frame's fourth k_onesweep)
The card's name and power limit are read in the same run.

    python tools/time_launch_chain.py [--frames 20] [--warmup 10] [--workload metric] [--out FILE.json]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from time_array_target import card, spread  # noqa: E402


def short_name(ev):
    name = ev["name"]
    if ev.get("cat") == "gpu_memset":
        return "memset"
    if ev.get("cat") == "gpu_memcpy":
        return "memcpy"
    name = name.split("(")[0]
    if name.startswith("void "):
        name = name[5:]
    return name.replace("gs::", "")


def frames_of(nodes):
    """Consecutive nodes split after each raster kernel: one draw per frame."""
    frames, cur = [], []
    for nd in nodes:
        cur.append(nd)
        if nd["name"].startswith("k_raster"):
            frames.append(cur)
            cur = []
    return frames


def frame_totals(fr, prev_end):
    t0 = fr[0]["t0"]
    end = max(nd["t0"] + nd["dur"] for nd in fr)
    busy, run_end = 0.0, t0
    for nd in sorted(fr, key=lambda x: x["t0"]):
        a, b = max(nd["t0"], run_end), nd["t0"] + nd["dur"]
        if b > a:
            busy += b - a
        run_end = max(run_end, b)
    sweeps = [nd for nd in fr if nd["name"].startswith("k_onesweep")]
    view = [nd for nd in fr if nd["name"].startswith("k_calc_view")]
    overlap = 0.0
    if len(sweeps) >= 4 and view:
        p3, v = sweeps[3], view[0]
        overlap = max(0.0, min(p3["t0"] + p3["dur"], v["t0"] + v["dur"]) - max(p3["t0"], v["t0"]))
    mem = [nd for nd in fr if nd["name"] == "memset"]
    return {"nodes": len(fr), "kernels": sum(nd["name"] not in ("memset", "memcpy") for nd in fr),
            "span_us": end - t0, "busy_us": busy, "idle_us": (end - t0) - busy,
            "gap_before_us": None if prev_end is None else t0 - prev_end,
            "memsets": len(mem), "memset_us": sum(nd["dur"] for nd in mem),
            "tile_order_us": sum(nd["dur"] for nd in fr if nd["name"].startswith("k_tile_order")),
            "view_pass3_overlap_us": overlap}, end


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20, help="traced frames")
    ap.add_argument("--warmup", type=int, default=10, help="untraced frames before them")
    ap.add_argument("--workload", default="metric")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    import unitygaussiansplatting_b200 as g
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    n, quality, w, h, fov, seed, _ = bench.WORKLOADS[args.workload]
    asset = bench.get_asset(n, quality, seed)
    stream = torch.cuda.Stream(priority=-1)   # as bench.py
    ctx = g.GaussianSplatContext(0, stream.cuda_stream)
    r = g.GaussianSplatRenderer(asset, ctx)
    cams = [bench.orbit_camera(k, w, h, fov) for k in range(args.warmup + args.frames)]
    fps = [r.frame_params(c) for c in cams]
    with torch.cuda.stream(stream):
        rt = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")
        for k in range(args.warmup):
            r.SortAndRenderSplats(cams[k], rt=rt, fp=fps[k])
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in range(args.warmup, args.warmup + args.frames):
                r.SortAndRenderSplats(cams[k], rt=rt, fp=fps[k])
            torch.cuda.synchronize()
    r.Dispose()
    ctx.close()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
    evs = trace["traceEvents"] if isinstance(trace, dict) else trace
    nodes = sorted(({"name": short_name(e), "t0": float(e["ts"]), "dur": float(e.get("dur", 0.0))}
                    for e in evs if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")),
                   key=lambda x: x["t0"])
    frames = frames_of(nodes)
    if len(frames) != args.frames:
        raise SystemExit("expected %d frames in the trace, found %d" % (args.frames, len(frames)))
    totals, prev_end = [], None
    for fr in frames:
        t, prev_end = frame_totals(fr, prev_end)
        totals.append(t)
    keys = [k for k in totals[0] if k not in ("nodes", "kernels", "memsets")]
    res = {"what": "torch.profiler trace (CUDA activities) of gs_frame, back-to-back orbit frames: nodes and the time between them",
           "workload": "%s: %d splats, %s, %dx%d, bench.orbit_camera frames %d..%d, device render target"
                       % (args.workload, n, quality, w, h, args.warmup, args.warmup + args.frames - 1),
           **card(),
           "per_frame_median_us": {k: statistics.median(t[k] for t in totals if t[k] is not None) for k in keys},
           "per_frame_spread_us": {k: spread([t[k] for t in totals if t[k] is not None]) for k in keys},
           "nodes_per_frame": totals[0]["nodes"], "kernels_per_frame": totals[0]["kernels"], "memsets_per_frame": totals[0]["memsets"],
           "frames": [{"totals": t, "nodes": [{"name": nd["name"], "start_us": round(nd["t0"] - fr[0]["t0"], 3), "dur_us": round(nd["dur"], 3)}
                                              for nd in fr]} for t, fr in zip(totals, frames)]}
    text = json.dumps(res, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "frames"}, indent=1))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
