#!/usr/bin/env python
"""Where the time of a depth-sort pass goes, per 8192-pair tile (a diagnostic, not a benchmark).

Runs the metric frame's orbit with GS_SORT_PHASES=1, which makes the depth sort launch an instantiation of k_onesweep that
records %globaltimer per tile at tile start, keys landed (after the tile histogram), prefix resolved and scatter done, plus
the look-back's polls and status words summed (gs_debug_sort_phases).  Per pass it prints the median and p90 of
  keys    keys landed - tile start (a CTA's next tile cannot start before its current one is done: the later of the two)
  prefix  prefix resolved - keys landed (ranking, the block scans of the tile's digit bases, then the look-back)
  rank    scatter done - prefix resolved (shared-memory scatter, global write-out)
  tile    scatter done - tile start
and the look-back polls against the tile index, for the first wave (the first 2 x SMs tiles) and the later ones.
The timed instantiation is not the product's: its absolute times are only indicative.

usage: time_sort_phases.py [workload=metric] [frames=10] [out.json]
"""
import json
import os
import sys
from pathlib import Path

os.environ["GS_SORT_PHASES"] = "1"
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import ctypes as C

import numpy as np

import bench

WORDS = 8


def pct(a, q):
    return float(np.percentile(a, q)) / 1e3 if len(a) else float("nan")   # ns -> us


def pass_report(rec, waves_tiles):
    rec = rec[rec[:, 3] != 0]                       # tiles this pass has
    t0, tk, tp, td = (rec[:, i].astype(np.int64) for i in range(4))
    tile, cta = rec[:, 6].astype(np.int64), (rec[:, 7] >> 32).astype(np.int64)
    start = t0.copy()
    order = np.lexsort((t0, cta))                    # per CTA in the order it took its tiles
    same = cta[order][1:] == cta[order][:-1]
    prev_done = np.zeros_like(td)
    prev_done[order[1:][same]] = td[order[:-1][same]]
    start = np.maximum(start, prev_done)
    ph = {"keys": tk - start, "prefix": tp - tk, "rank": td - tp, "tile": td - start}
    out = {"tiles": int(len(rec)), "pass_us": float(td.max() - t0.min()) / 1e3}
    for k, v in ph.items():
        out[k] = {"median_us": pct(v, 50), "p90_us": pct(v, 90)}
    polls = rec[:, 4].astype(np.int64)
    first = tile < waves_tiles
    buckets = []
    for lo in range(0, int(waves_tiles), 33):
        m = (tile >= lo) & (tile < lo + 33)
        if m.any():
            buckets.append({"tiles": [lo, lo + 32], "polls_median": float(np.median(polls[m])), "polls_max": int(polls[m].max()),
                            "prefix_median_us": pct(tp[m] - tk[m], 50)})
    out["first_wave"] = {"polls_median": float(np.median(polls[first])), "polls_p90": pct(polls[first], 90) * 1e3,
                         "polls_max": int(polls[first].max()), "by_tile": buckets}
    if (~first).any():
        out["later_waves"] = {"polls_median": float(np.median(polls[~first])), "polls_p90": pct(polls[~first], 90) * 1e3,
                              "polls_max": int(polls[~first].max()), "prefix_median_us": pct(tp[~first] - tk[~first], 50)}
    return out


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "metric"
    frames = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    out_path = sys.argv[3] if len(sys.argv) > 3 else None
    import torch
    import unitygaussiansplatting_b200 as g
    from unitygaussiansplatting_b200 import _native as N

    n, quality, w, h, fov, seed, _ = bench.WORKLOADS[name]
    asset = bench.get_asset(n, quality, seed)
    ctx = g.GaussianSplatContext(0)
    r = g.GaussianSplatRenderer(asset, ctx)
    rt = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for k in range(5):
        r.SortAndRenderSplats(bench.orbit_camera(k, w, h, fov), rt=rt)
    per_frame = []
    for k in range(5, 5 + frames):
        r.SortAndRenderSplats(bench.orbit_camera(k, w, h, fov), rt=rt)
        tiles = C.c_uint32(0)
        N.check(ctx.handle, N.native().gs_debug_sort_phases(ctx.handle, None, 0, C.byref(tiles)))
        buf = np.zeros(4 * tiles.value * WORDS, np.uint64)
        N.check(ctx.handle, N.native().gs_debug_sort_phases(ctx.handle, buf.ctypes.data, buf.size, C.byref(tiles)))
        per_frame.append(buf.reshape(4, tiles.value, WORDS))
    report = {"workload": name, "frames": frames, "gpu": torch.cuda.get_device_name(0), "sms": sms, "passes": []}
    for p in range(4):
        rec = np.concatenate([f[p] for f in per_frame])
        # tile statistics pool all frames; the pass time is the median over frames
        rep = pass_report(rec, 2 * sms)
        rep["pass_us"] = float(np.median([pass_report(f[p], 2 * sms)["pass_us"] for f in per_frame]))
        report["passes"].append(rep)
    for p, rep in enumerate(report["passes"]):
        print("pass %d: %d tiles, %.1f us | median/p90 us: keys %.2f/%.2f  prefix %.2f/%.2f  rank %.2f/%.2f  tile %.2f/%.2f" % (
            p, rep["tiles"] // frames, rep["pass_us"], rep["keys"]["median_us"], rep["keys"]["p90_us"], rep["prefix"]["median_us"],
            rep["prefix"]["p90_us"], rep["rank"]["median_us"], rep["rank"]["p90_us"], rep["tile"]["median_us"], rep["tile"]["p90_us"]))
        fw = rep["first_wave"]
        print("   first wave polls median %.0f p90 %.0f max %d; by tile: %s" % (
            fw["polls_median"], fw["polls_p90"], fw["polls_max"],
            " ".join("%d-%d:%.0f" % (b["tiles"][0], b["tiles"][1], b["polls_median"]) for b in fw["by_tile"])))
        if "later_waves" in rep:
            lw = rep["later_waves"]
            print("   later waves polls median %.0f p90 %.0f max %d, prefix median %.2f us" % (
                lw["polls_median"], lw["polls_p90"], lw["polls_max"], lw["prefix_median_us"]))
    if out_path:
        Path(out_path).parent.mkdir(parents=True, exist_ok=True)
        Path(out_path).write_text(json.dumps(report, indent=1))
    r.Dispose()


if __name__ == "__main__":
    main()
