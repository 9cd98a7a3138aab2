#!/usr/bin/env python
"""Drawing into a rectangle of a larger CUDA array (GS_MEM_ARRAY_RECT) against drawing into a whole array.

The bench.py metric scene (6,131,954 splats, Medium, orbiting camera), RGBA16F arrays created with cudaArraySurfaceLoadStore:

  frame_whole:        gs_frame into a whole 1920 x 1080 2-D array (GS_MEM_ARRAY);
  frame_rect_origin:  gs_frame into the 1920 x 1080 rectangle at (0, 0) of a 2560 x 1440 array (an HDRP render target
                      allocated larger than the camera);
  frame_rect_odd:     the same rectangle at (37, 19): a 16 x 16 raster tile's stores straddle more of the array's block-linear
                      tiles;
  quilt_one_array:    a 2 x 2 quilt of 960 x 540 cameras in one gs_frame_cameras call, each camera's render target its tile of
                      one 1920 x 1080 array;
  quilt_four_arrays:  the same four cameras into four separate 960 x 540 arrays.

The frame modes alternate in blocks, and so do the two quilt modes.  Each frame is timed with CUDA events on the library's stream
around everything it enqueues.  The card's name and power limit are read in the same run.

    python tools/time_array_rects.py [--blocks 8] [--frames 15] [--out FILE.json]
"""
import argparse
import dataclasses
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from time_array_target import card, spread  # noqa: E402
from time_layered_targets import make_array  # noqa: E402

import ctypes as C  # noqa: E402


def quilt_cameras(cam, offset=0.08):
    """Four views of the orbit camera, shifted on a 2 x 2 grid across its right and up axes (a small light-field quilt)."""
    right, up = cam.rotation[:, 0], cam.rotation[:, 1]
    return [dataclasses.replace(cam, position=cam.position + (i - 0.5) * offset * right + (0.5 - j) * offset * up)
            for j in range(2) for i in range(2)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=8, help="blocks per mode (alternating)")
    ap.add_argument("--frames", type=int, default=15, help="timed frames per block")
    ap.add_argument("--warmup", type=int, default=5, help="untimed frames per mode before the first block")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import torch
    import bench
    import unitygaussiansplatting_b200 as g
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    n, quality, _w, _h, fov, seed, _ = bench.WORKLOADS["metric"]
    w, h = 1920, 1080
    qw, qh = w // 2, h // 2
    asset = bench.get_asset(n, quality, seed)
    stream = torch.cuda.Stream()
    ctx = g.GaussianSplatContext(0, stream.cuda_stream)
    r = g.GaussianSplatRenderer(asset, ctx)
    cudart = C.CDLL("libcudart.so.12")   # the runtime torch loaded (same soname)
    whole, big, atlas = make_array(cudart, w, h, 0), make_array(cudart, 2560, 1440, 0), make_array(cudart, w, h, 0)
    tiles = [make_array(cudart, qw, qh, 0) for _ in range(4)]
    images = {"frame_whole": g.CudaArrayImage(whole, w, h),
              "frame_rect_origin": g.CudaArrayImage(big, w, h, origin=(0, 0)),
              "frame_rect_odd": g.CudaArrayImage(big, w, h, origin=(37, 19))}
    quilt = {"quilt_one_array": [g.CudaArrayImage(atlas, qw, qh, origin=(i * qw, j * qh)) for j in range(2) for i in range(2)],
             "quilt_four_arrays": [g.CudaArrayImage(t, qw, qh) for t in tiles]}
    k = 0

    def frame(mode):
        nonlocal k
        if mode in images:
            r.SortAndRenderSplats(bench.orbit_camera(k, w, h, fov), rt=images[mode])
        else:
            g.SortAndRenderCameras([r], quilt_cameras(bench.orbit_camera(k, qw, qh, fov)), quilt[mode])
        k += 1

    groups = [list(images), list(quilt)]
    acc = {}
    with torch.cuda.stream(stream):
        for modes in groups:
            for mode in modes:
                for _ in range(args.warmup):
                    frame(mode)
            ctx.sync()
            acc.update({mode: [] for mode in modes})
            for _b in range(args.blocks):
                for mode in modes:
                    evs = []
                    for _ in range(args.frames):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(stream)
                        frame(mode)
                        e1.record(stream)
                        evs.append((e0, e1))
                    stream.synchronize()
                    acc[mode] += [e0.elapsed_time(e1) for e0, e1 in evs]
        ctx.sync()
    r.Dispose()
    ctx.close()
    for a in [whole, big, atlas, *tiles]:
        cudart.cudaFreeArray(C.c_void_p(a))
    res = {"what": "frame device time (CUDA events on the library's stream, ms): gs_frame into a whole 1920x1080 RGBA16F array or "
                   "into a 1920x1080 rectangle of a 2560x1440 one at (0, 0) and at (37, 19); a 2x2 quilt of 960x540 cameras in one "
                   "gs_frame_cameras call into the tiles of one array or into four arrays",
           "workload": "%d splats, %s, bench.orbit_camera; quilt views 8 cm apart" % (n, quality),
           "blocks": args.blocks, "frames_per_block": args.frames, **card(),
           "modes": {mode: spread(v) for mode, v in acc.items()}}
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
