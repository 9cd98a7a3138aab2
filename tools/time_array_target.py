#!/usr/bin/env python
"""Render target in linear device memory vs in a CUDA array (GS_MEM_ARRAY, what an imported graphics render texture is).

The bench.py metric workload (6,131,954 splats, Medium, 1920x1080, orbiting camera) is rendered in alternating blocks of frames:
once with the render target and the camera target as torch RGBA16F tensors, once with both as RGBA16F CUDA arrays created with
cudaArraySurfaceLoadStore (written and read through surface objects).  Per target kind it reports the median and spread of the
library's per-stage device times (gs_get_stage_times: raster_ms, composite_ms, total_ms), plus the card's name and power limit
read in the same run.  Arrays are made with the CUDA runtime torch already loaded.

    python tools/time_array_target.py [--blocks 10] [--frames 20] [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


class _ChannelDesc(C.Structure):
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("z", C.c_int), ("w", C.c_int), ("f", C.c_int)]


def make_array(cudart, width, height):
    """A width x height RGBA16F CUDA array with cudaArraySurfaceLoadStore (cudaChannelFormatKindFloat = 2, flag 0x02)."""
    h = C.c_void_p()
    cudart.cudaMallocArray.argtypes = [C.POINTER(C.c_void_p), C.POINTER(_ChannelDesc), C.c_size_t, C.c_size_t, C.c_uint]
    rc = cudart.cudaMallocArray(C.byref(h), C.byref(_ChannelDesc(16, 16, 16, 16, 2)), width, height, 0x02)
    if rc != 0:
        raise RuntimeError("cudaMallocArray failed with CUDA error %d" % rc)
    return h.value


def card():
    """Name and power limit of GPU 0, read now (nvidia-smi query only)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30).stdout.strip()
        name, limit, sm_max = [f.strip() for f in out.split(",")]
        return {"gpu": name, "power_limit_w": float(limit), "sm_max_mhz": float(sm_max)}
    except Exception as e:   # the numbers below are still device times of this card; say what could not be read
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "card_query_error": str(e)}


def spread(v):
    q = statistics.quantiles(v, n=4) if len(v) >= 2 else [v[0]] * 3
    return {"median": statistics.median(v), "p25": q[0], "p75": q[2], "min": min(v), "max": max(v), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=10, help="blocks per target kind (alternating)")
    ap.add_argument("--frames", type=int, default=20, help="timed frames per block")
    ap.add_argument("--warmup", type=int, default=5, help="untimed frames per target kind before the first block")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import torch
    import bench
    import unitygaussiansplatting_b200 as g
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    n, quality, w, h, fov, seed, _ = bench.WORKLOADS["metric"]
    asset = bench.get_asset(n, quality, seed)
    stream = torch.cuda.Stream()
    ctx = g.GaussianSplatContext(0, stream.cuda_stream)
    r = g.GaussianSplatRenderer(asset, ctx)
    cudart = C.CDLL("libcudart.so.12")   # the runtime torch loaded (same soname)
    arrays = [make_array(cudart, w, h) for _ in range(2)]
    with torch.cuda.stream(stream):
        targets = {
            "tensor": (torch.zeros((h, w, 4), dtype=torch.float16, device="cuda"), torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")),
            "array": tuple(g.CudaArrayImage(a, w, h) for a in arrays),
        }
        k = 0

        def frame(kind):
            nonlocal k
            rt, tgt = targets[kind]
            r.SortAndRenderSplats(bench.orbit_camera(k, w, h, fov), rt=rt, camera_target=tgt)
            k += 1

        for kind in targets:
            for _ in range(args.warmup):
                frame(kind)
        ctx.sync()
        ctx.set_timing(True)
        acc = {kind: {"raster_ms": [], "composite_ms": [], "total_ms": []} for kind in targets}
        for _b in range(args.blocks):
            for kind in targets:
                for _ in range(args.frames):
                    frame(kind)
                    st = ctx.stage_times()   # synchronises the context stream
                    for f in acc[kind]:
                        acc[kind][f].append(getattr(st, f))
        ctx.set_timing(False)
        ctx.sync()
    r.Dispose()
    ctx.close()
    for a in arrays:
        cudart.cudaFreeArray(C.c_void_p(a))
    res = {"what": "gs_frame stage times, render target + camera target as torch RGBA16F tensors vs RGBA16F CUDA arrays (surface objects)",
           "workload": "%d splats, %s, %dx%d, bench.orbit_camera" % (n, quality, w, h),
           "blocks": args.blocks, "frames_per_block": args.frames, **card(),
           "targets": {kind: {f: spread(v) for f, v in fields.items()} for kind, fields in acc.items()}}
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
