#!/usr/bin/env python
"""Compositing onto R8G8B8A8_SRGB camera targets (four bytes per pixel, RGB sRGB-encoded: the colour buffer of LDR cameras)
against RGBA16F and B10G11R11_UFLOAT ones, in device memory and in a 2-D CUDA array made with cudaArraySurfaceLoadStore.

The bench.py metric scene (6,131,954 splats, Medium, orbiting camera), at 1920 x 1080 and 3840 x 2160:

  composite_<target>_<memory>:  gs_composite alone, of one RGBA16F render target in device memory (a frame of the scene drawn
                                once) onto an rgba16f, packed (B10G11R11) or srgb8 camera target; --calls calls between two CUDA events,
                                the time per call;
  frame_<target>_<memory>:      gs_frame with a camera target and no rt (the render target lives in library scratch), per frame.

With --baseline-lib, a libgsplat_b200.so built from another commit, the rgba16f composite is also timed through
that library (modes baseline_composite_*), on the same render target and the same targets, so that the two builds' composite
can be compared in one run.  Every mode of one size alternates with the others in blocks.  Device times come from CUDA events
on the library's stream; the card's name and power limit are read in the same run.

    python tools/time_srgb8_targets.py [--baseline-lib PATH] [--blocks 8] [--frames 15] [--calls 50] [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from time_array_target import card, spread  # noqa: E402

SIZES = [(1920, 1080), (3840, 2160)]
KIND_UNSIGNED, KIND_FLOAT = 1, 2


class _ChannelDesc(C.Structure):
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("z", C.c_int), ("w", C.c_int), ("f", C.c_int)]


def make_array(cudart, width, height, target):
    """A 2-D CUDA array with cudaArraySurfaceLoadStore for a camera target: RGBA16F, one 32-bit unsigned channel (B10G11R11) or
    four 8-bit unsigned channels (sRGB8)."""
    desc = {"rgba16f": (16, 16, 16, 16, KIND_FLOAT), "packed": (32, 0, 0, 0, KIND_UNSIGNED), "srgb8": (8, 8, 8, 8, KIND_UNSIGNED)}[target]
    cudart.cudaMallocArray.argtypes = [C.POINTER(C.c_void_p), C.POINTER(_ChannelDesc), C.c_size_t, C.c_size_t, C.c_uint]
    h = C.c_void_p()
    rc = cudart.cudaMallocArray(C.byref(h), C.byref(_ChannelDesc(*desc)), width, height, 0x02)
    if rc != 0:
        raise RuntimeError("cudaMallocArray failed with CUDA error %d" % rc)
    return h.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", default=None, help="a libgsplat_b200.so of another commit: also time its composite")
    ap.add_argument("--blocks", type=int, default=8, help="blocks per mode (alternating)")
    ap.add_argument("--frames", type=int, default=15, help="timed samples per block")
    ap.add_argument("--calls", type=int, default=50, help="gs_composite calls per composite sample")
    ap.add_argument("--warmup", type=int, default=5, help="untimed samples per mode before the first block")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import numpy as np
    import torch
    import bench
    import unitygaussiansplatting_b200 as g
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    n, quality, _w, _h, fov, seed, _ = bench.WORKLOADS["metric"]
    asset = bench.get_asset(n, quality, seed)
    stream = torch.cuda.Stream()
    ctx = g.GaussianSplatContext(0, stream.cuda_stream)
    r = g.GaussianSplatRenderer(asset, ctx)
    cudart = C.CDLL("libcudart.so.12")   # the runtime torch loaded (same soname)
    libs = {"": (N.native(), ctx.handle)}
    if args.baseline_lib:
        base = N._bind(C.CDLL(str(Path(args.baseline_lib).resolve())), N.NATIVE_SYMBOLS)
        h = C.c_void_p()
        N.check(None, base.gs_create(0, C.c_void_p(stream.cuda_stream), C.byref(h)))
        libs["baseline_"] = (base, h)
    arrays = []
    results = {}
    k = 0
    for w, h in SIZES:
        with torch.cuda.stream(stream):
            rt = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")
            r.SortAndRenderSplats(bench.orbit_camera(0, w, h, fov), rt=rt)
            ctx.sync()
            covered = float((rt[..., 3] > 0).float().mean())
            rt_im = _image(rt, w, h)
            rng = np.random.default_rng(1)
            bg = rng.random((h, w, 3), np.float32)
            targets, images = {}, {}
            for t in ("rgba16f", "packed", "srgb8"):
                if t == "packed":
                    host = g.pack_b10g11r11(bg)
                    targets[t, "device"] = torch.from_numpy(host.view(np.int32)).cuda()
                elif t == "srgb8":
                    host = g.encode_srgb8(np.concatenate([bg, np.ones((h, w, 1), np.float32)], -1))
                    targets[t, "device"] = torch.from_numpy(host).cuda()
                else:
                    host = np.concatenate([bg, np.ones((h, w, 1), np.float32)], -1).astype(np.float16)
                    targets[t, "device"] = torch.from_numpy(host).cuda()
                arr = make_array(cudart, w, h, t)
                arrays.append(arr)
                targets[t, "array"] = g.CudaArrayImage(arr, w, h, {"rgba16f": np.float16, "packed": np.uint32, "srgb8": np.uint8}[t])
            for key, tg in targets.items():
                images[key] = _image(tg, w, h)
            modes = {}
            for prefix, (lib, handle) in libs.items():
                for (t, mem), im in images.items():
                    if prefix and t != "rgba16f":
                        continue
                    modes["%scomposite_%s_%s" % (prefix, t, mem)] = ("composite", lib, handle, im)
            for t in ("rgba16f", "srgb8"):
                for mem in ("device", "array"):
                    modes["frame_%s_%s" % (t, mem)] = ("frame", None, None, targets[t, mem])

            def sample(mode):
                nonlocal k
                what, lib, handle, im = modes[mode]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                if what == "composite":
                    for _ in range(args.calls):
                        rc = lib.gs_composite(handle, C.byref(rt_im), C.byref(im))
                        if rc:
                            raise N.GsError(rc, str(lib.gs_last_error(handle)))
                else:
                    r.SortAndRenderSplats(bench.orbit_camera(k, w, h, fov), camera_target=im)
                    k += 1
                e1.record(stream)
                return e0, e1, args.calls if what == "composite" else 1

            for mode in modes:
                for _ in range(args.warmup):
                    sample(mode)
            ctx.sync()
            acc = {mode: [] for mode in modes}
            for _b in range(args.blocks):
                for mode in modes:
                    evs = [sample(mode) for _ in range(args.frames)]
                    stream.synchronize()
                    acc[mode] += [e0.elapsed_time(e1) / calls for e0, e1, calls in evs]
            ctx.sync()
            results["%dx%d" % (w, h)] = {"rt_covered_fraction": covered, "modes": {m: spread(v) for m, v in acc.items()}}
    for prefix, (lib, handle) in libs.items():
        if prefix:
            lib.gs_sync(handle)
            lib.gs_destroy(handle)
    r.Dispose()
    ctx.close()
    for a in arrays:
        cudart.cudaFreeArray(C.c_void_p(a))
    res = {"what": "device time in ms (CUDA events on the library's stream): composite_* is one gs_composite of a frame's RGBA16F "
                   "render target (device memory) onto a camera target; frame_* is one gs_frame with that camera target and no rt. "
                   "Targets: rgba16f / packed (B10G11R11_UFLOAT) / srgb8 (R8G8B8A8_SRGB), in device memory or a 2-D CUDA array. "
                   "baseline_* modes: the same composite through the library given as --baseline-lib",
           "workload": "%d splats, %s, bench.orbit_camera" % (n, quality), "baseline_lib": args.baseline_lib,
           "blocks": args.blocks, "samples_per_block": args.frames, "composite_calls_per_sample": args.calls, **card(),
           "sizes": results}
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
