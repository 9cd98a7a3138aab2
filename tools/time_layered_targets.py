#!/usr/bin/env python
"""A stereo pair drawn into the two layers of one layered CUDA array (an XR eye-texture array) three ways.

The bench.py metric scene (6,131,954 splats, Medium, orbiting camera) is rendered as a stereo pair, 1920 x 1920 per eye, eyes
64 mm apart, into the two layers of one layered RGBA16F array created with cudaArrayLayered | cudaArraySurfaceLoadStore:

  layers_one_call:   gs_frame_cameras with the two eyes' render targets as layers 0 and 1 (GS_MEM_ARRAY_LAYER): one camera run;
  arrays_then_copy:  gs_frame_cameras into two 2-D arrays (GS_MEM_ARRAY), then one cudaMemcpy3DAsync per eye into its layer,
                     what a host had to do before layers were images (the copy is 2 x 1920^2 x 8 B per frame);
  layers_per_eye:    one gs_frame per eye into its layer: the camera loop, two runs.

The three alternate in blocks of frames.  Each frame is timed with CUDA events on the library's stream around everything the
frame enqueues (copies included).  The card's name and power limit are read in the same run.

    python tools/time_layered_targets.py [--blocks 8] [--frames 15] [--out FILE.json]
"""
import argparse
import ctypes as C
import dataclasses
import json
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from time_array_target import card, spread  # noqa: E402


class _ChannelDesc(C.Structure):
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("z", C.c_int), ("w", C.c_int), ("f", C.c_int)]


class _Dim3(C.Structure):
    _fields_ = [("x", C.c_size_t), ("y", C.c_size_t), ("z", C.c_size_t)]   # cudaExtent and cudaPos


class _PitchedPtr(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("pitch", C.c_size_t), ("xsize", C.c_size_t), ("ysize", C.c_size_t)]


class _Memcpy3DParms(C.Structure):
    _fields_ = [("srcArray", C.c_void_p), ("srcPos", _Dim3), ("srcPtr", _PitchedPtr),
                ("dstArray", C.c_void_p), ("dstPos", _Dim3), ("dstPtr", _PitchedPtr), ("extent", _Dim3), ("kind", C.c_int)]


def make_array(cudart, width, height, layers):
    """An RGBA16F CUDA array with cudaArraySurfaceLoadStore; layers > 0: a layered one (cudaArrayLayered) of that many layers."""
    cudart.cudaMalloc3DArray.argtypes = [C.POINTER(C.c_void_p), C.POINTER(_ChannelDesc), _Dim3, C.c_uint]
    h = C.c_void_p()
    rc = cudart.cudaMalloc3DArray(C.byref(h), C.byref(_ChannelDesc(16, 16, 16, 16, 2)), _Dim3(width, height, layers),
                                  0x02 | (0x01 if layers else 0))
    if rc != 0:
        raise RuntimeError("cudaMalloc3DArray failed with CUDA error %d" % rc)
    return h.value


def eyes(cam, ipd=0.064):
    right = cam.rotation[:, 0]
    return [dataclasses.replace(cam, position=cam.position + s * 0.5 * ipd * right) for s in (-1.0, 1.0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=8, help="blocks per mode (alternating)")
    ap.add_argument("--frames", type=int, default=15, help="timed stereo frames per block")
    ap.add_argument("--warmup", type=int, default=5, help="untimed frames per mode before the first block")
    ap.add_argument("--size", type=int, default=1920, help="width and height of each eye")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import torch
    import bench
    import unitygaussiansplatting_b200 as g
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    n, quality, _w, _h, fov, seed, _ = bench.WORKLOADS["metric"]
    w = h = args.size
    asset = bench.get_asset(n, quality, seed)
    stream = torch.cuda.Stream()
    ctx = g.GaussianSplatContext(0, stream.cuda_stream)
    r = g.GaussianSplatRenderer(asset, ctx)
    cudart = C.CDLL("libcudart.so.12")   # the runtime torch loaded (same soname)
    cudart.cudaMemcpy3DAsync.argtypes = [C.POINTER(_Memcpy3DParms), C.c_void_p]
    eye_tex = make_array(cudart, w, h, 2)
    flat = [make_array(cudart, w, h, 0) for _ in range(2)]
    layers = [g.CudaArrayImage(eye_tex, w, h, layer=e) for e in range(2)]
    flats = [g.CudaArrayImage(a, w, h) for a in flat]
    copies = []
    for e in range(2):
        p = _Memcpy3DParms()
        p.srcArray, p.dstArray, p.dstPos = flat[e], eye_tex, _Dim3(0, 0, e)
        p.extent, p.kind = _Dim3(w, h, 1), 3   # cudaMemcpyDeviceToDevice
        copies.append(p)
    k = 0

    def frame(mode):
        nonlocal k
        pair = eyes(bench.orbit_camera(k, w, h, fov))
        k += 1
        if mode == "layers_one_call":
            g.SortAndRenderCameras([r], pair, layers)
        elif mode == "arrays_then_copy":
            g.SortAndRenderCameras([r], pair, flats)
            for p in copies:
                rc = cudart.cudaMemcpy3DAsync(C.byref(p), C.c_void_p(stream.cuda_stream))
                if rc != 0:
                    raise RuntimeError("cudaMemcpy3DAsync failed with CUDA error %d" % rc)
        else:
            for cam, im in zip(pair, layers):
                r.SortAndRenderSplats(cam, rt=im)

    modes = ["layers_one_call", "arrays_then_copy", "layers_per_eye"]
    with torch.cuda.stream(stream):
        for mode in modes:
            for _ in range(args.warmup):
                frame(mode)
        ctx.sync()
        acc = {mode: [] for mode in modes}
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
    for a in [eye_tex, *flat]:
        cudart.cudaFreeArray(C.c_void_p(a))
    res = {"what": "stereo frame device time (CUDA events on the library's stream, ms): the two eyes into the layers of one layered "
                   "RGBA16F array in one gs_frame_cameras call, into two 2-D arrays then cudaMemcpy3DAsync into the layers, or one "
                   "gs_frame per eye into its layer",
           "workload": "%d splats, %s, stereo pair %dx%d per eye (64 mm apart), bench.orbit_camera" % (n, quality, w, h),
           "copy_bytes_per_frame": 2 * w * h * 8,
           "blocks": args.blocks, "frames_per_block": args.frames, **card(),
           "modes": {mode: spread(v) for mode, v in acc.items()}}
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
