#!/usr/bin/env python
"""What reading the scene depth buffer in place from a CUDA array saves over copying it into linear memory first.

The bench.py metric scene (6,131,954 splats, Medium, orbiting camera) is drawn depth-tested against a wall at the scene
centre's view depth over the left 60 % of the screen (reversed Z), in two workloads:

  1920 x 1080, one gs_frame per frame:
    tensor:        the depth in a device tensor (scene_depth_on_device = 1);
    array:         the depth in a 2-D float32 CUDA array (GS_MEM_ARRAY), read in place;
    copy_tensor:   cudaMemcpy2DFromArrayAsync from that array into a device buffer on the context stream, then the tensor path:
                   what a host that imports its depth as a CUDA array had to do before.
  a stereo pair, 1920 x 1920 per eye (64 mm apart), one gs_frame_cameras call per frame:
    layers:        eye depth in layers 0 / 1 of a layered float32 array (GS_MEM_ARRAY_LAYER);
    copy_linear:   one cudaMemcpy3DAsync per eye from its layer into a device buffer, then the same call on linear depth.

Before timing, every arm of a workload draws the same camera from a reset draw order, and the render targets must be identical.
The arms alternate in blocks of frames; each frame is timed with CUDA events on the library's stream around everything it
enqueues (copies included).  The card's name and power limit are read in the same run.

    python tools/time_depth_arrays.py [--blocks 8] [--frames 15] [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from time_array_target import card, spread  # noqa: E402
from time_layered_targets import _ChannelDesc, _Dim3, _Memcpy3DParms, _PitchedPtr, eyes  # noqa: E402

D2D = 3   # cudaMemcpyDeviceToDevice


def depth_array(cudart, w, h, layers):
    """A float32 one-channel CUDA array with cudaArraySurfaceLoadStore (and cudaArrayLayered when layers > 0)."""
    cudart.cudaMalloc3DArray.argtypes = [C.POINTER(C.c_void_p), C.POINTER(_ChannelDesc), _Dim3, C.c_uint]
    a = C.c_void_p()
    rc = cudart.cudaMalloc3DArray(C.byref(a), C.byref(_ChannelDesc(32, 0, 0, 0, 2)), _Dim3(w, h, layers), 0x02 | (0x01 if layers else 0))
    if rc != 0:
        raise RuntimeError("cudaMalloc3DArray failed with CUDA error %d" % rc)
    return a.value


def wall(cam, w, h):
    clip = cam.gpuProjectionMatrix(True).astype(np.float64) @ np.array([0.0, 0.0, -float(np.linalg.norm(cam.position)), 1.0])
    d = np.zeros((h, w), np.float32)
    d[:, :int(w * 0.6)] = np.float32(clip[2] / clip[3])
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=8, help="blocks per arm (alternating)")
    ap.add_argument("--frames", type=int, default=15, help="timed frames per block")
    ap.add_argument("--warmup", type=int, default=5, help="untimed frames per arm before the first block")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import torch
    import bench
    import unitygaussiansplatting_b200 as g
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    n, quality, W, H, fov, seed, _ = bench.WORKLOADS["metric"]
    S = 1920
    asset = bench.get_asset(n, quality, seed)
    stream = torch.cuda.Stream()
    ctx = g.GaussianSplatContext(0, stream.cuda_stream)
    r = g.GaussianSplatRenderer(asset, ctx)
    cudart = C.CDLL("libcudart.so.12")   # the runtime torch loaded (same soname)
    cudart.cudaMemcpy3DAsync.argtypes = [C.POINTER(_Memcpy3DParms), C.c_void_p]
    cudart.cudaMemcpy3D.argtypes = [C.POINTER(_Memcpy3DParms)]
    cudart.cudaMemcpy2DFromArrayAsync.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                  C.c_int, C.c_void_p]
    sp = C.c_void_p(stream.cuda_stream)

    def check(rc, what):
        if rc != 0:
            raise RuntimeError("%s failed with CUDA error %d" % (what, rc))

    def upload(arr, host, layer=0):
        host = np.ascontiguousarray(host, np.float32)
        p = _Memcpy3DParms()
        p.srcPtr, p.dstArray, p.dstPos = _PitchedPtr(host.ctypes.data, host.shape[1] * 4, host.shape[1], host.shape[0]), arr, _Dim3(0, 0, layer)
        p.extent, p.kind = _Dim3(host.shape[1], host.shape[0], 1), 1
        check(cudart.cudaMemcpy3D(C.byref(p)), "cudaMemcpy3D")

    # ---- 1920 x 1080 ----
    cam0 = bench.orbit_camera(0, W, H, fov)
    d = wall(cam0, W, H)
    a2d = depth_array(cudart, W, H, 0)
    upload(a2d, d)
    d_tensor = torch.from_numpy(d).cuda()
    d_copy = torch.empty_like(d_tensor)
    rt = torch.zeros((H, W, 4), dtype=torch.float16, device="cuda")
    arr_depth = g.CudaArrayDepth(a2d, W, H)

    def frame_1080(arm, cam):
        if arm == "tensor":
            r.sceneDepth = d_tensor
        elif arm == "array":
            r.sceneDepth = arr_depth
        else:
            check(cudart.cudaMemcpy2DFromArrayAsync(C.c_void_p(d_copy.data_ptr()), W * 4, a2d, 0, 0, W * 4, H, D2D, sp),
                  "cudaMemcpy2DFromArrayAsync")
            r.sceneDepth = d_copy
        r.SortAndRenderSplats(cam, rt=rt)

    # ---- stereo 1920 x 1920 ----
    pair0 = eyes(bench.orbit_camera(0, S, S, fov))
    sd = [wall(c, S, S) for c in pair0]
    sd[1] = np.ascontiguousarray(sd[1][:, ::-1])   # the eyes' depths differ
    a_layers = depth_array(cudart, S, S, 2)
    for e in range(2):
        upload(a_layers, sd[e], e)
    lin = [torch.empty((S, S), dtype=torch.float32, device="cuda") for _ in range(2)]
    copies = []
    for e in range(2):
        p = _Memcpy3DParms()
        p.srcArray, p.srcPos = a_layers, _Dim3(0, 0, e)
        p.dstPtr = _PitchedPtr(lin[e].data_ptr(), S * 4, S, S)
        p.extent, p.kind = _Dim3(S, S, 1), D2D
        copies.append(p)
    eye_rts = [torch.zeros((S, S, 4), dtype=torch.float16, device="cuda") for _ in range(2)]
    layer_depths = [g.CudaArrayDepth(a_layers, S, S, layer=e) for e in range(2)]
    opt = N.GsRenderOptions()
    counts = (C.c_uint32 * 2)(1, 1)
    do_sort = (C.c_int32 * 2)(1, 1)
    assets = (C.c_void_p * 2)(C.cast(r._asset, C.c_void_p).value, C.cast(r._asset, C.c_void_p).value)
    ims = [_image(t, S, S) for t in eye_rts]
    rts_p = (C.POINTER(N.GsImage) * 2)(*[C.pointer(x) for x in ims])
    none_p = (C.POINTER(N.GsImage) * 2)(C.POINTER(N.GsImage)(), C.POINTER(N.GsImage)())

    def frame_stereo(arm, pair):
        if arm == "copy_linear":
            for p in copies:
                check(cudart.cudaMemcpy3DAsync(C.byref(p), sp), "cudaMemcpy3DAsync")
        depths = layer_depths if arm == "layers" else lin
        fps = (N.GsFrameParams * 2)()
        keep = []
        for e in range(2):
            fps[e], k = g.make_frame_params(pair[e], splat_count=r.splatCount, scene_depth=depths[e])
            keep.append(k)
        N.check(ctx.handle, ctx._lib.gs_frame_cameras(ctx.handle, 2, counts, assets, fps, do_sort, C.byref(opt), rts_p, none_p))

    workloads = {
        "1080p": (["tensor", "array", "copy_tensor"], lambda arm, k: frame_1080(arm, bench.orbit_camera(k, W, H, fov)), [rt]),
        "stereo_1920": (["layers", "copy_linear"], lambda arm, k: frame_stereo(arm, eyes(bench.orbit_camera(k, S, S, fov))), eye_rts),
    }
    res = {"what": "frame device time (CUDA events on the library's stream, ms), depth-tested against a wall: the depth read in place "
                   "from a CUDA array (layer) against the same depth in linear device memory, with and without the copy out of the array "
                   "a host needed before",
           "workload": "%d splats, %s, bench.orbit_camera; %dx%d gs_frame, and a stereo pair %dx%d per eye (64 mm apart) in one "
                       "gs_frame_cameras call; wall at the scene centre's view depth over the left 60 %%" % (n, quality, W, H, S, S),
           "copy_bytes_per_frame": {"1080p": W * H * 4, "stereo_1920": 2 * S * S * 4},
           "blocks": args.blocks, "frames_per_block": args.frames, **card(), "workloads": {}}
    with torch.cuda.stream(stream):
        for name, (arms, frame, outs) in workloads.items():
            ref = None
            for arm in arms:   # the same camera from a reset draw order: identical pixels
                r.ResetOrder()
                frame(arm, 0)
                ctx.sync()
                got = [o.cpu().numpy().view(np.uint16).copy() for o in outs]
                if ref is None:
                    ref = got
                    assert any(x.any() for x in got), name
                elif not all(np.array_equal(a, b) for a, b in zip(ref, got)):
                    raise SystemExit("%s: arm %s draws other pixels than %s" % (name, arm, arms[0]))
            k = 0
            for arm in arms:
                for _ in range(args.warmup):
                    frame(arm, k)
                    k += 1
            ctx.sync()
            acc = {arm: [] for arm in arms}
            for _b in range(args.blocks):
                for arm in arms:
                    evs = []
                    for _ in range(args.frames):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(stream)
                        frame(arm, k)
                        k += 1
                        e1.record(stream)
                        evs.append((e0, e1))
                    stream.synchronize()
                    acc[arm] += [e0.elapsed_time(e1) for e0, e1 in evs]
            ctx.sync()
            res["workloads"][name] = {"pixels_identical": True, "arms": {arm: spread(v) for arm, v in acc.items()}}
    r.Dispose()
    ctx.close()
    for a in (a2d, a_layers):
        cudart.cudaFreeArray(C.c_void_p(a))
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
