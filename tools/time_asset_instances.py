#!/usr/bin/env python
"""A further renderer of an uploaded asset: gs_asset_instance against gs_asset_upload.

Assets: the bench.py metric scene (6,131,954 splats, Medium) and the same scene packed VeryHigh.  Per asset:
  - wall time of gs_asset_upload and of gs_asset_instance (host clock around the call, which blocks until its device work is
    done), alternating the two, as median and interquartile range;
  - the device bytes each one adds, computed from the library's allocation rules (blob_bytes / per_renderer_bytes below), and
    the cudaMemGetInfo delta around each call, labelled indicative: other processes share the card;
  - one gs_frame_objects camera at 1920x1080 (bench.orbit_camera) drawing the source and an instance against the same call
    over two uploads: host clock from the call to the end of a full synchronise, alternating blocks.  Before timing, both arms
    draw the same frame and their render targets and draw orders are asserted bit-identical.
The card's name and power limit are read in the same run.

    python tools/time_asset_instances.py [--reps 5] [--blocks 6] [--frames 10] [--out profiles/h100_asset_instances.json]
"""
import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from time_array_target import card, spread  # noqa: E402  (tools/ is this script's directory)


def blob_bytes(d):
    """What gs_asset_upload allocates for the five blobs of GsAssetDesc d: each blob + 16 bytes of slack; a clustered SH
    palette backed to 65536 entries of 96 bytes; no chunk buffer without chunks."""
    clustered = d.sh_format > 3
    sh = max(d.sh_bytes, 65536 * 96 if clustered else 0)
    return (d.pos_bytes + 16) + (d.other_bytes + 16) + (sh + 16) + (d.color_bytes + 16) + ((d.chunk_bytes + 16) if d.chunk_bytes else 0)


def per_renderer_bytes(n):
    """What asset_init_work allocates per renderer (gs_asset_upload and gs_asset_instance alike): order, keys, key table and
    bin rectangles 4 B per splat each, draw records 48 B, view data 40 B + 16, the splat count 4 B, block bits
    (block_bits_words(n) + 16) words.  Not counted: the quad depths (4 B per splat + 16) allocated by the first frame with a
    scene depth buffer, and the group buffers of the gs_group_* calls."""
    block_bits_words = ((n + 255) // 256 + 31) // 32 + 1
    return 4 * n * 4 + 48 * n + (40 * n + 16) + 4 + (block_bits_words + 16) * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed calls per arm and asset (alternating)")
    ap.add_argument("--blocks", type=int, default=6, help="frame blocks per arm (alternating)")
    ap.add_argument("--frames", type=int, default=10, help="frames per block")
    ap.add_argument("--warmup", type=int, default=3, help="untimed frames per arm before the first block")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import numpy as np
    import torch
    import bench
    import unitygaussiansplatting_b200 as g
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    lib = N.native()
    n, quality, w, h, fov, seed, _ = bench.WORKLOADS["metric"]
    ctx = g.GaussianSplatContext(0)
    res = {"what": "gs_asset_instance (shares the blobs) vs gs_asset_upload (copies them), and one camera over source + instance vs "
                   "over two uploads", **card(),
           "fields": "upload_ms / instance_ms: host clock around the call (it blocks until its device work is done); "
                     "bytes_from_code: the library's allocation rules; mem_get_info_delta_bytes: cudaMemGetInfo before minus after, "
                     "INDICATIVE (the card is shared); frame_ms: host clock from gs_frame_objects to the end of a full synchronise",
           "assets": {}}

    def free_bytes():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    def upload(asset):
        hd, d = C.c_void_p(), asset.desc()
        t0 = time.perf_counter()
        N.check(ctx.handle, lib.gs_asset_upload(ctx.handle, C.byref(d), C.byref(hd)))
        return hd, (time.perf_counter() - t0) * 1e3

    def instance(src):
        hd = C.c_void_p()
        t0 = time.perf_counter()
        N.check(ctx.handle, lib.gs_asset_instance(src, C.byref(hd)))
        return hd, (time.perf_counter() - t0) * 1e3

    for q in ("Medium", "VeryHigh"):
        asset = bench.get_asset(n, quality, seed) if q == quality else g.synthetic_asset(g.SCENE_CLUSTERED, n, seed, q)
        d = asset.desc()
        src, _ = upload(asset)   # warms the copy path and keeps one source alive for the instances
        warm, _ = instance(src)
        lib.gs_asset_destroy(warm)
        times = {"upload_ms": [], "instance_ms": []}
        deltas = {"upload": [], "instance": []}
        for _r in range(args.reps):
            for arm in ("upload", "instance"):
                before = free_bytes()
                hd, ms = upload(asset) if arm == "upload" else instance(src)
                deltas[arm].append(before - free_bytes())
                times[arm + "_ms"].append(ms)
                lib.gs_asset_destroy(hd)
        blobs, own = blob_bytes(d), per_renderer_bytes(n)
        entry = {"splats": n, "quality": q,
                 "bytes_from_code": {"upload": blobs + own, "instance": own, "blobs": blobs, "per_renderer": own,
                                     "blobs_per_splat": blobs / n, "per_renderer_per_splat": own / n},
                 "mem_get_info_delta_bytes_indicative": {k: sorted(v) for k, v in deltas.items()},
                 **{k: spread(v) for k, v in times.items()}}
        # one camera, two objects: source + instance against two uploads, both drawn into device images
        rt = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")
        tgt = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda")
        rt_im, tgt_im = _image(rt, w, h), _image(tgt, w, h)
        host = g.GaussianSplatRenderer.from_device_asset(asset, src, ctx)
        arms = {"source_instance": [host, host.Instance()],
                "two_uploads": [g.GaussianSplatRenderer(asset, ctx), g.GaussianSplatRenderer(asset, ctx)]}
        place = [g.trs(position=(-1.2, 0.0, 0.5), scale=(0.6, 0.6, 0.6)), g.trs(position=(1.2, 0.1, 1.0), scale=(0.6, 0.6, 0.6))]
        for rs in arms.values():
            for r, m in zip(rs, place):
                r.localToWorldMatrix = m.astype(np.float32)

        def draw(rs, cam):
            fps, assets, ds = (N.GsFrameParams * 2)(), (C.c_void_p * 2)(), (C.c_int32 * 2)()
            for i, r in enumerate(rs):
                fps[i], assets[i], ds[i] = r.frame_params(cam), r._asset.value, 1
            t0 = time.perf_counter()
            N.check(ctx.handle, lib.gs_frame_objects(ctx.handle, 2, assets, fps, ds, N.GsRenderOptions(), rt_im, tgt_im))
            ctx.sync()
            return (time.perf_counter() - t0) * 1e3

        cam = bench.orbit_camera(0, w, h, fov)
        got = {}
        for arm, rs in arms.items():
            draw(rs, cam)
            got[arm] = (rt.clone(), [r.readback_order() for r in rs])
        assert got["source_instance"][0].view(torch.int16).equal(got["two_uploads"][0].view(torch.int16)), q + ": render targets differ"
        for a, b in zip(got["source_instance"][1], got["two_uploads"][1]):
            assert np.array_equal(a, b), q + ": draw orders differ"
        frame_no = 1
        for rs in arms.values():
            for _ in range(args.warmup):
                draw(rs, bench.orbit_camera(frame_no, w, h, fov))
                frame_no += 1
        acc = {arm: [] for arm in arms}
        for _b in range(args.blocks):
            for arm, rs in arms.items():
                for _ in range(args.frames):
                    acc[arm].append(draw(rs, bench.orbit_camera(frame_no, w, h, fov)))
                    frame_no += 1
        entry["frame_objects"] = {"screen": "%dx%d, bench.orbit_camera, sort every frame" % (w, h), "bit_identical": True,
                                  **{arm: {"frame_ms": spread(v)} for arm, v in acc.items()}}
        res["assets"][q] = entry
        for rs in arms.values():
            for r in rs:
                r.Dispose()   # host owns `src`
        del asset
    ctx.close()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
