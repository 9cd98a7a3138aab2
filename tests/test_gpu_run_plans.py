"""Camera and object runs at every bin-sort plan.  A run sorts its one appended bin list by the run's total bin count, and each
key is the bin id plus its camera's first bin in the run (bin base), so above 512 bins the high digit of a key is partly the
camera's offset.  Most cameras here have at most 512 bins alone: the per-camera loop sorts each in one pass while the call
sorts the whole run in two, so matching the loop bit for bit is a cross-check of two different plans.  Every comparison with
the loop covers every render target, camera target and every asset's draw order and sorted keys (`compare`).

The table RUNS states each camera set's runs, bin totals and plans; the CPU test below checks it against a restatement of
bin_sort_plan (gs_raster.cu, compiled from the source and compared) and of form_runs (gs_api.cu, with its limits read from
the source), so a change to either rule shows up there."""
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from frame_loops import Twins, call_cameras, compare, compare_frame, loop_cameras, orbit
from images import ca, launches  # noqa: F401
from util import PLAN_SCREENS, camera, pixels_per_unit, plan_scene, splat_records, world_at_pixel

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "unitygaussiansplatting_b200" / "csrc"

gpu = pytest.mark.gpu

# name: (camera sizes, runs of gs_frame_cameras with one object per camera); a run: (its cameras, bins, sort passes, digit
# bits).  The sets of a pair ("512" / "528", ...) differ in one camera's height, so their pairs and launches are the same but
# for the bin sort.
RUNS = {
    "512": ([(1024, 1024)] * 2, [((0, 1), 512, 1, 9)]),
    "528": ([(1024, 1024), (1024, 1088)], [((0, 1), 528, 2, 5)]),
    "stereo": ([(1920, 1080)] * 2, [((0, 1), 1020, 2, 5)]),
    "1024": ([(2048, 1024)] * 2, [((0, 1), 1024, 2, 5)]),
    "1056": ([(2048, 1024), (2048, 1088)], [((0, 1), 1056, 2, 6)]),
    "4096": ([(4096, 2048)] * 2, [((0, 1), 4096, 2, 6)]),
    "4160": ([(4096, 2048), (4096, 2112)], [((0, 1), 4160, 2, 7)]),
    "16384": ([(8160, 4096)] * 2, [((0, 1), 16384, 2, 7)]),
    "16512": ([(8160, 4096), (8160, 4160)], [((0, 1), 16512, 2, 8)]),
    "65536": ([(8160, 8160)] * 4, [((0, 1, 2, 3), 65536, 2, 8)]),                                  # exactly the run limit
    "65536+1": ([(8160, 8160)] * 4 + [(64, 64)], [((0, 1, 2, 3), 65536, 2, 8), ((4,), 1, 1, 5)]),   # one bin past it
    # camera 1 starts on a high-digit edge (544 = 17 x 32, 1024 = 16 x 64) and its bins straddle low-digit edges (575 | 576,
    # 1087 | 1088); camera 2 starts off an edge (769, 1296)
    "5-bit edges": ([(2048, 1088), (960, 960), (256, 256)], [((0, 1, 2), 785, 2, 5)]),
    "6-bit edges": ([(2048, 2048), (1088, 1024), (320, 200)], [((0, 1, 2), 1316, 2, 6)]),
}
EDGE_BASES = {"5-bit edges": (0, 544, 769), "6-bit edges": (0, 1024, 1296)}


def _bins(size):
    return -(-size[0] // 64) * -(-size[1] // 64)


def bin_sort_plan(bins):
    """(passes, digit bits) of the stable sort of a bin list over `bins` bins: one pass while a digit of at most 9 bits covers
    the bins, else two passes of the narrowest digit that covers them."""
    if bins <= 512:
        return 1, next(b for b in (5, 6, 7, 8, 9) if bins <= 1 << b)
    for b in (5, 6, 7, 8):
        if bins <= 1 << 2 * b:
            return 2, b
    raise ValueError("no plan sorts %d bins" % bins)


def form_runs(sizes, pairs, max_screen, max_bins, max_pairs):
    """The runs of one gs_frame_cameras call, as tuples of camera indices, for cameras of one pixel format with images of their
    own: consecutive cameras of at most max_screen px per axis share a run while the run holds at most max_pairs pairs and
    max_bins bins; a camera that joins no other is a run of its own."""
    runs, c = [], 0
    while c < len(sizes):
        e, run_pairs, run_bins = c, 0, 0
        while (e < len(sizes) and max(sizes[e]) <= max_screen and pairs[e] <= max_pairs and
               run_pairs + pairs[e] <= max_pairs and run_bins + _bins(sizes[e]) <= max_bins):
            run_pairs += pairs[e]
            run_bins += _bins(sizes[e])
            e += 1
        e = max(e, c + 1)
        runs.append(tuple(range(c, e)) if e - c >= 2 else (c,))
        c = e
    return runs


def _constant(path, name):
    m = re.search(r"\b%s = (\d+)u?\b" % name, path.read_text())
    assert m, "%s is not defined in %s" % (name, path.name)
    return int(m.group(1))


# ---- the table, without a device -------------------------------------------------------------------------------------------
def test_bin_sort_plan_restatement_matches_the_source(tmp_path):
    """gs_raster.cu's bin_sort_plan, compiled on its own, gives the plan bin_sort_plan here gives for every bin count up to the
    run limit, and every such plan's digits cover every key."""
    src = (CSRC / "gs_raster.cu").read_text()
    start = src.index("static void bin_sort_plan(")
    fn = src[start:src.index("\n}\n", start) + 3]
    prog = tmp_path / "plan.cpp"
    prog.write_text("#include <cstdint>\n#include <cstdio>\n" + fn +
                    "int main() {\n  for (uint32_t b = 1; b <= 65536; ++b) {\n    int bits, passes;\n"
                    "    bin_sort_plan(b, &bits, &passes);\n    std::printf(\"%d %d\\n\", passes, bits);\n  }\n}\n")
    exe = tmp_path / "plan"
    r = subprocess.run(["/usr/bin/g++", "-std=c++17", "-o", str(exe), str(prog)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True)
    assert r.returncode == 0, r.stdout
    got = np.array(subprocess.run([str(exe)], stdout=subprocess.PIPE, check=True, text=True).stdout.split(), np.int64).reshape(-1, 2)
    max_bins = _constant(CSRC / "gs_api.cu", "kMaxRunBins")
    want = np.array([bin_sort_plan(b) for b in range(1, 65537)])
    assert np.array_equal(got, want)
    assert max_bins <= 65536 and all(p * b >= (n - 1).bit_length() for n, (p, b) in enumerate(want[:max_bins].tolist(), 1))


def test_run_table():
    """Each camera set of RUNS splits into the stated runs, with the stated bin totals, pass counts and digit widths."""
    max_screen = _constant(CSRC / "gs_api.cu", "kMaxRunScreen")
    max_bins = _constant(CSRC / "gs_api.cu", "kMaxRunBins")
    max_pairs = _constant(CSRC / "gs_kernels.cuh", "kRunObjects")
    assert max_bins == 65536 == 4 * _bins((8160, 8160))
    for name, (sizes, runs) in RUNS.items():
        assert form_runs(sizes, [1] * len(sizes), max_screen, max_bins, max_pairs) == [r[0] for r in runs], name
        for cams, bins, passes, bits in runs:
            assert sum(_bins(sizes[c]) for c in cams) == bins, name
            assert bin_sort_plan(bins) == (passes, bits), name
    for name, bases in EDGE_BASES.items():
        sizes, [(_, _, _, bits)] = RUNS[name]
        assert tuple(np.cumsum([0] + [_bins(s) for s in sizes[:-1]]).tolist()) == bases
        assert bases[1] % (1 << bits) == 0 and bases[2] % (1 << bits) != 0, name
    # the oracle anchor: two objects per camera
    assert form_runs([(1024, 1088)] * 2, [2, 2], max_screen, max_bins, max_pairs) == [(0, 1)]
    assert bin_sort_plan(2 * _bins((1024, 1088))) == (2, 5)


# ---- on the GPU ------------------------------------------------------------------------------------------------------------
def _cameras(g, sizes):
    """One camera per size, each 0.25 units right of the one before: no two cameras of a run see the same picture."""
    return [camera(g, w, h, pos=(0.25 * c, 0.5, -6.0)) for c, (w, h) in enumerate(sizes)]


def _loop_and_call_passes(name):
    """Bin-sort passes of the loop (each camera alone) and of the call (one sort per run) of a RUNS set."""
    sizes, runs = RUNS[name]
    return sum(bin_sort_plan(_bins(s))[0] for s in sizes) + sum(r[2] for r in runs)


@gpu
@pytest.mark.parametrize("names", [("512", "528"), ("stereo",), ("1024", "1056"), ("4096", "4160"), ("16384", "16512")],
                         ids=lambda n: "-".join(n))
def test_camera_runs_at_plan_edges(g, ctx, ca, names):
    """Both sides of each plan edge equal the loop, every camera drawing its own scene with splats in its bottom-right bin;
    the launch counts differ by the bin-sort passes the table states (the 512-bin run takes one launch fewer than the 528)."""
    per_set = {}
    for name in names:
        sizes, _runs = RUNS[name]
        cams = _cameras(g, sizes)
        tw = Twins(g, ctx, [plan_scene(g, cam, 0) for cam in cams])
        try:
            n0 = launches(ctx)
            drawn = compare(g, ctx, ca, tw, [[0], [1]], cams, 0, np.float16, ["device", "host"], [None, "device"], name)
            per_set[name] = launches(ctx) - n0
            assert drawn == 2, name
        finally:
            tw.dispose()
    if len(names) == 2:
        a, b = names
        assert per_set[b] - per_set[a] == _loop_and_call_passes(b) - _loop_and_call_passes(a), per_set
    if names == ("512", "528"):
        assert per_set["528"] - per_set["512"] == 1


@gpu
def test_run_of_65536_bins_and_the_camera_past_it(g, ctx, ca):
    """Four 8160 x 8160 cameras fill one run's 65,536 bins exactly; a 64 x 64 fifth camera then goes to a run of its own.  Both
    equal the loop, and the fifth camera costs the call what it costs the loop."""
    sizes, _runs = RUNS["65536+1"]
    cams = _cameras(g, sizes)
    tw = Twins(g, ctx, [plan_scene(g, cam, 0) for cam in cams[:4]])
    try:
        n0 = launches(ctx)
        assert compare(g, ctx, ca, tw, [[0], [1], [2], [3]], cams[:4], 0, np.float16, ["device"] * 4, [None] * 4, "65536") == 4
        n1 = launches(ctx)
        assert compare(g, ctx, ca, tw, [[0], [1], [2], [3], [0]], cams, 0, np.float16, ["device"] * 5, [None] * 5, "65536+1") == 5
        n2 = launches(ctx)
        small = np.zeros((64, 64, 4), np.float16)
        loop_cameras(g, ctx, [[tw.loop[0]]], cams[4:], 0, [small], [None])
        alone = launches(ctx) - n2
        # the loop draws the fifth camera once more, and the call draws it as a run of one camera, as the loop does
        assert (n2 - n1) - (n1 - n0) == 2 * alone, (n1 - n0, n2 - n1, alone)
    finally:
        tw.dispose()


def _first_and_last_bin_scene(g, cam, seed):
    """A small clustered scene, and small splats inside the camera's first (top-left) and last (bottom-right) bins."""
    W, H = cam.pixelWidth, cam.pixelHeight
    x0, y0 = (-(-W // 64) - 1) * 64, (-(-H // 64) - 1) * 64
    depth = 6.0
    xs, ys = [20.5, 40.2, (x0 + W) / 2 - 0.3, W - 3.5], [18.3, 5.5, (y0 + H) / 2 + 0.2, H - 3.5]
    edges = splat_records(world_at_pixel(cam, xs, ys, depth), np.array([3.0, 2.0, 2.5]) / pixels_per_unit(cam, depth), 0.9,
                          (0.2, 0.9, 0.4))
    return g.create_asset(np.ascontiguousarray(np.concatenate([g.generate_input_splats(g.SCENE_CLUSTERED, 8000, seed), edges])),
                          "Medium")


@gpu
@pytest.mark.parametrize("name", ["5-bit edges", "6-bit edges"])
def test_camera_boundaries_on_digit_edges(g, O, ctx, ca, name):
    """Three cameras whose bin bases fall on and off the digit edges, each with splats in its first and last bin: the call
    equals the loop, and a fresh call equals the oracle camera by camera."""
    sizes, _runs = RUNS[name]
    cams = _cameras(g, sizes)
    assets = [_first_and_last_bin_scene(g, cam, 0x5EED1100 + c) for c, cam in enumerate(cams)]
    tw = Twins(g, ctx, assets)
    try:
        assert compare(g, ctx, ca, tw, [[0], [1], [2]], cams, 0, np.float16, ["host", "array", "device"], ["device", None, None],
                       name) == 3
    finally:
        tw.dispose()
    rs = [g.GaussianSplatRenderer(a, ctx) for a in assets]   # sorted from the identity, as the oracle sorts
    try:
        rts = [np.zeros((h, w, 4), np.float16) for w, h in sizes]
        call_cameras(g, ctx, [[r] for r in rs], cams, 0, rts, [None] * 3)
        for c, cam in enumerate(cams):
            W, H = cam.pixelWidth, cam.pixelHeight
            fp, _keep = g.make_frame_params(cam)
            want = O.frame(assets[c], fp, threads=O.max_threads())["rt"]
            assert want[:64, :64, 3].max() > 0 and want[(H - 1) // 64 * 64:, (W - 1) // 64 * 64:, 3].max() > 0, \
                "%s camera %d: nothing draws in the first or the last bin" % (name, c)
            assert np.array_equal(rts[c].astype(np.float32), want), "%s camera %d differs from the oracle" % (name, c)
    finally:
        for r in rs:
            r.Dispose()


@gpu
@pytest.mark.parametrize("name", ["stereo", "16512"], ids=["5-bit", "8-bit"])
def test_appended_lists_of_several_tiles_per_cta(g, ctx, name):
    """Two-pass camera runs whose appended list holds more than one 8192-pair tile for every CTA of the persistent bin sort
    (2 per SM), within the 4 Mi entries of a fresh context's list, which a camera run never grows: equal to the loop, and no
    overflow reported (the host render targets read the flag back)."""
    import torch
    grid_pairs = 2 * torch.cuda.get_device_properties(0).multi_processor_count * 8192
    ctx = g.GaussianSplatContext(0)   # a fresh context (not the session's): its list has the smallest capacity
    sizes, _runs = RUNS[name]
    cams = _cameras(g, sizes)
    tw = Twins(g, ctx, [plan_scene(g, cam, 11 * grid_pairs // 20) for cam in cams])
    try:
        compare(g, ctx, None, tw, [[0], [1]], cams, 0, np.float16, ["host", "host"], [None, None], name)
        entries = ctx.stage_times().tile_entries
        assert grid_pairs < entries < 4 << 20, "%d entries for a grid of %d pairs" % (entries, grid_pairs)
    finally:
        tw.dispose()
        ctx.close()


OBJECT_SCREENS = [(size, bins, blend, rt, tgt) for (size, bins, _, _), blend, rt, tgt in zip(
    [s for s in PLAN_SCREENS if s[1] in (513, 544, 1024, 1025, 4096, 4100)],
    [0, 1, 0, 1, 0, 1], ["host", "device", "array", "host", "device", "device"], [None, "host", "device", "array", None, "host"])]


@gpu
@pytest.mark.parametrize("size, bins, blend, rt_kind, tgt_kind", OBJECT_SCREENS, ids=["%d bins" % s[1] for s in OBJECT_SCREENS])
def test_object_runs_at_plan_edges(g, ctx, ca, size, bins, blend, rt_kind, tgt_kind):
    """gs_frame_objects with three objects on the two-pass screens at both edges of the 5- and 6-bit plans equals gs_frame per
    object (GS_FLAG_LOAD_RT from the second) plus gs_composite."""
    assert _bins(size) == bins
    cam = camera(g, *size)
    assets = [plan_scene(g, cam, 0), g.synthetic_asset(g.SCENE_CLUSTERED, 12000, 0x5EED1150, "VeryHigh"),
              g.synthetic_asset(g.SCENE_CLUSTERED, 6000, 0x5EED1151, "Medium")]

    def setup(i, r):
        if i:
            r.localToWorldMatrix = g.trs(position=(1.2 * i - 1.8, 0.2, 1.0 * i - 0.5), scale=(0.7, 0.7, 0.7)).astype(np.float32)

    tw = Twins(g, ctx, assets, setup)
    try:
        compare_frame(g, ctx, ca, tw, cam, blend, np.float16, rt_kind, tgt_kind, "%d bins" % bins)
    finally:
        tw.dispose()


@gpu
@pytest.mark.parametrize("variant", ["fp32 blend into rgba16f", "selection and depth", "array beside tensor", "rgba32f"])
def test_stereo_run_raster_variants(g, ctx, ca, variant):
    """The two-pass 1920 x 1080 stereo run with two objects per camera, one of them in both, through the MULTI raster's other
    instantiations: GS_BLEND_FP32 into RGBA16F (rounded at each object), selection beside a scene depth buffer per camera, a
    CUDA array beside a tensor, and RGBA32F."""
    import torch
    cams = [camera(g, 1920, 1080), camera(g, 1920, 1080, pos=(0.064, 0.5, -6.0))]
    assets = [plan_scene(g, cams[0], 0), g.synthetic_asset(g.SCENE_CLUSTERED, 12000, 0x5EED1160, "VeryHigh"),
              g.synthetic_asset(g.SCENE_CLUSTERED, 8000, 0x5EED1161, "Medium")]

    def setup(i, r):
        if i:
            r.localToWorldMatrix = g.trs(position=(1.5 * i - 2.2, 0.1 * i, 0.6 * i), scale=(0.7, 0.7, 0.7)).astype(np.float32)

    tw = Twins(g, ctx, assets, setup)
    try:
        idx = tw.gathered(g, [[0, 1], [0, 2]], cams)
        blend, dtype, rk, tk, extras = {
            "fp32 blend into rgba16f": (1, np.float16, ["device", "host"], [None, "device"], None),
            "selection and depth": (0, np.float16, ["host", "device"], ["device", None], True),
            "array beside tensor": (0, np.float16, ["array", "device"], ["device", "array"], None),
            "rgba32f": (1, np.float32, ["device", "host"], ["host", None], None),
        }[variant]
        if extras:
            rng = np.random.default_rng(5)
            sel = [rng.integers(0, 2 ** 32, (r.splatCount + 31) // 32, dtype=np.uint64).astype(np.uint32) for r in tw.loop]
            d0 = np.full((1080, 1920), 0.02, np.float32)
            d0[:, 960:] = 0.2
            d1 = torch.full((1080, 1920), 0.05, dtype=torch.float32, device="cuda")
            d1[400:600] = float("nan")
            # object 0 is depth-tested against its camera's buffer (host, then device); the others carry a selection
            extras = [[{"scene_depth": (d0, d1)[c]} if i == 0 else {"selected_bits": sel[i]} for i in idx[c]] for c in range(2)]
        assert compare(g, ctx, ca, tw, idx, cams, blend, dtype, rk, tk, variant, extras) == 2
    finally:
        tw.dispose()


@gpu
def test_two_pass_camera_run_against_the_oracle(g, O, ctx):
    """Two 1024 x 1088 cameras (544 bins: two 5-bit passes) with two objects each draw what the oracle draws from each camera's
    concatenated views in its objects' draw orders."""
    assets = [g.synthetic_asset(g.SCENE_CLUSTERED, n, 0x5EED1170 + i, "Medium") for i, n in enumerate([12000, 8000])]
    tw = Twins(g, ctx, assets)
    try:
        for i, r in enumerate(tw.loop + tw.call):
            r.localToWorldMatrix = g.trs(position=(1.3 * (i % 2) - 0.6, 0.0, 1.0 * (i % 2)), scale=(0.7, 0.7, 0.7)).astype(np.float32)
        cams = [orbit(g, 1, 1024, 1088), orbit(g, 1, 1024, 1088, phase=0.8)]
        idx = tw.gathered(g, [[0, 1], [0, 1]], cams)
        # camera 0's orders: what the loop's first camera leaves
        lo, hi = tw.pick(idx)
        rts = [np.zeros((1088, 1024, 4), np.float16) for _ in cams]
        loop_cameras(g, ctx, lo[:1], cams[:1], 0, rts[:1], [None])
        order0 = {i: tw.loop[i].readback_order() for i in idx[0]}
        call_cameras(g, ctx, hi, cams, 0, rts, [None, None])
        for c, cam in enumerate(cams):
            views, orders, base = [], [], 0
            for i in idx[c]:
                r = tw.call[i]
                fp, _keep = g.make_frame_params(cam, r.localToWorldMatrix)
                views.append(O.frame(r.m_Asset, fp, threads=O.max_threads())["view"])
                orders.append((order0[i] if c == 0 else r.readback_order()) + np.uint32(base))
                base += r.splatCount
            want = O.render(np.concatenate(views), np.concatenate(orders), cam.pixelWidth, cam.pixelHeight, 0, O.max_threads())
            assert rts[c].any() and np.array_equal(rts[c].astype(np.float32), want), "camera %d" % c
    finally:
        tw.dispose()
