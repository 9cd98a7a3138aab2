"""The two things the raster reads from textures the host owns, against the oracle bit for bit on the raw words:

1. the scene depth buffer of the pass's ZTest LEqual (reversed Z: a fragment draws when its quad depth >= the stored depth), at
   exact ties -- every stored value is a splat's own quad depth clip.z / clip.w or one ulp either side of it, in patterns that
   vary along both axes, with specials (+-0, NaN payloads, +-inf, a subnormal, 1, 2) scattered over them -- through every
   path that depth-tests and every memory kind a depth buffer can be in;
2. the render target's content under GS_FLAG_LOAD_RT, when that content is not the kernel's own output: alpha at, just
   under and above 1 in whole 16x16 tiles, whole 8x4 warp blocks and single pixels, alpha far above 1 and below 0, NaN and
   inf channels, -0, half subnormals, floats that are not halves, and NaN payloads (a signalling one too) where no splat
   reaches.  A pixel nothing blends into keeps its loaded words.

Screens are small so that the oracle draws quickly."""
import ctypes as C

import numpy as np
import pytest

from frame_loops import call_cameras, frame_args
from images import Image, bits, ca, to_device, to_host  # noqa: F401
from util import camera, splat_records, view_fields, world_at_pixel

W, H = 320, 240
RECT = (W + 61, H + 37, 37, 19)   # array width, height, and the rectangle's origin: non-zero in both axes
CANON16 = 0x7FFF                  # the half NaN a GPU conversion or blend produces


def _u32f(words):
    return np.asarray(words, np.uint32).view(np.float32)


def _hash(x, y, salt=0):
    """A per-pixel choice that varies along both axes."""
    h = (np.asarray(x, np.int64) * 73856093) ^ (np.asarray(y, np.int64) * 19349663) ^ (salt * 83492791)
    h = (h ^ (h >> 13)) * 0x5BD1E995
    return (h ^ (h >> 15)) & 0x7FFFFFFF


def _oracle_threads(O):
    return O.max_threads()


def quad_depths(O, asset, fp):
    """Per splat: the quad depth clip.z / clip.w in float32 (the oracle's and the kernel's), the pixel of its centre, and
    whether it is in front of the camera."""
    v = view_fields(O.calc_view(asset, fp))
    pos = v["pos"]
    with np.errstate(invalid="ignore", divide="ignore"):
        z = pos[:, 2] / pos[:, 3]
        cx = (pos[:, 0] / pos[:, 3] * np.float32(0.5) + np.float32(0.5)) * np.float32(fp.screen_w)
        cy = (pos[:, 1] / pos[:, 3] * np.float32(-0.5) + np.float32(0.5)) * np.float32(fp.screen_h)
    return z.astype(np.float32), cx, cy, pos[:, 3] > 0


def tie_classes(z, cls):
    """z itself (class 0), one ulp above (1: hides the splat) or one ulp below (2: draws it)."""
    z = np.asarray(z, np.float32)
    return np.where(cls == 0, z, np.where(cls == 1, np.nextafter(z, np.float32(np.inf)), np.nextafter(z, np.float32(-np.inf))))


# ---- scenes -------------------------------------------------------------------------------------------------------------
def separated_scene(g, cam):
    """An 8 x 6 grid of VeryHigh splats (float32 positions), 40 pixels apart, each at its own depth: no two footprints meet."""
    xs, ys = np.meshgrid(20.0 + 40.0 * np.arange(8), 20.0 + 40.0 * np.arange(6))
    n = xs.size
    depth = 4.0 + 0.05 * np.arange(n)
    pos = world_at_pixel(cam, xs.ravel() + 0.3, ys.ravel() + 0.2, depth)
    rng = np.random.default_rng(7)
    rec = splat_records(pos, 0.05, rng.uniform(0.7, 1.0, n), dc=rng.uniform(0.1, 0.9, (n, 3)))
    return g.create_asset(rec, "VeryHigh")


def dense_scene(g):
    return g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0F01, "VeryHigh")


def loaded_scene(g, cam):
    """3000 overlapping VeryHigh splats over the left 70 % of the screen; the rest of the screen no splat reaches."""
    rng = np.random.default_rng(0x10AD)
    n = 3000
    pos = world_at_pixel(cam, rng.uniform(8, 0.7 * W - 24, n), rng.uniform(-4, H + 4, n), rng.uniform(3.0, 8.0, n))
    rec = splat_records(pos, rng.uniform(0.015, 0.06, (n, 3)), rng.uniform(0.2, 1.0, n), dc=rng.uniform(0.0, 1.0, (n, 3)),
                        quat=rng.standard_normal((n, 4)))
    return g.create_asset(rec, "VeryHigh")


def voronoi_field(O, g, asset, cam, salt):
    """Every pixel takes the quad depth of the splat whose centre is nearest, or one ulp above or below it by a hash of (x, y)."""
    fp, _keep = g.make_frame_params(cam)
    z, cx, cy, front = quad_depths(O, asset, fp)
    assert front.all()
    yy, xx = np.mgrid[0:H, 0:W]
    d2 = (xx[..., None] + 0.5 - cx) ** 2 + (yy[..., None] + 0.5 - cy) ** 2
    near = np.argmin(d2, axis=-1)
    cls = _hash(xx, yy, salt) % 3
    return tie_classes(z[near], cls), cls


def stamped_field(O, g, asset, cam):
    """Each drawable splat stamps its quad depth (or a neighbour by one ulp) on the 3 x 3 pixels round its centre, in draw order."""
    fp, _keep = g.make_frame_params(cam)
    z, cx, cy, front = quad_depths(O, asset, fp)
    order = O.frame(asset, fp, threads=_oracle_threads(O))["order"]
    field = np.zeros((H, W), np.float32)
    for i in order:
        if not front[i] or not (0 <= cx[i] < W and 0 <= cy[i] < H):
            continue
        x0, y0 = int(cx[i]), int(cy[i])
        ys, xs = np.mgrid[max(y0 - 1, 0):min(y0 + 2, H), max(x0 - 1, 0):min(x0 + 2, W)]
        field[ys, xs] = tie_classes(z[i], _hash(xs, ys, 3) % 3)
    return field, z[front & (cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)]


def row_field(zs):
    """A field that varies only along y, each row one of the scene's quad depths."""
    zs = np.sort(np.asarray(zs, np.float32))
    return np.repeat(zs[(np.arange(H) * 97) % zs.size][:, None], W, axis=1).astype(np.float32)


def with_specials(field, seed):
    f = field.copy()
    rng = np.random.default_rng(seed)
    specials = _u32f([0x00000000, 0x80000000, 0x7FC00000, 0x7FA00001, 0xFFC12345, 0x7F800000, 0xFF800000, 0x00000001,
                      0x3F800000, 0x40000000])
    at = rng.random((H, W)) < 0.03
    f[at] = specials[rng.integers(0, specials.size, int(at.sum()))]
    return f


# ---- depth buffers in every memory kind -----------------------------------------------------------------------------------
def depth_kinds(g, ca, field):
    """The field as a depth buffer of every memory kind; the other texels of a layered or larger array hold 1.0."""
    return {kind: Image(g, ca, kind, field, "depth", start=1.0, layers=3, layer=1, rect=RECT).image
            for kind in ("host", "device", "array", "layer", "rect")}


def oracle_draw(O, g, asset, cam, field, staged, sel=None, blend=0, init=None):
    fp, _keep = g.make_frame_params(cam, splat_count=asset.splatCount, selected_bits=sel, scene_depth=field)
    if staged:   # gs_calc_view + gs_render after ResetOrder: the identity order
        order = np.arange(asset.splatCount, dtype=np.uint32)
        return O.render(O.calc_view(asset, fp, _oracle_threads(O)), order, W, H, blend, _oracle_threads(O), sel, field, init)
    return O.frame(asset, fp, blend_mode=blend, threads=_oracle_threads(O), init=init)["rt"]


def gpu_draw(r, cam, rt, staged):
    r.ResetOrder()
    if staged:
        r.CalcViewData(cam)
        r.DrawSplats(cam, rt)
    else:
        r.SortAndRenderSplats(cam, rt=rt)


def _halfbits(rt):
    """The oracle's float image narrowed to RGBA16F words (its fp16-ROP values are halves already); NaN is the canonical half."""
    with np.errstate(over="ignore", invalid="ignore"):
        w = rt.astype(np.float16).view(np.uint16)
    return np.where(np.isnan(rt), np.uint16(CANON16), w)


# ---- 1. scene depth at ties --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_scene_depth_ties_every_path_and_memory_kind(g, O, ctx, ca):
    cam = camera(g, W, H)
    sep, dense = separated_scene(g, cam), dense_scene(g)
    vor, cls = voronoi_field(O, g, sep, cam, 1)

    # precondition: the tie classes of the separated scene do what they say, and each has drawn pixels
    free = oracle_draw(O, g, sep, cam, None, False)
    tested = oracle_draw(O, g, sep, cam, vor, False)
    drawn = free[..., 3] > 0
    for c in range(3):
        assert (drawn & (cls == c)).sum() > 100, "tie class %d has too few drawn pixels" % c
    assert not tested[drawn & (cls == 1)].any(), "one ulp above the quad depth must hide it"
    assert np.array_equal(tested[cls != 1], free[cls != 1]), "the quad depth itself and one ulp below must draw"

    stamped, zs = stamped_field(O, g, dense, cam)
    fields = {
        "separated, ties": (sep, vor),
        "dense, stamped ties + specials": (dense, with_specials(stamped, 5)),
        "dense, rows only": (dense, row_field(zs)),
    }
    for fname, (asset, field) in fields.items():
        n = asset.splatCount
        sel = np.zeros((n + 31) // 32, np.uint32)
        sel[::3] = 0x11111111
        r = g.GaussianSplatRenderer(asset, ctx)
        kinds = depth_kinds(g, ca, field)
        for staged in (False, True):
            for selected in (None, sel):
                want = _halfbits(oracle_draw(O, g, asset, cam, field, staged, selected))
                assert not np.array_equal(want, _halfbits(oracle_draw(O, g, asset, cam, None, staged, selected))), fname
                r.m_SelectedBits = selected
                for kname, d in kinds.items():
                    r.sceneDepth = d
                    t = to_device(np.zeros((H, W, 4), np.float16))
                    gpu_draw(r, cam, t, staged)
                    got = bits(to_host(ctx, t))
                    bad = np.argwhere((got != want).any(-1))
                    assert bad.size == 0, "%s, %s depth, %s, selection %s: %d pixels differ, first at (y, x) = %s" % (
                        fname, kname, "gs_calc_view + gs_render" if staged else "gs_frame", selected is not None, len(bad), bad[:3].tolist())
        r.Dispose()


@pytest.mark.gpu
def test_scene_depth_ties_per_camera_and_per_object(g, O, ctx, ca):
    """gs_frame_cameras with a different tie pattern per camera (linear and layered depth), gs_frame_objects with one
    depth-tested object beside one that is not, and an emulated group on a host depth buffer."""
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.multigpu import GaussianSplatGroup
    from unitygaussiansplatting_b200.renderer import _image
    cams = [camera(g, W, H), camera(g, W, H, pos=(0.15, 0.45, -6.2), forward=(0.02, 0.0, 1.0))]
    sep = separated_scene(g, cams[0])
    fields = [voronoi_field(O, g, sep, cams[c], 11 + c)[0] for c in range(2)]
    r = g.GaussianSplatRenderer(sep, ctx)
    want = [_halfbits(oracle_draw(O, g, sep, cams[c], fields[c], False)) for c in range(2)]
    assert not np.array_equal(want[0], want[1])
    stack = ca.array(W, H, 2, np.float32, 1, fill=np.stack(fields))
    for dname, ds in (("device", [to_device(f) for f in fields]), ("layer", [g.CudaArrayDepth(stack, W, H, layer=c) for c in range(2)])):
        r.ResetOrder()
        rts = [to_device(np.zeros((H, W, 4), np.float16)) for _ in range(2)]
        assert call_cameras(g, ctx, [[r], [r]], cams, 0, rts, [None, None], [[{"scene_depth": d}] for d in ds], check=False) == 0
        for c in range(2):
            assert np.array_equal(bits(to_host(ctx, rts[c])), want[c]), "gs_frame_cameras, %s depth, camera %d" % (dname, c)

    # two objects, one depth-tested: drawing them one after the other onto one target
    cam = cams[0]
    dense = dense_scene(g)
    rd = g.GaussianSplatRenderer(dense, ctx)
    stamped, _ = stamped_field(O, g, dense, cam)
    dfield = with_specials(stamped, 9)
    for objs in ([(r, sep, fields[0]), (rd, dense, None)], [(rd, dense, dfield), (r, sep, None)]):
        first = oracle_draw(O, g, objs[0][1], cam, objs[0][2], False)
        expect = _halfbits(oracle_draw(O, g, objs[1][1], cam, objs[1][2], False, init=first))
        assets, fps, do_sort, keep = frame_args(g, [(cam, x, None if f is None else to_device(f)) for x, _, f in objs])
        for x, _, _ in objs:
            x.ResetOrder()
        t = to_device(np.zeros((H, W, 4), np.float16))
        im = _image(t, W, H)
        opt = N.GsRenderOptions()
        assert ctx._lib.gs_frame_objects(ctx.handle, 2, assets, fps, do_sort, C.byref(opt), C.byref(im), None) == 0
        assert np.array_equal(bits(to_host(ctx, t)), expect), "gs_frame_objects, depth on object %d" % (0 if objs[0][2] is not None else 1)

    # an emulated group of two on a host depth buffer: every member receives the whole frame
    grp = GaussianSplatGroup.create(dense, [0, 0], emulate=True)
    try:
        grp.sceneDepth = dfield
        rts = [np.zeros((H, W, 4), np.float16) for _ in range(2)]
        grp.SortAndRenderSplats(cam, rts=rts)
        grp.sync()
        want_g = _halfbits(oracle_draw(O, g, dense, cam, dfield, False))
        for i, x in enumerate(rts):
            assert np.array_equal(bits(x), want_g), "group member %d" % i
    finally:
        grp.close()
    r.Dispose()
    rd.Dispose()


# ---- 2. loaded targets --------------------------------------------------------------------------------------------------
NAN16 = np.array([0x7C01, 0xFC01, 0x7E00, 0x7D55, 0xFE12, 0x7FFE], np.uint16)                  # 0x7C01: signalling
NAN32 = np.array([0x7F800001, 0xFF800001, 0x7FC00000, 0x7FA5A5A5, 0xFFC12345, 0x7FFFFFFE], np.uint32)


def loaded_content(O, g, asset, cam, dtype):
    """(words, widened float32 image, family -> pixel mask): a target's content built around what the scene reaches."""
    fp, _keep = g.make_frame_params(cam)
    reach = O.render(O.calc_view(asset, fp, _oracle_threads(O)), np.arange(asset.splatCount, dtype=np.uint32), W, H, 1,
                     _oracle_threads(O))[..., 3] > 0
    assert reach.any() and not reach.all()
    rng = np.random.default_rng(0x5EED0F02 + np.dtype(dtype).itemsize)
    img = rng.random((H, W, 4), np.float32)
    img[..., 3] *= 0.6
    if dtype == np.float16:
        img = img.astype(np.float16).astype(np.float32)
    else:
        assert (img.astype(np.float16).astype(np.float32) != img).mean() > 0.9   # floats that are not halves
    fam = {}
    free = reach.copy()   # reached pixels no family has taken yet

    def take(name, mask):
        mask = mask & free
        free[mask] = False
        fam[name] = mask

    ty, tx = np.mgrid[0:H // 16, 0:W // 16]
    full = reach[:H // 16 * 16, :W // 16 * 16].reshape(H // 16, 16, W // 16, 16).all(axis=(1, 3))
    tiles = np.argwhere(full)[::3][:4]
    m = np.zeros((H, W), bool)
    for y, x in tiles:
        m[16 * y:16 * y + 16, 16 * x:16 * x + 16] = True
    take("alpha 1, 16x16 tiles", m)

    blocks = reach[:H // 4 * 4, :W // 8 * 8].reshape(H // 4, 4, W // 8, 8).all(axis=(1, 3))
    bl = [b for b in np.argwhere(blocks) if free[4 * b[0]:4 * b[0] + 4, 8 * b[1]:8 * b[1] + 8].all()]
    rng.shuffle(bl)
    for name, k0, k1 in (("alpha 1, 8x4 blocks", 0, 6), ("alpha 1.5, 8x4 blocks", 6, 10), ("alpha 1 + 2^-10, 8x4 blocks", 10, 13)):
        m = np.zeros((H, W), bool)
        for y, x in bl[k0:k1]:
            m[4 * y:4 * y + 4, 8 * x:8 * x + 8] = True
        take(name, m)

    singles = ["alpha 1", "alpha 1 - 2^-11", "alpha 1 + 2^-10", "alpha 1.5", "alpha 65504", "alpha -0.375", "alpha NaN",
               "inf colour", "NaN colour", "-0", "half subnormals"]
    idx = np.argwhere(free)
    rng.shuffle(idx)
    for k, name in enumerate(singles):
        m = np.zeros((H, W), bool)
        y, x = idx[k::len(singles)][:25].T
        m[y, x] = True
        take(name, m)
    m = np.zeros((H, W), bool)
    y, x = np.argwhere(~reach)[::997][:60].T
    m[y, x] = True
    fam["NaN payloads where no splat reaches"] = m

    alpha = {"alpha 1, 16x16 tiles": 1.0, "alpha 1, 8x4 blocks": 1.0, "alpha 1.5, 8x4 blocks": 1.5, "alpha 1 + 2^-10, 8x4 blocks": 1 + 2.0 ** -10,
             "alpha 1": 1.0, "alpha 1 - 2^-11": 1 - 2.0 ** -11, "alpha 1 + 2^-10": 1 + 2.0 ** -10, "alpha 1.5": 1.5,
             "alpha 65504": 65504.0, "alpha -0.375": -0.375}
    for name, a in alpha.items():
        img[fam[name], 3] = a
    img[fam["inf colour"], 0], img[fam["inf colour"], 1] = np.inf, -np.inf
    img[fam["-0"]] = -0.0
    img[fam["half subnormals"], :3] = np.float32([2.0 ** -24, 3 * 2.0 ** -24, 1023 * 2.0 ** -24])
    img[fam["half subnormals"], 3] = 2.0 ** -20
    if dtype == np.float16:
        words = img.astype(np.float16).view(np.uint16)
        nans = NAN16
    else:
        words = img.view(np.uint32).copy()
        nans = NAN32
    words[fam["alpha NaN"], 3] = nans[2]
    words[fam["NaN colour"], 1] = nans[4]
    y, x = np.nonzero(fam["NaN payloads where no splat reaches"])
    words[y, x] = nans[(np.arange(y.size)[:, None] + np.arange(4)) % nans.size]
    if dtype == np.float16:   # widened exactly, NaN payloads included
        wide = words.view(np.float16).astype(np.float32)
        assert np.array_equal(_halfbits(wide)[~np.isnan(wide)], words[~np.isnan(wide)])
    else:
        wide = words.view(np.float32)
    return words, np.ascontiguousarray(wide), fam


def expectedbits(rt, init, words, dtype):
    """The oracle's draw onto `init` as `dtype` words: what it left bit for bit unchanged is the loaded word, the rest narrowed."""
    if dtype == np.float32:
        return rt.view(np.uint32)
    same = rt.view(np.uint32) == init.view(np.uint32)
    return np.where(same, words, _halfbits(rt))


def loaded_target(g, ca, kind, words, dtype):
    """A render target of one memory kind holding `words`; in a layer or a rectangle, every other texel holds a sentinel."""
    return Image(g, ca, kind, words.view(dtype), layers=2, layer=1, rect=RECT)


def _check(got, want, init_words, what):
    bad = np.argwhere((got != want).any(-1))
    if bad.size:
        y, x = bad[0]
        raise AssertionError("%s: %d pixels differ; first (y, x) = (%d, %d): got %s, want %s, loaded %s" % (
            what, len(bad), y, x, [hex(v) for v in got[y, x]], [hex(v) for v in want[y, x]], [hex(v) for v in init_words[y, x]]))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,blend", [(np.float16, 0), (np.float16, 1), (np.float32, 0), (np.float32, 1)],
                         ids=["rgba16f-rop", "rgba16f-fp32", "rgba32f-rop", "rgba32f-fp32"])
def test_loaded_target_content(g, O, ctx, ca, dtype, blend):
    cam = camera(g, W, H)
    asset = loaded_scene(g, cam)
    n = asset.splatCount
    words, init, fam = loaded_content(O, g, asset, cam, dtype)
    fp, _keep = g.make_frame_params(cam)
    z, _, _, _ = quad_depths(O, asset, fp)
    yy, xx = np.mgrid[0:H, 0:W]
    field = z[_hash(xx // 3, yy // 2, 7) % n]
    sel = np.zeros((n + 31) // 32, np.uint32)
    sel[::5] = 0x01010101
    r = g.GaussianSplatRenderer(asset, ctx)
    r.blend_mode = blend
    r.load_rt = True
    for staged in (False, True):
        for extras in (False, True):
            selected, depth = (sel, field) if extras else (None, None)
            rt = oracle_draw(O, g, asset, cam, depth, staged, selected, blend, init)
            want = expectedbits(rt, init, words, dtype)
            # preconditions: every family is in the image, the reached ones where splats blend, and some pixels are untouched
            untouched = (rt.view(np.uint32) == init.view(np.uint32)).all(-1)
            for name, m in fam.items():
                assert m.sum() >= 4, name
            assert untouched[fam["NaN payloads where no splat reaches"]].all()
            assert untouched.sum() > 1000 and (~untouched).sum() > 1000
            if not extras:
                for name in ("alpha 1.5, 8x4 blocks", "alpha 1 + 2^-10, 8x4 blocks", "alpha 1.5", "alpha 65504", "alpha -0.375", "alpha NaN",
                             "alpha 1 - 2^-11"):
                    assert (~untouched[fam[name]]).mean() > 0.5, name + " is mostly not blended into"
            r.m_SelectedBits = selected
            r.sceneDepth = None if depth is None else to_device(depth)
            for kind in ("host", "device", "array", "layer", "rect"):
                t = loaded_target(g, ca, kind, words, dtype)
                gpu_draw(r, cam, t.image, staged)
                _check(bits(t.read(ctx)), want, words, "%s target, %s, %s" % (kind, "gs_calc_view + gs_render" if staged else "gs_frame",
                                                                        "selection + depth" if extras else "plain"))
    r.Dispose()


@pytest.mark.gpu
def test_partitioned_draw_keeps_unowned_rows(g, O, ctx):
    """partition_count 2: a member draws the 64-pixel rows it owns and must hand back every other row as it was loaded."""
    cam = camera(g, W, H)
    asset = loaded_scene(g, cam)
    words, init, _fam = loaded_content(O, g, asset, cam, np.float16)
    want = expectedbits(oracle_draw(O, g, asset, cam, None, False, init=init), init, words, np.float16)
    r = g.GaussianSplatRenderer(asset, ctx)
    r.load_rt = True
    for index in (0, 1):
        owned = ((np.arange(H) // 64) % 2 == index)
        expect = np.where(owned[:, None, None], want, words)
        assert not np.array_equal(expect, want) and not np.array_equal(expect, words)
        r.partition = (index, 2, 1)
        for kind in ("host", "device"):
            t = loaded_target(g, None, kind, words, np.float16)
            gpu_draw(r, cam, t.image, False)
            _check(bits(t.read(ctx)), expect, words, "partition %d of 2, %s target" % (index, kind))
    r.Dispose()
