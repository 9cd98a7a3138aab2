"""The loop-versus-call harness: one gs_frame_objects call against the gs_frame loop it stands for (gs_frame per object,
GS_FLAG_LOAD_RT from the second on, then gs_composite), and one gs_frame_cameras call against the gs_frame_objects loop.
The loop and the call each own a copy of every asset, on one context (`Twins`), and every comparison is bit for bit, on
every render target, every camera target and every asset's persistent draw order and sorted keys."""
import ctypes as C

import numpy as np

from images import Image, bits
from util import camera

QUALITIES = ["Medium", "VeryHigh", "Low", "VeryLow", "Medium", "VeryHigh", "Medium", "VeryHigh"]
SIZES = [6000, 7000, 20000, 9000, 10000, 5000, 4000, 3000]    # Low clusters SH into 16k entries: it needs more splats than that
CAM_SIZES = [(320, 200), (256, 256), (97, 61), (200, 320), (64, 48)]


def mixed_assets(g, n, seed=0xCA3E0F00):
    return [g.synthetic_asset(g.SCENE_CLUSTERED, SIZES[i], seed + i, QUALITIES[i]) for i in range(n)]


def g_trs(**kw):
    import unitygaussiansplatting_b200 as pkg
    return pkg.trs(**kw).astype(np.float32)


def mixed_setup(i, r):
    s = -1.0 if i == 1 else 1.0
    r.localToWorldMatrix = g_trs(position=(1.4 * i - 2.0, 0.2 * i, 0.8 * (i % 2)), scale=(0.8 * s, 0.8, 0.8))
    r.m_SHOrder = (3, 1, 0, 2, 3, 1)[i % 6]
    r.m_SortNthFrame = (1, 2, 1, 3, 1, 2)[i % 6]
    if i == 0:
        r.m_Cutouts = [(np.diag([1 / 0.8, 1 / 0.8, 1 / 0.8, 1.0]).astype(np.float32), 1 | 0x100)]
    if i == 2:
        b = np.random.default_rng(i).integers(0, 2 ** 32, (r.splatCount + 31) // 32, dtype=np.uint64).astype(np.uint32)
        r.m_DeletedBits = b & np.uint32(0x11111111)


def opt(N, blend, flags=0):
    o = N.GsRenderOptions()
    o.blend_mode, o.flags = blend, flags
    return o


def next_sort(r):
    """do_sort of r's next frame (every m_SortNthFrame-th); the frame is counted, and r remembers having sorted once."""
    s = 1 if r.m_FrameCounter % max(1, int(r.m_SortNthFrame)) == 0 else 0
    r.m_FrameCounter += 1
    r.sorted_once = getattr(r, "sorted_once", False) or bool(s)
    return s


def orbit(g, f, W=320, H=200, radius=6.0, phase=0.0):
    t = 0.35 * f + phase
    pos = np.array([radius * np.sin(t), 0.6, -radius * np.cos(t)])
    return camera(g, W, H, pos=tuple(pos), forward=tuple(-pos / np.linalg.norm(pos)))


def frame_args(g, pairs, extras=None, sort=None):
    """gs_frame_objects / gs_frame_cameras arguments for (camera, renderer, depth) pairs in call order: each renderer's frame
    parameters at its camera with `depth` as its scene depth buffer, updated by extras[i] (make_frame_params keywords) when
    given; do_sort from sort(renderer), or 1 without one.  Returns (assets, fps, do_sort, keep): keep holds what fps point to."""
    from unitygaussiansplatting_b200 import _native as N
    n = len(pairs)
    assets, fps, ds, keep = (C.c_void_p * n)(), (N.GsFrameParams * n)(), (C.c_int32 * n)(), []
    for i, (cam, r, depth) in enumerate(pairs):
        kw = dict(localToWorld=r.localToWorldMatrix, splat_scale=r.m_SplatScale, opacity_scale=r.m_OpacityScale,
                  sh_order=r.m_SHOrder, sh_only=r.m_SHOnly, cutouts=r.m_Cutouts, deleted_bits=r.m_DeletedBits,
                  splat_count=r.splatCount, selected_bits=r.m_SelectedBits, scene_depth=depth)
        kw.update(extras[i] if extras else {})
        fps[i], k = g.make_frame_params(cam, **kw)
        assets[i], ds[i] = C.cast(r._asset, C.c_void_p).value, sort(r) if sort else 1
        keep.append(k)
    return assets, fps, ds, keep


def images(N, ims):
    """A GsImage * array of the images (None: a null pointer)."""
    PI = C.POINTER(N.GsImage)
    return (PI * len(ims))(*[C.pointer(x) if x is not None else PI() for x in ims])


def _image(im, cam):
    from unitygaussiansplatting_b200.renderer import _image
    return _image(im, cam.pixelWidth, cam.pixelHeight) if im is not None else None


def _ref(im):
    return C.byref(im) if im is not None else None


def loop_frame(g, ctx, rs, cam, blend, rt, tgt):
    """The definition of gs_frame_objects: gs_frame per object, GS_FLAG_LOAD_RT from the second on, then gs_composite."""
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    a, b = _image(rt, cam), _image(tgt, cam)
    assets, fps, ds, keep = frame_args(g, [(cam, r, r.sceneDepth) for r in rs], sort=next_sort)
    for k in range(len(rs)):
        o = opt(N, blend, N.GS_FLAG_LOAD_RT if k else 0)
        N.check(ctx.handle, lib.gs_frame(ctx.handle, assets[k], C.byref(fps[k]), C.byref(o), ds[k], C.byref(a), None))
    if b is not None:
        N.check(ctx.handle, lib.gs_composite(ctx.handle, C.byref(a), C.byref(b)))


def call_frame(g, ctx, rs, cam, blend, rt, tgt, flags=0, check=True):
    from unitygaussiansplatting_b200 import _native as N
    assets, fps, ds, keep = frame_args(g, [(cam, r, r.sceneDepth) for r in rs], sort=next_sort)
    rc = N.native().gs_frame_objects(ctx.handle, len(rs), assets, fps, ds, C.byref(opt(N, blend, flags)), _ref(_image(rt, cam)),
                                     _ref(_image(tgt, cam)))
    if check:
        N.check(ctx.handle, rc)
    return rc


def _camera_args(g, per_cam, cams, extras):
    """Camera-major frame_args of per_cam[c] = renderers of camera c; extras[c][k]: make_frame_params overrides."""
    pairs = [(cam, r, r.sceneDepth) for rs, cam in zip(per_cam, cams) for r in rs]
    flat = [e for c, rs in enumerate(per_cam) for e in extras[c][:len(rs)]] if extras else None
    return frame_args(g, pairs, flat, sort=next_sort)


def loop_cameras(g, ctx, per_cam, cams, blend, rts, tgts, extras=None):
    """The definition of gs_frame_cameras: gs_frame_objects per camera."""
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    assets, fps, ds, keep = _camera_args(g, per_cam, cams, extras)
    off = 0
    for c, cam in enumerate(cams):
        k = len(per_cam[c])
        rc = lib.gs_frame_objects(ctx.handle, k, C.cast(C.byref(assets, off * C.sizeof(C.c_void_p)), C.POINTER(C.c_void_p)),
                                  C.cast(C.byref(fps, off * C.sizeof(N.GsFrameParams)), C.POINTER(N.GsFrameParams)),
                                  C.cast(C.byref(ds, off * 4), C.POINTER(C.c_int32)), C.byref(opt(N, blend)),
                                  _ref(_image(rts[c], cam)), _ref(_image(tgts[c], cam)))
        N.check(ctx.handle, rc)
        off += k


def call_cameras(g, ctx, per_cam, cams, blend, rts, tgts, extras=None, flags=0, check=True, counts=None, patch=None):
    from unitygaussiansplatting_b200 import _native as N
    assets, fps, ds, keep = _camera_args(g, per_cam, cams, extras)
    ims = [(_image(rt, cam), _image(tg, cam)) for rt, tg, cam in zip(rts, tgts, cams)]
    if patch:
        patch(ims)
    counts = counts if counts is not None else [len(rs) for rs in per_cam]
    rc = N.native().gs_frame_cameras(ctx.handle, len(cams), (C.c_uint32 * len(cams))(*counts), assets, fps, ds,
                                     C.byref(opt(N, blend, flags)), images(N, [a for a, _ in ims]), images(N, [b for _, b in ims]))
    if check:
        N.check(ctx.handle, rc)
    return rc


class Twins:
    """Every asset twice on one context: `loop` draws with the loop, `call` with the one call; setup(i, r) sets both copies
    of asset i up."""

    def __init__(self, g, ctx, assets, setup=None):
        self.loop = [g.GaussianSplatRenderer(a, ctx) for a in assets]
        self.call = [g.GaussianSplatRenderer(a, ctx) for a in assets]
        for i, (p, q) in enumerate(zip(self.loop, self.call)):
            if setup:
                setup(i, p)
                setup(i, q)

    def pick(self, idx_per_cam):
        return [[self.loop[i] for i in ix] for ix in idx_per_cam], [[self.call[i] for i in ix] for ix in idx_per_cam]

    def gathered(self, g, subsets, cams):
        """GatherSplatsForCamera order of each camera's subset of the assets."""
        out = []
        for ix, cam in zip(subsets, cams):
            rs = g.GatherSplatsForCamera([self.loop[i] for i in ix], cam)
            out.append([self.loop.index(r) for r in rs])
        return out

    def ordered(self, g, cam):
        """Every asset in GatherSplatsForCamera order: (loop copies, call copies)."""
        lo, hi = self.pick(self.gathered(g, [range(len(self.loop))], [cam]))
        return lo[0], hi[0]

    def check_state(self):
        for p, q in zip(self.loop, self.call):
            assert np.array_equal(p.readback_order(), q.readback_order()), "draw order"
            assert getattr(p, "sorted_once", False) == getattr(q, "sorted_once", False)
            if getattr(p, "sorted_once", False):   # the keys buffer of an asset never sorted holds whatever its allocation held
                assert np.array_equal(p.readback_keys(), q.readback_keys()), "sorted keys"

    def dispose(self):
        for r in self.loop + self.call:
            r.Dispose()


def _image_of(g, ca, kind, content):
    return Image(g, ca, kind, content) if kind is not None else None


def _read(ctx, im):
    return im.read(ctx) if im is not None else None


def compare_frame(g, ctx, ca, tw, cam, blend, dtype, rt_kind, tgt_kind, what):
    """gs_frame_objects of every asset against the loop, each image in its memory kind (None: no image).  Returns the
    render target."""
    W, H = cam.pixelWidth, cam.pixelHeight
    rng = np.random.default_rng(W + H)
    tgt0 = (rng.random((H, W, 4), np.float32) * 0.5).astype(dtype)
    lo, hi = tw.ordered(g, cam)
    # without an rt the call draws into RGBA16F library scratch, as gs_frame does
    loop_rt = _image_of(g, ca, rt_kind or "device", np.zeros((H, W, 4), dtype if rt_kind else np.float16))
    loop_tgt, call_tgt = _image_of(g, ca, tgt_kind, tgt0), _image_of(g, ca, tgt_kind, tgt0)
    call_rt = _image_of(g, ca, rt_kind, np.full((H, W, 4), 7, dtype))   # the call clears the target itself
    loop_frame(g, ctx, lo, cam, blend, loop_rt.image, loop_tgt and loop_tgt.image)
    call_frame(g, ctx, hi, cam, blend, call_rt and call_rt.image, call_tgt and call_tgt.image)
    want_rt, want_tgt = loop_rt.read(ctx), _read(ctx, loop_tgt)
    assert want_rt.any(), what
    if call_rt is not None:
        assert np.array_equal(bits(call_rt.read(ctx)), bits(want_rt)), what + ": render target"
    if call_tgt is not None:
        assert np.array_equal(bits(call_tgt.read(ctx)), bits(want_tgt)), what + ": camera target"
    tw.check_state()
    return want_rt


def compare(g, ctx, ca, tw, idx_per_cam, cams, blend, dtype, rt_kinds, tgt_kinds, what, extras=None):
    """gs_frame_cameras of idx_per_cam[c] at cams[c] against the camera loop; dtype: one, or one per camera.  Returns how many
    cameras drew something into their render target."""
    lo, hi = tw.pick(idx_per_cam)
    loop_rts, call_rts, loop_tgts, call_tgts = [], [], [], []
    for c, cam in enumerate(cams):
        W, H = cam.pixelWidth, cam.pixelHeight
        dt = dtype[c] if isinstance(dtype, (list, tuple)) else dtype
        tgt0 = (np.random.default_rng(W * 7 + H + c).random((H, W, 4), np.float32) * 0.5).astype(dt)
        rk, tk = rt_kinds[c], tgt_kinds[c]
        loop_rts.append(_image_of(g, ca, rk, np.zeros((H, W, 4), dt)))
        call_rts.append(_image_of(g, ca, rk, np.full((H, W, 4), 7, dt)))   # the call clears each target itself
        loop_tgts.append(_image_of(g, ca, tk, tgt0))
        call_tgts.append(_image_of(g, ca, tk, tgt0))

    def ims(xs):
        return [x and x.image for x in xs]

    loop_cameras(g, ctx, lo, cams, blend, ims(loop_rts), ims(loop_tgts), extras)
    call_cameras(g, ctx, hi, cams, blend, ims(call_rts), ims(call_tgts), extras)
    drawn = 0
    for c in range(len(cams)):
        want_rt, want_tgt = _read(ctx, loop_rts[c]), _read(ctx, loop_tgts[c])
        if want_rt is not None:
            drawn += int(want_rt.any())
            assert np.array_equal(bits(call_rts[c].read(ctx)), bits(want_rt)), "%s: camera %d render target" % (what, c)
        if want_tgt is not None:
            assert np.array_equal(bits(call_tgts[c].read(ctx)), bits(want_tgt)), "%s: camera %d camera target" % (what, c)
    tw.check_state()
    return drawn
