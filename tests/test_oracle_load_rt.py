"""The oracle's draw onto a given target (GS_FLAG_LOAD_RT): it starts from the content it is handed instead of clearing it.
The GPU draws with that flag are compared with it (tests/test_gpu_raster_inputs.py), so its blend on content the kernel never
writes itself -- alpha at, above and below 1, NaN, inf, NaN payloads -- is pinned here against the blend formula written out
in numpy, on one small splat."""
import numpy as np
import pytest

from util import camera, one_splat

W, H = 96, 72


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _u32(v):
    return np.uint32(v).view(np.float32)


@pytest.fixture(scope="module")
def scene(g, O):
    cam = camera(g, W, H, pos=(0, 0, -4.0))
    asset = one_splat(g, pos=(0.02, 0.01, 0.0), scale=(0.08, 0.08, 0.08), opacity=0.6, dc0=(0.8, 0.4, 0.2))
    fp, keep = g.make_frame_params(cam)
    return asset, fp, keep, O.calc_view(asset, fp)


def test_zero_init_is_the_cleared_draw(g, O, scene):
    asset, fp, _keep, view = scene
    order = np.arange(asset.splatCount, dtype=np.uint32)
    zeros = np.zeros((H, W, 4), np.float32)
    depth = np.full((H, W), 0.5, np.float32)
    depth[:, : W // 2] = 0.0
    for blend in (0, 1):
        want = O.render(view, order, W, H, blend)
        assert want[..., 3].any()
        assert np.array_equal(_bits(O.render(view, order, W, H, blend, init=zeros)), _bits(want))
        want_d = O.render(view, order, W, H, blend, scene_depth=depth)
        assert np.array_equal(_bits(O.render(view, order, W, H, blend, scene_depth=depth, init=zeros)), _bits(want_d))
        assert np.array_equal(_bits(O.frame(asset, fp, blend_mode=blend, init=zeros)["rt"]), _bits(O.frame(asset, fp, blend_mode=blend)["rt"]))


def test_loaded_content_follows_the_blend_loop(g, O, scene):
    asset, _fp, _keep, view = scene
    order = np.arange(asset.splatCount, dtype=np.uint32)
    # one splat: a pixel it reaches blends once, and the draw onto zeros in float32 is the source term (premultiplied colour,
    # alpha) itself
    src = O.render(view, order, W, H, 1)
    reached = src[..., 3] > 0
    ys, xs = np.nonzero(reached)
    assert ys.size > 40
    init = np.zeros((H, W, 4), np.float32)
    init[..., :3] = 0.25
    init[..., 3] = 0.5
    families = {   # (colour, alpha) of the loaded pixel
        "alpha 1": ((0.3, 0.2, 0.1), 1.0),
        "alpha 1, inf colour": ((np.inf, -np.inf, 0.5), 1.0),
        "alpha 1, NaN colour": ((_u32(0x7FC01234), 0.0, 0.0), 1.0),
        "alpha 1.5": ((0.5, 0.25, 2.0), 1.5),
        "alpha 65504": ((1.0, 1.0, 1.0), 65504.0),
        "alpha -0.25": ((0.125, -0.5, 0.0), -0.25),
        "alpha 1 - 2^-11": ((0.5, 0.5, 0.5), 1.0 - 2.0 ** -11),
        "alpha NaN": ((0.5, 0.5, 0.5), _u32(0x7FC0BEEF)),
        "alpha inf": ((0.5, 0.5, 0.5), np.inf),
        "inf colour": ((np.inf, -np.inf, 0.0), 0.5),
        "NaN colour": ((_u32(0xFFC00001), 0.5, 0.5), 0.5),
        "-0 and a subnormal": ((-0.0, 2.0 ** -140, -(2.0 ** -149)), 0.0),
    }
    where = {}
    for k, (name, (rgb, a)) in enumerate(families.items()):
        sel = slice(k, None, len(families))
        py, px = ys[sel], xs[sel]
        init[py, px, :3] = np.asarray(rgb, np.float32)
        init[py, px, 3] = np.float32(a)
        where[name] = (py, px)
    # pixels no splat reaches keep every bit: signalling and quiet NaNs with payloads, -0, inf
    far = np.argwhere(~reached)
    specials = np.array([0x7F800001, 0xFF812345, 0x7FC00001, 0xFFFFFFFF, 0x80000000, 0x7F800000, 0x00000001], np.uint32).view(np.float32)
    for k, (py, px) in enumerate(far[:: max(1, far.shape[0] // 70)][:70]):
        init[py, px] = specials[(k + np.arange(4)) % specials.size]

    # the loop as written: dst.a == 1 keeps the pixel; else om = 1 - dst.a, dst = fma(src, om, dst) (fp16 ROP: rounded to
    # half), a NaN result being the canonical NaN
    blendable = reached & ~(init[..., 3] == 1.0)
    with np.errstate(invalid="ignore", over="ignore"):
        om = (np.float32(1.0) - init[..., 3]).astype(np.float64)[..., None]
        fused = (src.astype(np.float64) * om + init.astype(np.float64)).astype(np.float32)
    canonical = 0x7FFFFFFF   # the NaN a GPU blend stores, in either blend mode
    for blend in (1, 0):
        got = O.render(view, order, W, H, blend, init=init)
        want = fused if blend else fused.astype(np.float16).astype(np.float32)
        want = np.where(np.isnan(want), np.uint32(canonical).view(np.float32), want)
        want = np.where(blendable[..., None], want, init)
        assert np.array_equal(_bits(got), _bits(want)), blend
        # spot checks of what the families promise
        for name in ("alpha 1", "alpha 1, inf colour", "alpha 1, NaN colour"):
            py, px = where[name]
            assert np.array_equal(_bits(got[py, px]), _bits(init[py, px])), name
        py, px = where["alpha 1.5"]
        assert (got[py, px, 3] < 1.5).all()            # om < 0: alpha above 1 keeps blending, downwards
        py, px = where["alpha -0.25"]
        assert (got[py, px, 3] > -0.25).all()
        py, px = where["alpha NaN"]
        assert (_bits(got[py, px]) == np.uint32(canonical)).all()
        py, px = where["inf colour"]
        assert (got[py, px, 0] == np.inf).all() and (got[py, px, 1] == -np.inf).all()
        py, px = where["NaN colour"]
        assert (_bits(got[py, px, 0]) == np.uint32(canonical)).all() and np.isfinite(got[py, px, 1:]).all()
        assert np.array_equal(_bits(got[~reached]), _bits(init[~reached]))
