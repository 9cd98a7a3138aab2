"""Shared scene builders for the tests."""
import dataclasses
from collections import namedtuple

import numpy as np

from unitygaussiansplatting_b200.camera import Camera


def camera(g, width=256, height=256, fov=39.09651, pos=(0.0, 0.5, -6.0), forward=(0.0, 0.0, 1.0)):
    return g.Camera(position=np.array(pos, np.float64), rotation=g.look_rotation(forward), fieldOfView=fov, pixelWidth=width,
                    pixelHeight=height)


@dataclasses.dataclass
class ProjCamera(Camera):
    """A Camera whose projectionMatrix is a given OpenGL-style 4x4 (`proj`) instead of the symmetric perspective of
    fieldOfView / aspect.  make_frame_params, SortAndRenderCameras and the group calls all read cam.gpuProjectionMatrix(True),
    so the matrix reaches every entry point unchanged."""
    proj: np.ndarray = None

    @property
    def projectionMatrix(self) -> np.ndarray:
        return np.asarray(self.proj, np.float32)


def with_projection(cam, proj):
    """`cam` (pose, clip planes, screen) with the OpenGL-style projection `proj`."""
    fields = {f.name: getattr(cam, f.name) for f in dataclasses.fields(Camera)}
    return ProjCamera(**fields, proj=np.asarray(proj, np.float64))


def off_axis(cam, l, r, b, t):
    """glFrustum from the near-plane extents (l, r, b, t) at cam.nearClipPlane: an XR eye's projection (P[0,2], P[1,2] != 0)."""
    n, f = cam.nearClipPlane, cam.farClipPlane
    P = np.array([[2 * n / (r - l), 0, (r + l) / (r - l), 0], [0, 2 * n / (t - b), (t + b) / (t - b), 0],
                  [0, 0, -(f + n) / (f - n), -2 * f * n / (f - n)], [0, 0, -1, 0]], np.float64)
    return with_projection(cam, P)


def oblique(cam, plane):
    """Camera.CalculateObliqueMatrix: the near plane of cam's projection replaced by `plane` (a, b, c, d), a camera-space
    plane with the camera on its negative side, as a planar-reflection camera uses it (Lengyel's construction)."""
    P = np.asarray(cam.projectionMatrix, np.float64)
    c = np.asarray(plane, np.float64)
    q = np.linalg.inv(P) @ np.array([np.sign(c[0]), np.sign(c[1]), 1.0, 1.0])
    c = c * (2.0 / (c @ q))
    P = P.copy()
    P[2] = c - P[3]
    return with_projection(cam, P)


def mirrored(cam):
    """P diag(-1, 1, 1, 1): a mirror camera's projection (x flipped, so p00 < 0)."""
    return with_projection(cam, np.asarray(cam.projectionMatrix, np.float64) @ np.diag([-1.0, 1.0, 1.0, 1.0]))


def orthographic(cam, half_height):
    """glOrtho of `half_height` world units up and down (and the screen's aspect across) between cam's clip planes: clip.w
    is 1 everywhere, so no splat is behind the camera and only the view depth tells the chunk cull where the camera plane is."""
    n, f, hw = cam.nearClipPlane, cam.farClipPlane, half_height * cam.aspect
    return with_projection(cam, [[1 / hw, 0, 0, 0], [0, 1 / half_height, 0, 0], [0, 0, -2 / (f - n), -(f + n) / (f - n)], [0, 0, 0, 1]])


def rolled(cam, deg):
    """`cam` turned by `deg` degrees about its own view axis."""
    a = np.radians(deg)
    rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]], np.float64)
    return dataclasses.replace(cam, rotation=np.asarray(cam.rotation, np.float64) @ rz)


# Camera poses XR and walk-through users render, at screens the oracle draws quickly (tests/test_gpu_camera_poses.py).
# The clustered scene has its clusters in [-8, 8] x [-2, 3] x [-8, 8] and a shell of splats at radius 8..30, so every "inside"
# pose is among the splats; `inside-near` looks at the cluster next to it.
XR_EYE = (-1.4, 0.9, -1.2, 1.1)        # near-plane extents / n of the left eye; the right eye is its mirror image


def xr_eye(g, eye, width=256, height=256, pos=(0.3, 0.4, -1.0), forward=(0.2, -0.1, 1.0), ipd=0.064):
    """The left (eye 0) or right (eye 1) eye of a head at `pos`: an off-axis frustum about 97 degrees across each way."""
    l, r, b, t = XR_EYE
    if eye:
        l, r = -r, -l
    head = camera(g, width, height, pos=pos, forward=forward)
    right = np.asarray(head.rotation, np.float64)[:, 0]
    c = dataclasses.replace(head, position=np.asarray(pos, np.float64) + (eye - 0.5) * ipd * right)
    n = c.nearClipPlane
    return off_axis(c, l * n, r * n, b * n, t * n)


def _poses():
    def inside(forward, pos=(0.0, 0.5, 0.0), width=256, height=256, fov=90.0):
        return lambda g: camera(g, width, height, fov=fov, pos=pos, forward=forward)

    return {
        "inside-z": inside((0.0, 0.0, 1.0)),
        "inside-back": inside((0.0, 0.0, -1.0)),
        "inside-near": inside((0.45, -0.35, 0.8), pos=(-1.3, 0.4, 1.6)),
        "xr-left": lambda g: xr_eye(g, 0),
        "xr-right": lambda g: xr_eye(g, 1),
        "roll-30": lambda g: rolled(camera(g, 320, 240, pos=(0.4, 0.8, -5.0), forward=(-0.1, -0.1, 1.0)), 30.0),
        "roll-90": lambda g: rolled(camera(g, 320, 240, pos=(0.4, 0.8, -5.0), forward=(-0.1, -0.1, 1.0)), 90.0),
        "roll-180": lambda g: rolled(camera(g, 320, 240, pos=(0.4, 0.8, -5.0), forward=(-0.1, -0.1, 1.0)), 180.0),
        "fov-110": lambda g: camera(g, 320, 240, fov=110.0, pos=(0.0, 0.5, -3.0)),
        "fov-3": lambda g: camera(g, 320, 240, fov=3.0, pos=(0.0, 0.5, -20.0), forward=(0.05, 0.0, 1.0)),
        "portrait": lambda g: camera(g, 240, 320, fov=60.0, pos=(0.5, 0.5, -4.0)),
        "strip-wide": lambda g: camera(g, 1024, 64, fov=12.0, pos=(0.0, 0.5, -6.0)),
        "strip-tall": lambda g: camera(g, 64, 1024, fov=90.0, pos=(0.0, 0.5, -6.0)),
        "mirrored": lambda g: mirrored(camera(g, 320, 240, fov=60.0, pos=(0.6, 0.7, -4.5), forward=(-0.15, -0.05, 1.0))),
        "ortho-inside": lambda g: orthographic(camera(g, 256, 256, pos=(0.0, 0.5, 0.0), forward=(1.0, 0.0, 0.2)), 1.0),
        "oblique": lambda g: oblique(camera(g, 320, 240, fov=60.0, pos=(0.0, 1.5, -5.0), forward=(0.0, -0.2, 1.0)),
                                     (0.0, 0.35, -0.94, -2.5)),
    }


POSES = _poses()

# The near-plane scene: splats at view depths NEAR_DEPTHS whose centres lie NEAR_OFFSETS pixels outside each edge of the
# screen -- across the 11,880 px far_off reach of a clamped quad (quad_reach of an unbounded footprint), the 4096 px axis
# clamp, and the 1e7 px no-raster cut-off of splat_footprint.
NEAR_DEPTHS = (1e-3, -1e-3, 1e-6, -1e-6, 0.0)
NEAR_OFFSETS = (-20.0, 40.0, 3900.0, 4300.0, 11000.0, 12500.0, 9.8e6, 1.03e7)
NEAR_SCALES = (0.002, 0.03, 0.4)


def near_plane_camera(g):
    """An XR left eye at the origin looking along +z: its view matrix is diag(1, 1, -1, 1), so view depth is world z exactly."""
    return xr_eye(g, 0, 256, 256, pos=(0.0, 0.0, 0.0), forward=(0.0, 0.0, 1.0), ipd=0.0)


def near_plane_scene(g, cam):
    """VeryHigh asset of the near-plane scene seen by `cam` (near_plane_camera)."""
    P = cam.gpuProjectionMatrix(True).astype(np.float64)
    W, H = cam.pixelWidth, cam.pixelHeight
    rng = np.random.default_rng(11)
    pos, scale = [], []
    for d in NEAR_DEPTHS:
        a = abs(d) if d else 1e-3
        for o in NEAR_OFFSETS:
            for edge in range(4):
                for s in NEAR_SCALES:
                    t = rng.uniform(0.2, 0.8)
                    px, py = ((-o, t * H), (W + o, t * H), (t * W, -o), (t * W, H + o))[edge]
                    ndx, ndy = 2 * px / W - 1, 1 - 2 * py / H
                    # clip = P (x, y, -a, 1): clip.w = a, clip.x = P00 x - P02 a, clip.y = P11 y - P12 a
                    pos.append(((ndx + P[0, 2]) * a / P[0, 0], (ndy + P[1, 2]) * a / P[1, 1], d))
                    scale.append((s, s * rng.uniform(0.05, 1.0), s * rng.uniform(0.05, 1.0)))
    n = len(pos)
    rec = splat_records(np.array(pos), np.array(scale), rng.uniform(0.3, 1.0, n), dc=rng.uniform(0, 1, (n, 3)),
                        quat=rng.standard_normal((n, 4)))
    return g.create_asset(rec, "VeryHigh")


def lattice_camera(g, width=256, height=256):
    # cfg1: 1k lattice in [-1,1]^3 seen from -z, axis aligned so the un-jittered z planes tie
    return camera(g, width, height, fov=39.09651, pos=(0.0, 0.0, -4.0))


def one_splat(g, pos=(0, 0, 0), scale=(0.1, 0.1, 0.1), quat=(0, 0, 0, 1), opacity=0.8, dc0=(0.9, 0.5, 0.2), sh=None, n_pad=0,
              quality="VeryHigh"):
    """Asset with one hand-made splat (+ optional far-away padding splats)."""
    import ctypes as C
    from unitygaussiansplatting_b200 import _native as N
    n = 1 + n_pad
    rec = np.zeros((n, 62), np.float32)
    q = np.asarray(quat, np.float32)
    q = q / np.linalg.norm(q)
    packed = np.zeros(4, np.float32)
    N.asset_lib().gsa_pack_smallest3(q.ctypes.data, packed.ctypes.data)
    for i in range(n):
        rec[i, 0:3] = pos if i == 0 else (1000.0 + i, 1000.0, 1000.0)
        rec[i, 6:9] = dc0
        if sh is not None and i == 0:
            rec[i, 9:54] = np.asarray(sh, np.float32).reshape(45)
        rec[i, 54] = opacity
        rec[i, 55:58] = scale
        rec[i, 58:62] = packed
    return g.create_asset(rec, quality)


def splat_records(pos, scale, opacity, dc=(0.9, 0.5, 0.2), quat=(0, 0, 0, 1)):
    """(n, 62) float32 InputSplatData records; every argument is one value for all splats or one row per splat."""
    from unitygaussiansplatting_b200 import _native as N
    pos = np.atleast_2d(np.asarray(pos, np.float32))
    n = pos.shape[0]
    q = np.broadcast_to(np.atleast_2d(np.asarray(quat, np.float64)), (n, 4))
    uq, inv = np.unique(q, axis=0, return_inverse=True)
    packed = np.zeros((uq.shape[0], 4), np.float32)
    for k in range(uq.shape[0]):
        u = (uq[k] / np.linalg.norm(uq[k])).astype(np.float32)
        N.asset_lib().gsa_pack_smallest3(u.ctypes.data, packed[k].ctypes.data)
    rec = np.zeros((n, 62), np.float32)
    rec[:, 0:3] = pos
    rec[:, 6:9] = dc
    rec[:, 54] = opacity
    rec[:, 55:58] = scale
    rec[:, 58:62] = packed[inv.reshape(-1)]
    return rec


def world_at_pixel(cam, x, y, depth):
    """World points whose screen centre is at pixel coordinates (x, y) (pixel (i, j) spans [i, i+1) x [j, j+1)), `depth`
    world units in front of the camera: the inverse of the D3D viewport transform and the projection, in float64."""
    x, y, depth = np.broadcast_arrays(*(np.asarray(v, np.float64) for v in (x, y, depth)))
    p = cam.gpuProjectionMatrix(True).astype(np.float64)
    ndx, ndy = 2.0 * x / cam.pixelWidth - 1.0, 1.0 - 2.0 * y / cam.pixelHeight
    v = np.stack([ndx * depth / p[0, 0], ndy * depth / p[1, 1], -depth, np.ones_like(depth)], axis=-1)
    w = v @ np.linalg.inv(cam.worldToCameraMatrix.astype(np.float64)).T
    return w[..., :3]


def pixels_per_unit(cam, depth):
    """Screen pixels per world unit, across the screen, at `depth` in front of the camera."""
    return cam.gpuProjectionMatrix(True).astype(np.float64)[0, 0] * cam.pixelWidth * 0.5 / depth


def view_fields(view):
    """(n,10) uint32 SplatViewData -> dict of float arrays."""
    v = np.ascontiguousarray(view, np.uint32)
    f = v.view(np.float32)
    col = v[:, 8:10]
    def h(x):
        return (x & 0xFFFF).astype(np.uint16).view(np.float16).astype(np.float32)
    return {"pos": f[:, 0:4], "axis1": f[:, 4:6], "axis2": f[:, 6:8], "r": h(col[:, 0] >> 16), "g": h(col[:, 0]), "b": h(col[:, 1] >> 16),
            "a": h(col[:, 1])}



def unsortable(keys):
    """The float32 view depths the sortable uint32 distance keys encode."""
    k = keys.astype(np.uint32)
    u = np.where(k & 0x80000000, k ^ np.uint32(0x80000000), ~k).astype(np.uint32)
    return u.view(np.float32)


def screen_cov(v):
    """The 2-D screen covariance 0.5 (axis1 axis1^T + axis2 axis2^T) of view_fields' axes, in float64."""
    a1, a2 = v["axis1"].astype(np.float64), v["axis2"].astype(np.float64)
    return 0.5 * (a1[:, :, None] * a1[:, None, :] + a2[:, :, None] * a2[:, None, :])


# ---- the bin list at its capacity ---------------------------------------------------------------------------------------
CAP_W, CAP_H = 4096, 2048         # 64 x 32 bins: two 6-bit sort passes
CAP_ENTRIES = 4 << 20             # clamp(8 N, 4 Mi, 768 Mi) for N < 512 Ki
CAP_SPLATS = CAP_ENTRIES // 64    # one full bin row (64 entries) each


def bin_row_splats(cam, n, seed):
    """n wide, flat splats: each one's visible part spans the whole screen width and 5 rows inside one 64-pixel bin row, so
    it emits exactly 64 (bin, splat) entries while the oracle visits only about 4096 x 9 pixels of it."""
    rng = np.random.default_rng(seed)
    i = np.arange(n)
    depth = 5.0 + 3.0 * rng.random(n)
    cy = 64.0 * (i % (CAP_H // 64)) + 20.0 + (i // (CAP_H // 64)) % 25
    pos = world_at_pixel(cam, CAP_W / 2, cy, depth)
    ppu = pixels_per_unit(cam, depth)[:, None]
    scale = np.array([0.3 * CAP_W, 0.01, 0.01]) / ppu      # axis1 ~ 0.42 W: the quad reaches 0.85 W beyond the centre
    dc = rng.random((n, 3)) * 2.0 - 0.5
    return splat_records(pos, scale, 0.05 + 0.3 * rng.random(n), dc)


# ---- the bin sort's plans at their edges --------------------------------------------------------------------------------
# (width, height): bins = ceil(W/64) * ceil(H/64); bin_sort_plan takes one pass up to 512 bins (5, 6, 7, 8, 9 bits at 32, 64,
# 128, 256, 512), else two passes of 5, 6, 7, 8 bits up to 1024, 4096, 16384, 65536 bins.  Each plan up to 7 bits at its upper
# edge and one past it.
PLAN_SCREENS = [
    ((512, 256), 32, 1, 5), ((704, 192), 33, 1, 6),
    ((512, 512), 64, 1, 6), ((832, 320), 65, 1, 7),
    ((1024, 512), 128, 1, 7), ((2752, 192), 129, 1, 8),
    ((1024, 1024), 256, 1, 8), ((2752, 384), 258, 1, 9),        # 257 bins is prime: it would need a 16448-pixel row
    ((1920, 1080), 510, 1, 9), ((2048, 1024), 512, 1, 9),
    ((2048, 1088), 544, 2, 5), ((1728, 1216), 513, 2, 5),
    ((2048, 2048), 1024, 2, 5), ((2624, 1600), 1025, 2, 6),
    ((4096, 4096), 4096, 2, 6), ((5248, 3200), 4100, 2, 7),
    ((8160, 8160), 16384, 2, 7),                                # also the largest camera a camera run takes
]


def plan_scene(g, cam, entries):
    """The clustered scene, a few small splats in the bottom-right bin (where a digit one bit too narrow mis-sorts), and,
    when `entries` is set, wide flat splats across the whole screen on the bin-row boundaries: 2 x binsX entries each,
    as many as give about `entries`."""
    W, H = cam.pixelWidth, cam.pixelHeight
    base = g.generate_input_splats(g.SCENE_CLUSTERED, 60000, 0x5EED0002)
    ppu = pixels_per_unit(cam, 6.0)
    corner = splat_records(world_at_pixel(cam, [W - 20.5, W - 6.0, W - 40.2], [H - 18.3, H - 40.0, H - 5.5], 6.0),
                           np.array([3.0, 2.0, 2.5]) / ppu, 0.9, (0.2, 0.9, 0.4))
    parts = [base, corner]
    if entries:
        bins_x, bins_y = -(-W // 64), -(-H // 64)
        n = -(-entries // (2 * bins_x))
        rng = np.random.default_rng(W * H)
        depth = 5.0 + 3.0 * rng.random(n)
        cy = 64.0 * (1 + np.arange(n) % (bins_y - 1))
        scale = np.array([0.3 * W, 0.01, 0.01]) / pixels_per_unit(cam, depth)[:, None]
        parts.append(splat_records(world_at_pixel(cam, W / 2, cy, depth), scale, 0.1 + 0.3 * rng.random(n), rng.random((n, 3))))
    return g.create_asset(np.ascontiguousarray(np.concatenate(parts)), "Medium")


# ---- asset format combinations no preset uses ------------------------------------------------------------------------------
# The importer's Custom quality lets a user pick any (position, scale, colour, SH) format.  One list of combinations, chosen so
# that between them they reach every decode path of the view, distance and export kernels (tests/test_format_cases.py checks
# that they still do); tests/test_gpu_formats.py, tests/test_gpu_pack.py and the reference-shader fixtures all draw from it.
# Codes: vector 0 Float32, 1 Norm16, 2 Norm11, 3 Norm6; colour 0 Float32x4, 1 Float16x4, 2 Norm8x4, 3 BC7;
# SH 0 Float32, 1 Float16, 2 Norm11, 3 Norm6, 4..8 Cluster64k..Cluster4k.
# `n` is the splat count of the GPU comparison; `indices`: the clustered palette indices are rewritten over all of 0..65535.
FormatCase = namedtuple("FormatCase", "name formats n indices")
FORMAT_CASES = (
    FormatCase("norm6pos-f16sh", (3, 3, 0, 1), 4865, False),      # Norm6 position; 6-byte `other`; chunked Float32x4 colour
    FormatCase("f32pos-bc7-f16sh", (0, 1, 3, 1), 5003, False),    # chunked Float32 position; Float16 SH with BC7
    FormatCase("f32sh-bc7", (1, 0, 3, 0), 3001, False),           # 16-byte `other`; chunked but not lerped Float32 SH
    FormatCase("norm11sh-bc7", (2, 3, 3, 2), 2819, False),        # 6-byte `other`; Norm11 SH with BC7
    FormatCase("norm6sh-bc7", (3, 2, 3, 3), 4098, False),         # 8-byte `other`; Norm6 SH with BC7; the one even count
    FormatCase("f32sh-chunked", (0, 2, 0, 0), 2305, False),       # Float32 SH and colour, chunked because scale is Norm11
    FormatCase("norm11sh-f16col", (2, 2, 1, 2), 2561, False),     # Norm11 SH without BC7
    FormatCase("norm6sh-norm8col", (1, 3, 2, 3), 3331, False),    # Norm6 SH without BC7; 6-byte `other`
    FormatCase("cluster64k", (0, 0, 1, 4), 4099, True),           # clustered 18-byte `other` (Float32 scale at 2-aligned)
    FormatCase("cluster32k", (1, 2, 0, 5), 4353, True),           # clustered 10-byte `other`
    FormatCase("cluster16k", (1, 3, 1, 6), 4611, True),           # clustered 8-byte `other` with Norm6 scale
    FormatCase("cluster8k", (2, 1, 2, 7), 8195, False),           # clustered 12-byte `other`, packed by the host
    FormatCase("cluster4k", (3, 0, 1, 8), 4097, False),           # clustered 18-byte `other` with Norm6 position
    FormatCase("cluster4k-oob-bc7", (3, 0, 3, 8), 4391, True),    # ... with BC7, and indices past the 4096-entry palette
)
FORMAT_SEED = 0x5EED0C00


def format_case(name):
    return next(c for c in FORMAT_CASES if c.name == name)


def case_asset(g, case, n=None, seed=FORMAT_SEED):
    """The asset of a FormatCase: a clustered scene of `n` (default case.n) splats packed by the host.  Host k-means at 16k,
    32k and 64k entries is too slow for a test, so those are a host-packed Cluster4k asset with the same vector and colour
    formats whose palette is replaced by a seeded one of that size; where case.indices is set, every splat's palette index
    (the trailing u16 of its `other` record) is replaced by a seeded value in 0..65535, a quarter or more of them >= 32768."""
    pf, sf, cf, shf = case.formats
    n = case.n if n is None else n
    host_sh = 8 if shf in (4, 5, 6) else shf
    asset = g.create_asset(g.generate_input_splats(1, n, seed), formats=(pf, sf, cf, host_sh))   # 1: SCENE_CLUSTERED
    rng = np.random.default_rng(seed + case.formats[3])
    if shf != host_sh:
        entries = 65536 >> (shf - 4)
        pal = np.zeros((entries, 48), np.float16)            # SHTableItemFloat16: 45 halfs + 3 of padding = 96 bytes
        pal[:, :45] = rng.uniform(-0.6, 0.6, (entries, 45))
        asset.shData = pal.view(np.uint8).reshape(-1)
        asset.shFormat = g.SHFormat(shf)
    if case.indices:
        stride = 4 + (12, 6, 4, 2)[sf] + 2
        rec = asset.otherData[:n * stride].reshape(n, stride)
        idx = rng.integers(0, 65536, n, dtype=np.uint16)
        assert (idx >= 32768).mean() >= 0.25
        rec[:, stride - 2:] = idx.view(np.uint8).reshape(n, 2)
    return asset


def palette_backed(asset):
    """`asset` with a clustered palette zero-padded to 65536 entries: any u16 index names an entry, and the device backs all
    of them with zeros (gs_asset_upload), so this is the asset a host-side decoder has to read to see the same splats."""
    if asset.shFormat <= 3 or asset.shData.nbytes >= 65536 * 96:
        return asset
    sh = np.zeros(65536 * 96, np.uint8)
    sh[:asset.shData.nbytes] = asset.shData
    return dataclasses.replace(asset, shData=sh)
