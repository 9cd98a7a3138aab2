"""Host-side mirror of GaussianSplatRenderer (package/Runtime/GaussianSplatRenderer.cs) on top of
the C ABI.  Same member names, argument meaning and order of operations as the C# component for
the hot path; everything it does is a call into libgsplat_b200.so (there is no CPU path here).

  C#                                          here
  ------------------------------------------  ------------------------------------------------
  OnEnable -> CreateResourcesForAsset (:373)   GaussianSplatRenderer(asset)  -> gs_asset_upload
  (a further renderer of the same asset)       renderer.Instance()           -> gs_asset_instance
  SortPoints(cmd, cam, matrix)        (:612)   SortPoints(cam)               -> gs_sort
  CalcViewData(cmb, cam)              (:579)   CalcViewData(cam)             -> gs_calc_view
  cmb.DrawProcedural(matSplats)       (:165)   DrawSplats(cam, rt)           -> gs_render
  composite DrawProcedural            (:206)   Composite(rt, target)         -> gs_composite
  SortAndRenderSplats(cam, cmb)       (:108)   SortAndRenderSplats(cam, ...) -> gs_frame
  (several objects of one camera)              SortAndRenderSplatsMulti(...) -> gs_frame_objects
  camera loop, OnPreCullCamera        (:187)   SortAndRenderCameras(...)     -> gs_frame_cameras
                                               (via_event=True: GS_UNITY_EVENT_FRAME_CAMERAS, the render-thread event)
  OnDisable / DisposeResourcesForAsset(:533)   Dispose()
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _native as N
from .asset import GaussianSplatAsset
from .camera import Camera, colmajor

_PIX_DTYPES = {N.GS_PIX_RGBA16F: np.float16, N.GS_PIX_RGBA32F: np.float32}


class GaussianSplatContext:
    """One per CUDA device (GsContext)."""

    def __init__(self, device: int = 0, stream: int = 0):
        self._lib = N.native()
        h = C.c_void_p()
        N.check(None, self._lib.gs_create(device, C.c_void_p(stream) if stream else None, C.byref(h)))
        self.handle = h
        self.device = device

    @classmethod
    def from_handle(cls, handle, device: int = -1):
        """A context the library owns (the members of gs_group_create): wrapped, never destroyed from here."""
        self = cls.__new__(cls)
        self._lib = N.native()
        self.handle = C.c_void_p(handle) if not isinstance(handle, C.c_void_p) else handle
        self.device = device
        self._borrowed = True
        return self

    def sync(self):
        N.check(self.handle, self._lib.gs_sync(self.handle))

    def set_timing(self, enabled: bool):
        N.check(self.handle, self._lib.gs_set_timing(self.handle, 1 if enabled else 0))

    def stage_times(self) -> N.GsStageTimes:
        t = N.GsStageTimes()
        N.check(self.handle, self._lib.gs_get_stage_times(self.handle, C.byref(t)))
        return t

    @property
    def stream(self) -> int:
        return int(self._lib.gs_context_stream(self.handle) or 0)

    def sort_pairs(self, keys: np.ndarray, payload: np.ndarray):
        """GpuSorting.Dispatch on host arrays (in place)."""
        assert keys.dtype == np.uint32 and payload.dtype == np.uint32 and keys.size == payload.size
        assert keys.flags.c_contiguous and payload.flags.c_contiguous
        N.check(self.handle, self._lib.gs_sort_pairs_host(self.handle, keys.ctypes.data, payload.ctypes.data, keys.size))

    def sort_pairs_device(self, d_keys: int, d_payload: int, count: int):
        N.check(self.handle, self._lib.gs_sort_pairs_device(self.handle, d_keys, d_payload, count))

    def close(self):
        if self.handle:
            if not getattr(self, "_borrowed", False):
                self._lib.gs_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _array_descriptor(what, handle, layer, origin):
    """The GsArrayLayer / GsArrayRect a CUDA-array image or depth buffer points to (None for a whole 2-D array), and its memory
    kind.  origin (x, y): the texel of the array that holds pixel (0, 0), a GS_MEM_ARRAY_RECT rectangle."""
    if layer is not None:
        layer = int(layer)
        if not 0 <= layer < 2 ** 32:
            raise ValueError("%s layer must be a non-negative 32-bit index" % what)
    if origin is None:
        if layer is None:
            return None, N.GS_MEM_ARRAY
        return N.GsArrayLayer(handle, layer, 0), N.GS_MEM_ARRAY_LAYER
    try:
        x, y = origin
    except (TypeError, ValueError):
        raise ValueError("%s origin must be a pair (x, y)" % what) from None
    return N.GsArrayRect(handle, layer or 0, _index32(what, "origin", x), _index32(what, "origin", y), 0), N.GS_MEM_ARRAY_RECT


def _index32(what, name, v):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not 0 <= int(v) < 2 ** 32:
        raise ValueError("%s %s must hold non-negative 32-bit integers" % (what, name))
    return int(v)


class CudaArrayImage:
    """A 2-D CUDA array (cudaArray_t, e.g. an imported graphics render texture) of RGBA float16 or float32 texels, given to the
    library as an image (GS_MEM_ARRAY): it is rendered into / composited onto in place.  dtype uint32: an array of one 32-bit
    unsigned channel holding GS_PIX_B10G11R11_UFLOAT texels (a URP / HDRP camera colour buffer), a camera target only.  dtype
    uint8: an array of four 8-bit unsigned channels holding GS_PIX_R8G8B8A8_SRGB texels (an LDR camera's colour buffer), a
    camera target only.  The host creates the array, with cudaArraySurfaceLoadStore, and keeps it alive; the library never
    allocates or frees one.

    layer: the array is a layered one (cudaArrayLayered, e.g. an XR eye-texture array or a cube map) and the image is this
    layer of it (GS_MEM_ARRAY_LAYER); the other layers are left as they are.
    origin (x, y): the image is the width x height rectangle at texel (x, y) of the array (of its `layer` when it is layered;
    GS_MEM_ARRAY_RECT), e.g. a camera's part of a larger HDRP render target, or one view's tile of an atlas.  The texels outside
    the rectangle are left as they are."""

    def __init__(self, handle: int, width: int, height: int, dtype=np.float16, layer=None, origin=None):
        self.handle = int(handle)
        self.width, self.height = int(width), int(height)
        self.dtype = np.dtype(dtype)
        if self.dtype not in (np.float16, np.float32, np.uint32, np.uint8):
            raise ValueError("CudaArrayImage dtype must be float16, float32, uint32 or uint8")
        # the descriptor a GS_MEM_ARRAY_LAYER / GS_MEM_ARRAY_RECT image points to, alive as long as this object
        self._layer_desc, self.memory = _array_descriptor("CudaArrayImage", self.handle, layer, origin)
        self.layer = None if layer is None else int(layer)
        self.origin = None if origin is None else (int(origin[0]), int(origin[1]))

    @property
    def shape(self):
        return (self.height, self.width) if self.dtype == np.uint32 else (self.height, self.width, 4)


class CudaArrayDepth:
    """A scene depth buffer in a CUDA array (cudaArray_t, e.g. a camera's depth copied into an imported R32 float texture): a
    2-D array of one float32 channel (GS_MEM_ARRAY), or with `layer` that layer of a layered one (GS_MEM_ARRAY_LAYER, e.g. one
    eye of an XR eye-depth array), or with `origin` (x, y) the width x height rectangle at that texel of either
    (GS_MEM_ARRAY_RECT, e.g. the camera's part of a larger HDRP depth texture).  Texel (x + px, y + py) is the depth of pixel
    (px, py), reversed Z as for a depth tensor.  The array must have been created with cudaArraySurfaceLoadStore (and
    cudaArrayLayered for a layer); the host keeps it alive."""

    def __init__(self, handle: int, width: int, height: int, layer=None, origin=None):
        self.handle = int(handle)
        self.width, self.height = int(width), int(height)
        if self.width < 1 or self.height < 1:
            raise ValueError("CudaArrayDepth width and height must be positive")
        # the descriptor a GS_MEM_ARRAY_LAYER / GS_MEM_ARRAY_RECT depth buffer points to, alive as long as this object
        self._layer_desc, self.memory = _array_descriptor("CudaArrayDepth", self.handle, layer, origin)
        self.layer = None if layer is None else int(layer)
        self.origin = None if origin is None else (int(origin[0]), int(origin[1]))

    @property
    def shape(self):
        return (self.height, self.width)


def _image(arr, width: int, height: int) -> N.GsImage:
    """numpy (host) array or torch CUDA tensor of shape (H, W, 4), float16/float32 or uint8 (GS_PIX_R8G8B8A8_SRGB texels), or
    (H, W) uint32 (int32 for a tensor) of packed GS_PIX_B10G11R11_UFLOAT texels, or a CudaArrayImage -> GsImage."""
    im = N.GsImage()
    im.width, im.height = width, height
    if isinstance(arr, CudaArrayImage):
        if arr.shape[:2] != (height, width):
            raise ValueError("CUDA array is %dx%d, the image must be %dx%d" % (arr.width, arr.height, width, height))
        im.format = {np.float16: N.GS_PIX_RGBA16F, np.float32: N.GS_PIX_RGBA32F, np.uint32: N.GS_PIX_B10G11R11_UFLOAT,
                     np.uint8: N.GS_PIX_R8G8B8A8_SRGB}[arr.dtype.type]
        if arr._layer_desc is None:
            im.data, im.memory = arr.handle, N.GS_MEM_ARRAY
        else:
            im.data, im.memory = C.addressof(arr._layer_desc), arr.memory
            im._layer_desc = arr._layer_desc   # the descriptor lives as long as the image that points to it
        im.row_pitch_bytes = 0
        return im
    if isinstance(arr, np.ndarray):
        if arr.dtype == np.uint32:
            if arr.shape != (height, width) or not arr.flags.c_contiguous:
                raise ValueError("a packed image must be C-contiguous (H, W) uint32")
            im.format = N.GS_PIX_B10G11R11_UFLOAT
        else:
            if arr.shape != (height, width, 4) or not arr.flags.c_contiguous:
                raise ValueError("image must be C-contiguous (H, W, 4)")
            if arr.dtype == np.float16:
                im.format = N.GS_PIX_RGBA16F
            elif arr.dtype == np.float32:
                im.format = N.GS_PIX_RGBA32F
            elif arr.dtype == np.uint8:
                im.format = N.GS_PIX_R8G8B8A8_SRGB
            else:
                raise ValueError("image dtype must be float16, float32, uint8 (sRGB) or (packed) uint32")
        im.data, im.memory = arr.ctypes.data, N.GS_MEM_HOST
        im.row_pitch_bytes = arr.strides[0]
        return im
    # torch tensor (duck-typed so torch stays optional)
    if str(arr.dtype) in ("torch.int32", "torch.uint32"):
        if tuple(arr.shape) != (height, width) or not arr.is_contiguous():
            raise ValueError("a packed image must be contiguous (H, W)")
        im.format = N.GS_PIX_B10G11R11_UFLOAT
        im.data = arr.data_ptr()
        im.memory = N.GS_MEM_DEVICE if arr.is_cuda else N.GS_MEM_HOST
        im.row_pitch_bytes = width * 4
        return im
    if tuple(arr.shape) != (height, width, 4) or not arr.is_contiguous():
        raise ValueError("image must be contiguous (H, W, 4)")
    es = arr.element_size()
    im.format = N.GS_PIX_R8G8B8A8_SRGB if str(arr.dtype) == "torch.uint8" else N.GS_PIX_RGBA16F if es == 2 else N.GS_PIX_RGBA32F
    im.data = arr.data_ptr()
    im.memory = N.GS_MEM_DEVICE if arr.is_cuda else N.GS_MEM_HOST
    im.row_pitch_bytes = width * 4 * es
    return im


def _to_ufloat(x: np.ndarray, m: int) -> np.ndarray:
    """float32 -> unsigned float of 5 exponent bits (bias 15) and m mantissa bits, as include/gsplat_b200.h states it."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.int64)
    inf = 31 << m
    e = (u >> 23) - 127
    mant = u & 0x7FFFFF
    sub = e < -14   # a denormal code (its value below 2^-14)
    shift = np.where(sub, 23 - m + np.clip(-14 - e, 0, 40), 23 - m)
    mant = np.where(sub, mant | 0x800000, mant)
    h = np.where(sub, 0, np.clip(e + 15, 0, 64) << m) + (mant >> np.minimum(shift, 40))
    rem = mant & ((np.int64(1) << shift) - 1)
    half = np.int64(1) << (shift - 1)
    h = h + ((rem > half) | ((rem == half) & ((h & 1) == 1)))
    h = np.where((e < -15 - m), 0, np.minimum(h, inf))
    h = np.where(u == 0x7F800000, inf, h)
    h = np.where((u >> 31) == 1, 0, h)
    h = np.where((u & 0x7FFFFFFF) > 0x7F800000, inf | ((1 << m) - 1), h)
    return h.astype(np.uint32)


def _from_ufloat(c: np.ndarray, m: int) -> np.ndarray:
    c = np.asarray(c, np.uint32)
    e, mant = (c >> m) & 31, c & ((1 << m) - 1)
    normal = (((e + 112) << 23) | (mant << (23 - m))).astype(np.uint32).view(np.float32)
    special = np.where(mant != 0, np.uint32(0x7FC00000) | (mant << (23 - m)), np.uint32(0x7F800000)).astype(np.uint32).view(np.float32)
    denormal = mant.astype(np.float32) * np.float32(2.0 ** (-14 - m))
    return np.where(e == 0, denormal, np.where(e == 31, special, normal))


def pack_b10g11r11(rgb) -> np.ndarray:
    """(..., 3) float32 linear colours -> (...) uint32 GS_PIX_B10G11R11_UFLOAT texels (R bits 0-10, G 11-21, B 22-31), rounded as
    the library's composite rounds them."""
    rgb = np.asarray(rgb, np.float32)
    return _to_ufloat(rgb[..., 0], 6) | (_to_ufloat(rgb[..., 1], 6) << 11) | (_to_ufloat(rgb[..., 2], 5) << 22)


def unpack_b10g11r11(texels) -> np.ndarray:
    """(...) uint32 GS_PIX_B10G11R11_UFLOAT texels -> (..., 3) float32, exactly."""
    t = np.asarray(texels, np.uint32)
    return np.stack([_from_ufloat(t & 0x7FF, 6), _from_ufloat((t >> 11) & 0x7FF, 6), _from_ufloat(t >> 22, 5)], axis=-1)


def _srgb_oetf(x: np.ndarray) -> np.ndarray:
    with np.errstate(invalid="ignore"):
        return np.where(x <= 0.0031308, 12.92 * x, 1.055 * np.power(np.maximum(x, 0.0), 1.0 / 2.4) - 0.055)


def encode_srgb8(linear_rgba) -> np.ndarray:
    """(..., 4) float32 linear RGBA -> (..., 4) uint8 GS_PIX_R8G8B8A8_SRGB texels, rounded as the library's composite rounds
    them (include/gsplat_b200.h): RGB sRGB-encoded to the nearest code in the encoded domain, NaN and x <= 0 to 0, x >= 1 to 255;
    alpha clamped to [0, 1] and 255 a rounded to nearest, NaN to 0.  Evaluated in float64, whose error lies far below the
    distance of any float32 from a decision boundary."""
    with np.errstate(invalid="ignore"):   # signalling NaNs among arbitrary bit patterns
        x = np.asarray(linear_rgba, np.float32).astype(np.float64)
    bad = ~(x > 0)   # NaN and x <= 0
    xc = np.where(bad, 0.0, np.minimum(x, 1.0))
    rgb = np.floor(255.0 * _srgb_oetf(xc[..., :3]) + 0.5)
    a = np.floor(255.0 * xc[..., 3:] + 0.5)   # exact: a float32 times 255 fits in float64
    out = np.clip(np.concatenate([rgb, a], -1), 0, 255)
    out = np.where(bad, 0, np.where(x >= 1.0, 255, out))
    return out.astype(np.uint8)


_V8 = np.arange(256, dtype=np.float64) / 255.0
_SRGB8_DECODE = np.where(_V8 <= 0.04045, _V8 / 12.92, ((_V8 + 0.055) / 1.055) ** 2.4).astype(np.float32)


def decode_srgb8(texels) -> np.ndarray:
    """(..., 4) uint8 GS_PIX_R8G8B8A8_SRGB texels -> (..., 4) float32 linear RGBA: RGB through the float32 nearest the sRGB EOTF
    at c / 255, alpha the float32 nearest a / 255."""
    t = np.asarray(texels, np.uint8)
    return np.concatenate([_SRGB8_DECODE[t[..., :3]], (t[..., 3:].astype(np.float32) / np.float32(255.0)).astype(np.float32)], -1)


_EYE4 = np.eye(4, dtype=np.float32)
_inv_cache = {}


def _inverse_cached(m: np.ndarray) -> np.ndarray:
    """transform.worldToLocalMatrix: Unity keeps it alongside localToWorldMatrix; here it is cached per matrix value."""
    key = m.tobytes()
    hit = _inv_cache.get(key)
    if hit is None:
        if len(_inv_cache) > 64:
            _inv_cache.clear()
        hit = _inv_cache[key] = np.linalg.inv(m.astype(np.float64)).astype(np.float32)
    return hit


def decompose_trs(m):
    """Rotation (xyzw) and scale of a shear-free T*R*S matrix: what Transform.localRotation / localScale hold in Unity."""
    m = np.asarray(m, np.float64)[:3, :3]
    scale = np.linalg.norm(m, axis=0)
    if not (scale > 0).all():
        raise ValueError("degenerate transform: a basis vector has zero length")
    if np.linalg.det(m) < 0:
        scale[0] = -scale[0]          # a mirrored transform: Unity reports one negative scale component
    r = m / scale
    t = np.trace(r)
    if t > 0:
        s4 = np.sqrt(t + 1.0) * 2
        q = [(r[2, 1] - r[1, 2]) / s4, (r[0, 2] - r[2, 0]) / s4, (r[1, 0] - r[0, 1]) / s4, 0.25 * s4]
    else:
        i = int(np.argmax(np.diag(r)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s4 = np.sqrt(1.0 + r[i, i] - r[j, j] - r[k, k]) * 2
        q = [0.0, 0.0, 0.0, (r[k, j] - r[j, k]) / s4]
        q[i], q[j], q[k] = 0.25 * s4, (r[j, i] + r[i, j]) / s4, (r[k, i] + r[i, k]) / s4
    return np.asarray(q, np.float32), scale.astype(np.float32)


def bake_transform(records: np.ndarray, localToWorld, rotation=None, scale=None) -> np.ndarray:
    """In place: exported records (n x 62) moved into world space (gsa_bake_transform); rotation / scale default to the
    decomposition of the matrix."""
    if not (records.dtype == np.float32 and records.ndim == 2 and records.shape[1] == 62 and records.flags.c_contiguous):
        raise ValueError("records must be a C-contiguous (n, 62) float32 array")
    if rotation is None or scale is None:
        q, s = decompose_trs(localToWorld)
        rotation = q if rotation is None else rotation
        scale = s if scale is None else scale
    m = colmajor(np.asarray(localToWorld, np.float32))
    q = np.ascontiguousarray(rotation, np.float32)
    s = np.ascontiguousarray(scale, np.float32)
    if N.asset_lib().gsa_bake_transform(records.ctypes.data, records.shape[0], m.ctypes.data, q.ctypes.data, s.ctypes.data) != 0:
        raise ValueError("gsa_bake_transform failed (degenerate matrix?)")
    return records


def cutout_array(cutouts):
    """[(4x4 matrix = cutout worldToLocal * renderer localToWorld, type_and_flags)] -> GsCutout[] (R/GaussianCutout.cs:26-40)."""
    arr = (N.GsCutout * len(cutouts))()
    for i, (m, tf) in enumerate(cutouts):
        arr[i].mat[:] = colmajor(m).tolist()
        arr[i].type_and_flags = int(tf)
    return arr


def make_frame_params(cam: Camera, localToWorld=None, splat_scale=1.0, opacity_scale=1.0, sh_order=3, sh_only=False, cutouts=None,
                      deleted_bits=None, splat_count=0, selected_bits=None, scene_depth=None):
    """The uniforms C# binds in CalcViewData / SortPoints (R/GaussianSplatRenderer.cs:586-606,617-631).
    Returns (GsFrameParams, keepalive list for the borrowed host pointers)."""
    fp = N.GsFrameParams()
    o2w = _EYE4 if localToWorld is None else np.asarray(localToWorld, np.float32)
    w2o = _inverse_cached(o2w)
    for field, m in ((N.GsFrameParams.mat_object_to_world, o2w), (N.GsFrameParams.mat_world_to_object, w2o),
                     (N.GsFrameParams.mat_view, cam.worldToCameraMatrix), (N.GsFrameParams.mat_proj_gpu, cam.gpuProjectionMatrix(True))):
        cm = colmajor(m)   # 16 contiguous float32, UnityEngine.Matrix4x4 memory order
        C.memmove(C.addressof(fp) + field.offset, cm.ctypes.data, 64)
    fp.screen_w, fp.screen_h = float(cam.pixelWidth), float(cam.pixelHeight)
    pos = np.asarray(cam.position, np.float32)
    fp.cam_pos_world[0], fp.cam_pos_world[1], fp.cam_pos_world[2] = float(pos[0]), float(pos[1]), float(pos[2])
    fp.splat_scale, fp.opacity_scale = float(splat_scale), float(opacity_scale)
    fp.sh_order, fp.sh_only = int(sh_order), 1 if sh_only else 0
    keep = []
    if cutouts:
        arr = cutout_array(cutouts)
        fp.cutouts, fp.cutout_count = C.cast(arr, C.c_void_p), len(cutouts)
        keep.append(arr)
    if deleted_bits is not None:
        bits = np.ascontiguousarray(deleted_bits, np.uint32)
        assert bits.size >= (splat_count + 31) // 32
        fp.deleted_bits = bits.ctypes.data
        keep.append(bits)
    if selected_bits is not None:
        bits = np.ascontiguousarray(selected_bits, np.uint32)
        assert bits.size >= (splat_count + 31) // 32
        fp.selected_bits = bits.ctypes.data
        keep.append(bits)
    if scene_depth is not None:    # (H, W) float32: numpy host array, torch CUDA tensor or CudaArrayDepth
        if isinstance(scene_depth, CudaArrayDepth):
            if scene_depth.shape != (cam.pixelHeight, cam.pixelWidth):
                raise ValueError("the depth CUDA array is %dx%d, the screen %dx%d" % (scene_depth.width, scene_depth.height,
                                                                                   cam.pixelWidth, cam.pixelHeight))
            if scene_depth._layer_desc is None:
                fp.scene_depth, fp.scene_depth_on_device = scene_depth.handle, N.GS_MEM_ARRAY
            else:
                fp.scene_depth, fp.scene_depth_on_device = C.addressof(scene_depth._layer_desc), scene_depth.memory
            depth = scene_depth   # keeps its layer / rectangle descriptor alive with the frame params
        elif isinstance(scene_depth, np.ndarray):
            depth = np.ascontiguousarray(scene_depth, np.float32)
            assert depth.shape == (cam.pixelHeight, cam.pixelWidth)
            fp.scene_depth, fp.scene_depth_on_device = depth.ctypes.data, 0
        else:
            depth = scene_depth.contiguous()
            assert tuple(depth.shape) == (cam.pixelHeight, cam.pixelWidth) and depth.element_size() == 4
            fp.scene_depth, fp.scene_depth_on_device = depth.data_ptr(), 1 if depth.is_cuda else 0
        keep.append(depth)
    return fp, keep


class GaussianSplatRenderer:
    def __init__(self, asset: GaussianSplatAsset, context: Optional[GaussianSplatContext] = None):
        self._init_state(asset, context)
        d = asset.desc()
        h = C.c_void_p()
        N.check(self.context.handle, self._lib.gs_asset_upload(self.context.handle, C.byref(d), C.byref(h)))
        self._asset = h

    @classmethod
    def from_device_asset(cls, asset: GaussianSplatAsset, handle: C.c_void_p, context: GaussianSplatContext):
        """A renderer on a GsAsset that is already in HBM (gs_pack_asset's asset_out); it takes ownership of `handle`.
        `asset` is the host copy of the same blobs."""
        self = cls.__new__(cls)
        self._init_state(asset, context)
        self._asset = handle
        return self

    def Instance(self) -> "GaussianSplatRenderer":
        """A further renderer of this renderer's asset on its context (gs_asset_instance): the blobs in HBM are shared, not
        uploaded again; the new renderer has its own draw order, view data and knobs (at their defaults) and its own Dispose().
        It behaves exactly like GaussianSplatRenderer(self.m_Asset, self.context), and outlives this renderer if need be."""
        h = C.c_void_p()
        N.check(self.context.handle, self._lib.gs_asset_instance(self._asset, C.byref(h)))
        return GaussianSplatRenderer.from_device_asset(self.m_Asset, h, self.context)

    def _init_state(self, asset: GaussianSplatAsset, context: Optional[GaussianSplatContext]):
        self.context = context or GaussianSplatContext(0)
        self._lib = self.context._lib
        self.m_Asset = asset
        # serialized knobs, R/GaussianSplatRenderer.cs:225-251
        self.m_SplatScale = 1.0
        self.m_OpacityScale = 1.0
        self.m_SHOrder = 3
        self.m_SHOnly = False
        self.m_SortNthFrame = 1
        self.m_RenderOrder = 0       # R/GaussianSplatRenderer.cs:236: higher values draw first
        self.m_FrameCounter = 0
        self.localToWorldMatrix = np.eye(4, dtype=np.float32)  # transform of the GameObject
        self.localRotation = None    # xyzw / None = derived from the matrix (tr.localRotation, tr.localScale; export only)
        self.localScale = None
        self.m_Cutouts = []          # list of (4x4 matrix, type_and_flags)
        self.m_DeletedBits = None    # np.uint32[ceil(N/32)] or None
        self.m_SelectedBits = None   # np.uint32[ceil(N/32)] or None (m_GpuEditSelected, R/GaussianSplatRenderer.cs:496)
        self.sceneDepth = None       # (H, W) float32 camera depth buffer (reversed Z) the splats are depth-tested against (numpy,
                                     # torch CUDA tensor or CudaArrayDepth), or None
        self.blend_mode = N.GS_BLEND_FP16_ROP
        self.partition = (0, 0, 1)   # index, count, band_rows
        self.band_packed = False
        self.rows = (0, 0)           # contiguous partition: 16-pixel rows [begin, end) (GsRenderOptions.row_begin/row_end)
        self.load_rt = False         # GS_FLAG_LOAD_RT: blend under what the target already holds (several renderers, one RT)
        self.async_readback = False  # host render targets are filled asynchronously (pinned memory; context.sync() completes them)
        self._asset = None
        self._keep = None

    # -- resources ---------------------------------------------------------------------------
    @property
    def splatCount(self) -> int:
        return self.m_Asset.splatCount

    def Dispose(self):
        if self._asset:
            self._lib.gs_asset_destroy(self._asset)
            self._asset = None

    def __del__(self):
        try:
            self.Dispose()
        except Exception:
            pass

    def ResetOrder(self):
        N.check(self.context.handle, self._lib.gs_asset_reset_order(self._asset))

    # -- uniforms ------------------------------------------------------------------------------
    def frame_params(self, cam: Camera) -> N.GsFrameParams:
        fp, self._keep = make_frame_params(cam, self.localToWorldMatrix, self.m_SplatScale, self.m_OpacityScale, self.m_SHOrder,
                                           self.m_SHOnly, self.m_Cutouts, self.m_DeletedBits, self.splatCount, self.m_SelectedBits,
                                           self.sceneDepth)
        return fp

    def _options(self) -> N.GsRenderOptions:
        o = N.GsRenderOptions()
        o.blend_mode = self.blend_mode
        o.partition_index, o.partition_count, o.band_rows = self.partition
        o.band_packed = 1 if self.band_packed else 0
        o.flags = (N.GS_FLAG_ASYNC_READBACK if self.async_readback else 0) | (N.GS_FLAG_LOAD_RT if self.load_rt else 0)
        o.row_begin, o.row_end = self.rows
        return o

    # -- the hot path ----------------------------------------------------------------------------
    def SortPoints(self, cam: Camera):
        fp = self.frame_params(cam)
        N.check(self.context.handle, self._lib.gs_sort(self.context.handle, self._asset, C.byref(fp)))

    def CalcViewData(self, cam: Camera):
        fp = self.frame_params(cam)
        N.check(self.context.handle, self._lib.gs_calc_view(self.context.handle, self._asset, C.byref(fp)))

    def DrawSplats(self, cam: Camera, rt):
        fp, opt = self.frame_params(cam), self._options()
        im = _image(rt, cam.pixelWidth, rt.shape[0])
        N.check(self.context.handle, self._lib.gs_render(self.context.handle, self._asset, C.byref(fp), C.byref(opt), C.byref(im)))

    def Composite(self, rt, camera_target):
        h, w = rt.shape[0], rt.shape[1]
        a, b = _image(rt, w, h), _image(camera_target, w, h)
        N.check(self.context.handle, self._lib.gs_composite(self.context.handle, C.byref(a), C.byref(b)))

    def SortAndRenderSplats(self, cam: Camera, rt=None, camera_target=None, fp=None):
        """One frame: sort every m_SortNthFrame-th call (:120-121), view-calc, draw, optional composite.
        fp: uniforms built ahead with frame_params(cam) (a host that knows its camera path); default: built here."""
        do_sort = 1 if (self.m_FrameCounter % max(1, int(self.m_SortNthFrame)) == 0) else 0
        self.m_FrameCounter += 1
        fp, opt = (self.frame_params(cam) if fp is None else fp), self._options()
        a = _image(rt, cam.pixelWidth, rt.shape[0]) if rt is not None else None
        b = _image(camera_target, cam.pixelWidth, cam.pixelHeight) if camera_target is not None else None
        N.check(self.context.handle,
                self._lib.gs_frame(self.context.handle, self._asset, C.byref(fp), C.byref(opt), do_sort,
                                   C.byref(a) if a is not None else None, C.byref(b) if b is not None else None))

    # -- test hooks --------------------------------------------------------------------------------
    def readback_order(self) -> np.ndarray:
        out = np.empty(self.splatCount, np.uint32)
        N.check(self.context.handle, self._lib.gs_readback_order(self._asset, out.ctypes.data))
        return out

    def readback_keys(self) -> np.ndarray:
        out = np.empty(self.splatCount, np.uint32)
        N.check(self.context.handle, self._lib.gs_readback_keys(self._asset, out.ctypes.data))
        return out

    def readback_view(self) -> np.ndarray:
        out = np.empty((self.splatCount, 10), np.uint32)
        N.check(self.context.handle, self._lib.gs_readback_view(self._asset, out.ctypes.data))
        return out

    # ---- export (R/GaussianSplatRenderer.cs:936-958 EditExportData, E/GaussianSplatRendererEditor.cs:394-445 ExportPlyFile) ----
    def EditExportData(self, bakeTransform: bool = False) -> np.ndarray:
        """CSExportData on the GPU: (n, 62) float32 raw .ply attribute records; nor = 1 marks splats the cutouts remove."""
        out = np.empty((self.splatCount, 62), np.float32)
        arr = cutout_array(self.m_Cutouts) if self.m_Cutouts else None
        count = len(self.m_Cutouts) if self.m_Cutouts else 0
        N.check(self.context.handle, self._lib.gs_export_splats(self.context.handle, self._asset, arr, count, 0, out.ctypes.data))
        if bakeTransform:   # the _ExportTransformFlags branch of CSExportData, run as a host pass (include/gsplat_asset.h)
            bake_transform(out, self.localToWorldMatrix, self.localRotation, self.localScale)
        return out

    def ExportPlyFile(self, path: str, bakeTransform: bool = False) -> int:
        """Writes the .ply the reference's "Export PLY" writes: alive (not deleted, not cut) splats only.  Returns their count."""
        from .asset import write_ply
        return write_ply(path, self.EditExportData(bakeTransform), self.m_DeletedBits)

    def upload_order(self, order: np.ndarray):
        order = np.ascontiguousarray(order, np.uint32)
        assert order.size == self.splatCount
        N.check(self.context.handle, self._lib.gs_upload_order(self._asset, order.ctypes.data))


def GatherSplatsForCamera(renderers, cam: Camera):
    """GaussianSplatRenderSystem.GatherSplatsForCamera (R/GaussianSplatRenderer.cs:73-105): the active splat objects in draw
    order -- m_RenderOrder descending, then camera-space depth of the object's transform position ascending."""
    w2c = cam.worldToCameraMatrix.astype(np.float64)

    def depth(r):
        m = r.localToWorldMatrix   # None (a group object's default): identity
        p = np.asarray(_EYE4 if m is None else m, np.float64)[:3, 3]
        return -float((w2c @ np.r_[p, 1.0])[2])     # camTr.InverseTransformPoint(pos).z: +z forward (the view matrix looks down -z)
    return sorted(renderers, key=lambda r: (-int(r.m_RenderOrder), depth(r)))


def draws_in_one_call(active) -> bool:
    """Whether gs_frame_objects can draw these renderers: one context, whole-screen options (no partition, row range or band
    packing) and one blend mode and read-back mode.  Otherwise SortAndRenderSplatsMulti draws them one gs_frame at a time."""
    r0 = active[0]
    return all(r.context is r0.context and r.blend_mode == r0.blend_mode and bool(r.async_readback) == bool(r0.async_readback)
               and int(r.partition[1]) <= 1 and int(r.partition[0]) == 0 and tuple(r.rows) == (0, 0) and not r.band_packed
               for r in active)


def SortAndRenderSplatsMulti(renderers, cam: Camera, rt, camera_target=None):
    """GaussianSplatRenderSystem.SortAndRenderSplats (R/GaussianSplatRenderer.cs:108-169) for several splat objects of one
    camera: ONE render target, cleared once (:196), every object blended under what the earlier ones left, then the composite
    onto camera_target (when given).  One gs_frame_objects call when draws_in_one_call(active); else one gs_frame per object
    (GS_FLAG_LOAD_RT from the second on) and gs_composite.  Returns the active renderers in draw order."""
    active = GatherSplatsForCamera(renderers, cam)
    if not active:
        return active
    if draws_in_one_call(active):
        _frame_objects(active, cam, rt, camera_target)
        return active
    if rt is None:
        raise ValueError("drawing the objects one gs_frame at a time needs a render target")
    for i, r in enumerate(active):
        keep = r.load_rt
        r.load_rt = i > 0
        try:
            r.SortAndRenderSplats(cam, rt=rt)
        finally:
            r.load_rt = keep
    if camera_target is not None:
        active[0].Composite(rt, camera_target)
    return active


def cameras_in_one_call(actives) -> bool:
    """Whether gs_frame_cameras can draw these cameras (each a non-empty list of active renderers in draw order): every list
    passes draws_in_one_call, all on one context with one blend mode, and nobody asks for asynchronous read-back."""
    r0 = actives[0][0]
    return all(draws_in_one_call(a) and a[0].context is r0.context and a[0].blend_mode == r0.blend_mode and not a[0].async_readback
               for a in actives)


def SortAndRenderCameras(renderers, cams, rts, camera_targets=None, via_event=False):
    """The camera loop of GaussianSplatRenderSystem (R/GaussianSplatRenderer.cs:187-211): SortAndRenderSplatsMulti for each
    camera in turn -- GatherSplatsForCamera per camera, each renderer's m_FrameCounter advanced once per camera that draws it
    -- in one gs_frame_cameras call when cameras_in_one_call holds for the cameras that draw something, else camera by camera.
    rts[c] / camera_targets[c] may be None (not both for a camera that draws).  Returns each camera's active renderers.
    via_event: the one call goes through the render-thread event GS_UNITY_EVENT_FRAME_CAMERAS, run on this thread, instead of
    gs_frame_cameras (what the tests compare the two with); the cameras must then pass cameras_in_one_call."""
    camera_targets = camera_targets if camera_targets is not None else [None] * len(cams)
    actives = [GatherSplatsForCamera(renderers, cam) for cam in cams]
    drawn = [c for c, a in enumerate(actives) if a]
    if not drawn:
        return actives
    one_call = cameras_in_one_call([actives[c] for c in drawn])
    if via_event and not one_call:
        raise ValueError("the render-thread event draws the cameras in one call: they must pass cameras_in_one_call")
    if one_call:
        (_frame_cameras_event if via_event else _frame_cameras)([actives[c] for c in drawn], [cams[c] for c in drawn],
                                                                [rts[c] for c in drawn], [camera_targets[c] for c in drawn])
        return actives
    for c in drawn:
        SortAndRenderSplatsMulti(renderers, cams[c], rts[c], camera_targets[c])
    return actives


def _frame_cameras(actives, cams, rts, camera_targets):
    ctx, counts, assets, fps, do_sort, opt, images, keep = _camera_call(actives, cams, rts, camera_targets)
    a = (C.POINTER(N.GsImage) * len(cams))(*[C.pointer(x) if x is not None else C.POINTER(N.GsImage)() for x, _ in images])
    b = (C.POINTER(N.GsImage) * len(cams))(*[C.pointer(y) if y is not None else C.POINTER(N.GsImage)() for _, y in images])
    N.check(ctx.handle, ctx._lib.gs_frame_cameras(ctx.handle, len(cams), counts, assets, fps, do_sort, C.byref(opt), a, b))
    del keep


def _frame_cameras_event(actives, cams, rts, camera_targets):
    """_frame_cameras through the payload a CommandBuffer would carry (GsUnityFrameCamerasEvent, images by value)."""
    ctx, counts, assets, fps, do_sort, opt, images, keep = _camera_call(actives, cams, rts, camera_targets)
    a, b = N.image_array([x for x, _ in images]), N.image_array([y for _, y in images])
    ev = N.GsUnityFrameCamerasEvent(ctx=ctx.handle.value, camera_count=len(cams), object_counts=C.addressof(counts),
                                    assets=C.addressof(assets), fps=C.addressof(fps), do_sort=C.addressof(do_sort), options=opt,
                                    rts=C.addressof(a), camera_targets=C.addressof(b), status=N.GS_ERR_NOT_READY)
    N.check(ctx.handle, N.unity_event(N.GS_UNITY_EVENT_FRAME_CAMERAS, ev))
    del keep


def _camera_call(actives, cams, rts, camera_targets):
    """gs_frame_cameras' arguments for the cameras' active renderers: (context, object counts, assets, frame parameters,
    do_sort, options, [(rt image, camera target image)], keep), keep holding what they point to.  Each renderer's frame counter
    advances once per camera."""
    n = sum(len(a) for a in actives)
    fps = (N.GsFrameParams * n)()
    assets = (C.c_void_p * n)()
    do_sort = (C.c_int32 * n)()
    counts = (C.c_uint32 * len(cams))(*[len(a) for a in actives])
    keep = []
    i = 0
    for active, cam in zip(actives, cams):
        for r in active:
            do_sort[i] = 1 if (r.m_FrameCounter % max(1, int(r.m_SortNthFrame)) == 0) else 0
            r.m_FrameCounter += 1
            fps[i], k = make_frame_params(cam, r.localToWorldMatrix, r.m_SplatScale, r.m_OpacityScale, r.m_SHOrder, r.m_SHOnly,
                                          r.m_Cutouts, r.m_DeletedBits, r.splatCount, r.m_SelectedBits, r.sceneDepth)
            keep.append(k)
            assets[i] = r._asset.value if isinstance(r._asset, C.c_void_p) else r._asset
            i += 1
    opt = actives[0][0]._options()
    opt.flags &= ~N.GS_FLAG_LOAD_RT
    images = [(_image(rt, cam.pixelWidth, cam.pixelHeight) if rt is not None else None,
               _image(tg, cam.pixelWidth, cam.pixelHeight) if tg is not None else None) for cam, rt, tg in zip(cams, rts, camera_targets)]
    return actives[0][0].context, counts, assets, fps, do_sort, opt, images, keep


def _frame_objects(active, cam: Camera, rt, camera_target):
    k = len(active)
    fps = (N.GsFrameParams * k)()
    assets = (C.c_void_p * k)()
    do_sort = (C.c_int32 * k)()
    for i, r in enumerate(active):
        do_sort[i] = 1 if (r.m_FrameCounter % max(1, int(r.m_SortNthFrame)) == 0) else 0
        r.m_FrameCounter += 1
        fps[i] = r.frame_params(cam)     # r._keep holds the host buffers it points to
        assets[i] = r._asset.value if isinstance(r._asset, C.c_void_p) else r._asset
    opt = active[0]._options()
    opt.flags &= ~N.GS_FLAG_LOAD_RT
    a = _image(rt, cam.pixelWidth, cam.pixelHeight) if rt is not None else None
    b = _image(camera_target, cam.pixelWidth, cam.pixelHeight) if camera_target is not None else None
    ctx = active[0].context
    N.check(ctx.handle, ctx._lib.gs_frame_objects(ctx.handle, k, assets, fps, do_sort, C.byref(opt), C.byref(a) if a is not None else None,
                                                  C.byref(b) if b is not None else None))
