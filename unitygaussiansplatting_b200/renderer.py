"""Host-side mirror of GaussianSplatRenderer (package/Runtime/GaussianSplatRenderer.cs) on top of
the C ABI.  Same member names, argument meaning and order of operations as the C# component for
the hot path; everything it does is a call into libgsplat_b200.so (there is no CPU path here).

  C#                                          here
  ------------------------------------------  ------------------------------------------------
  OnEnable -> CreateResourcesForAsset (:373)   GaussianSplatRenderer(asset)  -> gs_asset_upload
  SortPoints(cmd, cam, matrix)        (:612)   SortPoints(cam)               -> gs_sort
  CalcViewData(cmb, cam)              (:579)   CalcViewData(cam)             -> gs_calc_view
  cmb.DrawProcedural(matSplats)       (:165)   DrawSplats(cam, rt)           -> gs_render
  composite DrawProcedural            (:206)   Composite(rt, target)         -> gs_composite
  SortAndRenderSplats(cam, cmb)       (:108)   SortAndRenderSplats(cam, ...) -> gs_frame
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


def _image(arr, width: int, height: int) -> N.GsImage:
    """numpy (host) array or torch CUDA tensor of shape (H, W, 4), float16/float32 -> GsImage."""
    im = N.GsImage()
    im.width, im.height = width, height
    if isinstance(arr, np.ndarray):
        if arr.shape != (height, width, 4) or not arr.flags.c_contiguous:
            raise ValueError("image must be C-contiguous (H, W, 4)")
        if arr.dtype == np.float16:
            im.format = N.GS_PIX_RGBA16F
        elif arr.dtype == np.float32:
            im.format = N.GS_PIX_RGBA32F
        else:
            raise ValueError("image dtype must be float16 or float32")
        im.data, im.memory = arr.ctypes.data, N.GS_MEM_HOST
        im.row_pitch_bytes = arr.strides[0]
        return im
    # torch tensor (duck-typed so torch stays optional)
    if tuple(arr.shape) != (height, width, 4) or not arr.is_contiguous():
        raise ValueError("image must be contiguous (H, W, 4)")
    es = arr.element_size()
    im.format = N.GS_PIX_RGBA16F if es == 2 else N.GS_PIX_RGBA32F
    im.data = arr.data_ptr()
    im.memory = N.GS_MEM_DEVICE if arr.is_cuda else N.GS_MEM_HOST
    im.row_pitch_bytes = width * 4 * es
    return im


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
    if scene_depth is not None:    # (H, W) float32: numpy host array or torch CUDA tensor
        if isinstance(scene_depth, np.ndarray):
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
        self.sceneDepth = None       # (H, W) float32 camera depth buffer (reversed Z) the splats are depth-tested against, or None
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
        p = np.asarray(r.localToWorldMatrix, np.float64)[:3, 3]
        return -float((w2c @ np.r_[p, 1.0])[2])     # camTr.InverseTransformPoint(pos).z: +z forward (the view matrix looks down -z)
    return sorted(renderers, key=lambda r: (-int(r.m_RenderOrder), depth(r)))


def SortAndRenderSplatsMulti(renderers, cam: Camera, rt):
    """GaussianSplatRenderSystem.SortAndRenderSplats (R/GaussianSplatRenderer.cs:108-169) for several splat objects of one
    camera: ONE render target, cleared once (:196), every object blended under what the earlier ones left
    (GS_FLAG_LOAD_RT from the second object on).  All renderers must live on one context."""
    active = GatherSplatsForCamera(renderers, cam)
    for i, r in enumerate(active):
        keep = r.load_rt
        r.load_rt = i > 0
        try:
            r.SortAndRenderSplats(cam, rt=rt)
        finally:
            r.load_rt = keep
    return active
