"""Several GPUs of one box (SURVEY.md 8e; the reference is single-GPU).

Two schemes live here, the second only as the baseline the first is measured against:

* GaussianSplatGroup (below, second half) -- the product path: gs_group_* of the C ABI.  The depth sort is sharded by key range,
  view-calc / binning / compositing by contiguous ranges of 16-pixel rows, the exchanges (NVLink peer stores or NCCL) are
  made by the library itself; order and pixels are bit-identical to one GPU.  Python only holds the handles.
* BandPartition / render_partitioned (first half) -- round 1's scheme: every rank sorts and view-calcs the whole asset
  redundantly and composites only its own interleaved bands of 64-pixel bin rows, band-packed into its slice of an
  all-gather buffer; ONE torch.distributed all-gather moves the bands and gs_unshuffle_bands assembles the image.  The
  partition arithmetic is mirrored by the device code in csrc/gs_raster.cu (struct Partition) and tested against it.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

from . import _native as N

TILE = 64   # band granularity in pixels: the library bins (and partitions) in 64-pixel rows (csrc/gs_common.cuh kBin)


@dataclass
class BandPartition:
    height: int
    count: int
    index: int
    band_rows: int = 1   # tile rows per band

    @property
    def tiles_y(self) -> int:
        return (self.height + TILE - 1) // TILE

    def owner(self, tile_row: int) -> int:
        return 0 if self.count <= 1 else (tile_row // self.band_rows) % self.count

    def own_rows_below(self, y: int, index=None) -> int:
        """number of tile rows in [0, y) owned by partition `index`"""
        index = self.index if index is None else index
        if self.count <= 1:
            return y
        cyc = self.band_rows * self.count
        q, r = divmod(y, cyc)
        lo = index * self.band_rows
        return q * self.band_rows + min(max(r - lo, 0), self.band_rows)

    def own_tile_rows(self, index=None) -> int:
        return self.own_rows_below(self.tiles_y, index)

    def kth_own_row(self, k: int, index=None) -> int:
        index = self.index if index is None else index
        if self.count <= 1:
            return k
        return ((k // self.band_rows) * self.count + index) * self.band_rows + (k % self.band_rows)

    @property
    def rows_per_partition(self) -> int:
        """pixel rows of every rank's slice in the gather buffer (max over ranks, so slices are equal-sized)"""
        return TILE * max(self.own_tile_rows(i) for i in range(max(1, self.count)))

    def options(self):
        return (self.index, self.count if self.count > 1 else 0, self.band_rows)

    def source_row(self, y: int):
        """image row y -> (partition, row inside that partition's band-packed buffer)"""
        ty = y // TILE
        o = self.owner(ty)
        return o, self.own_rows_below(ty, o) * TILE + (y - ty * TILE)


def alloc_gather(part: BandPartition, width: int, device, dtype=None):
    import torch
    return torch.zeros((max(1, part.count), part.rows_per_partition, width, 4), dtype=dtype or torch.float16, device=device)


def render_partitioned(renderer, cam, part: BandPartition, gathered, out_image):
    """One frame of the round-1 interleaved-band scheme: replicated sort + view-calc, own bands composited band-packed,
    one all-gather through torch.distributed, unshuffle.  Kept as the simple baseline the group path (GaussianSplatGroup,
    gs_group_frame: NCCL inside the library) is measured against.  The library works on the context's stream and NCCL on
    torch's current stream, so the three steps are ordered explicitly with events."""
    import torch
    import torch.distributed as dist
    own_px = part.own_tile_rows() * TILE
    mine = gathered[part.index]
    renderer.partition = part.options()
    renderer.band_packed = True
    lib_stream = torch.cuda.ExternalStream(renderer.context.stream)
    cur = torch.cuda.current_stream()
    if lib_stream.cuda_stream != cur.cuda_stream:
        lib_stream.wait_stream(cur)          # whoever produced / still reads `gathered` on torch's stream goes first
    if own_px:
        renderer.SortAndRenderSplats(cam, rt=mine[:own_px])
    else:   # more partitions than 64-pixel rows: nothing to composite here, but keep the draw order current
        renderer.SortPoints(cam)
    if part.count > 1:
        if lib_stream.cuda_stream != cur.cuda_stream:
            cur.wait_stream(lib_stream)      # the collective reads our slice only after the compositor wrote it
        dist.all_gather_into_tensor(gathered.view(-1), mine.reshape(-1))   # in place: input is our slice of the output
        if lib_stream.cuda_stream != cur.cuda_stream:
            lib_stream.wait_stream(cur)      # ... and the unshuffle reads the gathered bands only after the collective
    unshuffle(renderer.context, gathered, part, out_image)


def unshuffle(context, gathered, part: BandPartition, out_image):
    from .renderer import _image
    h, w = out_image.shape[0], out_image.shape[1]
    im = _image(out_image, w, h)
    fmt = N.GS_PIX_RGBA16F if gathered.element_size() == 2 else N.GS_PIX_RGBA32F
    N.check(context.handle, N.native().gs_unshuffle_bands(context.handle, C.c_void_p(gathered.data_ptr()), max(1, part.count), part.band_rows,
                                                          part.rows_per_partition, fmt, C.byref(im)))


# ---------------------------------------------------------------------------------------------------------------------
# The group path (include/gsplat_b200.h "several GPUs"): key-range-sharded sort + row-range-sharded view-calc / binning /
# compositing; the exchanges (peer stores over NVLink, or NCCL) are made by the library on its own streams.  Python only holds
# the handles.
# ---------------------------------------------------------------------------------------------------------------------
def group_unique_id() -> bytes:
    """Rank 0 creates the id; every other process needs the same 128 bytes (send them over any host channel)."""
    buf = C.create_string_buffer(N.GS_GROUP_ID_BYTES)
    N.check(None, N.native().gs_group_unique_id(buf))
    return buf.raw


def share_unique_id_torch(rank: int) -> bytes:
    """The id exchange through an existing torch.distributed process group (plumbing only)."""
    import torch
    import torch.distributed as dist
    obj = [group_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(obj, src=0)
    return obj[0]


class GaussianSplatGroup:
    """Mirror of GaussianSplatRenderer for a group of GPUs: same knobs, SortAndRenderSplats drives gs_group_frame."""

    def __init__(self, handle, asset, lib):
        from .renderer import GaussianSplatContext
        self._lib = lib
        self.handle = handle
        self.m_Asset = asset
        self.size = int(lib.gs_group_size(handle))
        self.local_count = int(lib.gs_group_local_count(handle))
        self.contexts = [GaussianSplatContext.from_handle(lib.gs_group_context(handle, i)) for i in range(self.local_count)]
        self._assets = _upload(lib, handle, asset, self.local_count)
        _init_knobs(self)
        self.blend_mode = N.GS_BLEND_FP16_ROP
        self.async_readback = False  # host images are filled asynchronously (pinned memory; sync() completes them)
        self._objects = []           # further splat objects (add_object), drawn with SortAndRenderSplatsMulti

    @classmethod
    def join(cls, asset, context, rank: int, world: int, unique_id: bytes):
        """One process per GPU: `context` is this process's GaussianSplatContext."""
        lib = N.native()
        h = C.c_void_p()
        N.check(context.handle, lib.gs_group_join(context.handle, world, rank, unique_id, C.byref(h)))
        grp = cls(h, asset, lib)
        grp._owner_ctx = context   # keep the caller's context alive as long as the group
        return grp

    @classmethod
    def create(cls, asset, devices, emulate: bool = False):
        """One process driving len(devices) GPUs; emulate=True lets indices repeat (contexts on one device, copies as exchange)."""
        lib = N.native()
        h = C.c_void_p()
        arr = (C.c_int * len(devices))(*devices)
        N.check(None, lib.gs_group_create(arr, len(devices), N.GS_GROUP_EMULATE if emulate else 0, C.byref(h)))
        return cls(h, asset, lib)

    @property
    def splatCount(self) -> int:
        return self.m_Asset.splatCount

    def frame_params(self, cam):
        fp, self._keep = _frame_params(self, cam)
        return fp

    def add_object(self, asset) -> "GaussianSplatGroupObject":
        """Another splat object on the group: `asset` is uploaded to every member (gs_group_asset_upload).  The returned object
        carries the renderer's knobs; draw it with SortAndRenderSplatsMulti.  The group itself stays usable as an object."""
        o = GaussianSplatGroupObject(self, asset)
        self._objects.append(o)
        return o

    def add_instance(self, source) -> "GaussianSplatGroupObject":
        """Another splat object drawing the asset of `source` (this group or one of its objects): on every member an instance of
        source's asset (gs_asset_instance), which shares its blobs in HBM and keeps its own draw order.  Behaves like
        add_object(source.m_Asset); freed by the group's close()."""
        if source._group() is not self:
            raise ValueError("the source belongs to another group")
        o = GaussianSplatGroupObject(self, source.m_Asset, share=source)
        self._objects.append(o)
        return o

    def SortAndRenderSplats(self, cam, rts=None, fp=None):
        """rts: one image per LOCAL member (numpy host array, torch CUDA tensor, CudaArrayImage, or None); each receives the
        whole frame."""
        do_sort = 1 if (self.m_FrameCounter % max(1, int(self.m_SortNthFrame)) == 0) else 0
        self.m_FrameCounter += 1
        if fp is None:
            fp = self.frame_params(cam)
        opt = self._options()
        ims = []
        ptrs = self._images(rts, cam, ims)
        N.check(self.contexts[0].handle, self._lib.gs_group_frame(self.handle, self._assets, C.byref(fp), C.byref(opt), do_sort, ptrs))

    def SortAndRenderSplatsMulti(self, objects, cam, rts=None, camera_targets=None, via_event=False):
        """One camera's frame with several splat objects (the group itself and / or add_object's objects): ordered by
        GatherSplatsForCamera, the first drawn into a cleared target and each later one under it, one row exchange, then the
        composite onto every given camera target (gs_group_frame_objects).  rts / camera_targets: one image per LOCAL member
        or None, as in SortAndRenderSplats.  Returns the objects in the order they were drawn.  With no objects nothing is
        drawn or composited, as OnPreCullCamera returns early when the camera has no active splat object.
        via_event: the call goes through the render-thread event GS_UNITY_EVENT_GROUP_FRAME_OBJECTS, run on this thread (what
        the tests compare the two with)."""
        from .renderer import GatherSplatsForCamera
        objects = list(objects)
        for k, o in enumerate(objects):   # checked before any object's frame counter moves
            if o._group() is not self:
                raise ValueError("object %d belongs to another group" % k)
        if len(set(map(id, objects))) != len(objects):
            raise ValueError("an object is listed twice")
        if not objects:
            return []
        active = GatherSplatsForCamera(objects, cam)
        K, L = len(active), self.local_count
        assets = (C.c_void_p * (K * L))()
        fps = (N.GsFrameParams * K)()
        do_sort = (C.c_int32 * K)()
        keep = []
        for k, o in enumerate(active):
            for i in range(L):
                assets[k * L + i] = o._assets[i]
            fps[k], kp = _frame_params(o, cam)
            keep.append(kp)
            do_sort[k] = 1 if (o.m_FrameCounter % max(1, int(o.m_SortNthFrame)) == 0) else 0
        opt = self._options()
        ims = []
        ptrs, cptrs = self._images(rts, cam, ims), self._images(camera_targets, cam, ims)
        for o in active:   # the uniforms and images were accepted: now the frame counts (:120-121)
            o.m_FrameCounter += 1
        if via_event:
            a, b = (N.image_array([p.contents if p else None for p in pp]) for pp in (ptrs, cptrs))
            ev = N.GsUnityGroupFrameObjectsEvent(group=self.handle.value, object_count=K, assets=C.addressof(assets), fps=C.addressof(fps),
                                                 do_sort=C.addressof(do_sort), options=opt, rts=C.addressof(a), camera_targets=C.addressof(b),
                                                 status=N.GS_ERR_NOT_READY)
            N.check(self.contexts[0].handle, N.unity_event(N.GS_UNITY_EVENT_GROUP_FRAME_OBJECTS, ev))
        else:
            N.check(self.contexts[0].handle, self._lib.gs_group_frame_objects(self.handle, K, assets, fps, do_sort, C.byref(opt), ptrs, cptrs))
        return active

    def _group(self):
        return self

    def _options(self) -> N.GsRenderOptions:
        opt = N.GsRenderOptions()
        opt.blend_mode = self.blend_mode
        opt.flags = N.GS_FLAG_ASYNC_READBACK if self.async_readback else 0
        return opt

    def _images(self, images, cam, keep):
        from .renderer import _image
        ptrs = (C.POINTER(N.GsImage) * self.local_count)()
        if images is not None:
            if not isinstance(images, (list, tuple)):
                images = [images]
            for i, a in enumerate(images):
                if a is not None:
                    im = _image(a, cam.pixelWidth, cam.pixelHeight)
                    keep.append(im)
                    ptrs[i] = C.pointer(im)
        return ptrs

    def sync(self, via_event=False):
        """gs_group_sync; via_event: through the render-thread event GS_UNITY_EVENT_GROUP_SYNC, run on this thread."""
        if via_event:
            ev = N.GsUnityGroupSyncEvent(group=self.handle.value, status=N.GS_ERR_NOT_READY)
            N.check(self.contexts[0].handle, N.unity_event(N.GS_UNITY_EVENT_GROUP_SYNC, ev))
        else:
            N.check(self.contexts[0].handle, self._lib.gs_group_sync(self.handle))

    def row_costs(self, rows: int):
        """gs_group_row_costs: the per-row costs the last call measured, summed over its objects (what the row split two calls
        later is balanced on)."""
        import numpy as np
        out = np.zeros(rows, np.uint32)
        N.check(self.contexts[0].handle, self._lib.gs_group_row_costs(self.handle, out.ctypes.data, rows))
        return out

    def stats(self) -> N.GsGroupStats:
        st = N.GsGroupStats()
        N.check(self.contexts[0].handle, self._lib.gs_group_get_stats(self.handle, C.byref(st)))
        return st

    def readback_order(self, local: int = 0):
        import numpy as np
        out = np.empty(self.splatCount, np.uint32)
        N.check(self.contexts[local].handle, self._lib.gs_readback_order(self._assets[local], out.ctypes.data))
        return out

    def close(self):
        if self.handle:
            def free_assets():
                for holder in [self] + self._objects:
                    for i in range(self.local_count):
                        if holder._assets[i]:
                            self._lib.gs_asset_destroy(holder._assets[i])
                            holder._assets[i] = None
            if getattr(self, "_owner_ctx", None) is not None:
                # joined group: the context is the caller's and outlives the group; the group goes first so that the peers'
                # mappings of this process's order buffers are closed before the buffers are freed
                self._lib.gs_group_destroy(self.handle)
                free_assets()
            else:
                # created group: the library owns the contexts, so the assets (which live on them) go first
                free_assets()
                self._lib.gs_group_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class GaussianSplatGroupObject:
    """A further splat object on a GaussianSplatGroup (GaussianSplatGroup.add_object): the renderer's knobs and the object's
    asset on every local member.  Its assets are freed by the group's close()."""

    def __init__(self, group: GaussianSplatGroup, asset, share=None):
        import weakref
        self._group = weakref.ref(group)
        self._lib = group._lib
        self.m_Asset = asset
        if share is None:
            self._assets = _upload(group._lib, group.handle, asset, group.local_count)
        else:   # `share`: the group or an object of it whose asset this object instances (add_instance)
            self._assets = _instance(group._lib, share._assets)
        _init_knobs(self)

    @property
    def splatCount(self) -> int:
        return self.m_Asset.splatCount

    def frame_params(self, cam):
        fp, self._keep = _frame_params(self, cam)
        return fp

    def readback_order(self, local: int = 0):
        import numpy as np
        out = np.empty(self.splatCount, np.uint32)
        N.check(None, self._lib.gs_readback_order(self._assets[local], out.ctypes.data))
        return out


def _upload(lib, handle, asset, local_count):
    d = asset.desc()
    assets = (C.c_void_p * local_count)()
    N.check(None, lib.gs_group_asset_upload(handle, C.byref(d), assets))
    return assets


def _instance(lib, sources):
    """gs_asset_instance of every member's asset; on a failure the instances made so far are destroyed."""
    assets = (C.c_void_p * len(sources))()
    for i, src in enumerate(sources):
        h = C.c_void_p()
        rc = lib.gs_asset_instance(src, C.byref(h))
        if rc != N.GS_OK:
            for j in range(i):
                lib.gs_asset_destroy(assets[j])
            N.check(None, rc)
        assets[i] = h.value
    return assets


def _init_knobs(o):
    """The serialized knobs of GaussianSplatRenderer (R/GaussianSplatRenderer.cs:225-251) on a group object."""
    o.m_SplatScale, o.m_OpacityScale, o.m_SHOrder, o.m_SHOnly = 1.0, 1.0, 3, False
    o.m_SortNthFrame, o.m_FrameCounter = 1, 0
    o.m_RenderOrder = 0          # higher values draw first (GatherSplatsForCamera)
    o.localToWorldMatrix = None  # None: identity
    o.m_Cutouts, o.m_DeletedBits, o.m_SelectedBits, o.sceneDepth = [], None, None, None
    o._keep = None


def _frame_params(o, cam):
    from .renderer import make_frame_params
    return make_frame_params(cam, o.localToWorldMatrix, o.m_SplatScale, o.m_OpacityScale, o.m_SHOrder, o.m_SHOnly, o.m_Cutouts,
                             o.m_DeletedBits, o.splatCount, o.m_SelectedBits, o.sceneDepth)


def balance_rows(row_cost, parts: int):
    """gs_group_balance_rows: the library's row balancer (pure host arithmetic)."""
    import numpy as np
    cost = np.ascontiguousarray(row_cost, np.uint32)
    out = np.zeros(parts + 1, np.uint32)
    N.check(None, N.native().gs_group_balance_rows(cost.ctypes.data, cost.size, parts, out.ctypes.data))
    return out
