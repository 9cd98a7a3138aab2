"""CreateAsset on the GPU (gs_pack_asset): the same blobs create_asset writes, packed by libgsplat_b200.so.

create_asset (csrc/asset_creator.cpp) stays the specification and the host path; pack_asset is its device twin for
finite input.  It reads its input without modifying it, and can leave the packed asset in HBM, ready to render.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _native as N
from .asset import INPUT_SPLAT_FLOATS, QUALITY, ColorFormat, GaussianSplatAsset, SHFormat, VectorFormat
from .renderer import GaussianSplatContext, GaussianSplatRenderer


def pack_sizes(n: int, formats) -> N.GsPackSizes:
    pf, sf, cf, shf = (int(f) for f in formats)
    sz = N.GsPackSizes()
    N.check(None, N.native().gs_pack_sizes(n, pf, sf, cf, shf, C.byref(sz)))
    return sz


def pack_asset(splats, quality: str = "Medium", formats=None, context: Optional[GaussianSplatContext] = None,
               keep_on_device: bool = False):
    """Packs `splats` ((n, 62) float32 InputSplatData records: a numpy array, or a CUDA torch tensor read in place) on the
    GPU.  Returns the GaussianSplatAsset create_asset would return for the same input; with keep_on_device=True returns
    (asset, renderer), the renderer built on the packed device asset without uploading the blobs again."""
    pf, sf, cf, shf = formats if formats is not None else QUALITY[quality]
    context = context or GaussianSplatContext(0)
    desc = N.GsPackDesc()
    if isinstance(splats, np.ndarray):
        if not (splats.dtype == np.float32 and splats.ndim == 2 and splats.shape[1] == INPUT_SPLAT_FLOATS and splats.flags.c_contiguous):
            raise ValueError("splats must be a C-contiguous (n, 62) float32 array")
        desc.splats, desc.memory = splats.ctypes.data, N.GS_MEM_HOST
    else:   # torch tensor (duck-typed so torch stays optional)
        import torch
        if not (splats.dtype == torch.float32 and splats.dim() == 2 and splats.shape[1] == INPUT_SPLAT_FLOATS and splats.is_contiguous()):
            raise ValueError("splats must be a contiguous (n, 62) float32 tensor")
        if not splats.is_cuda or splats.device.index != context.device:
            raise ValueError("a tensor input must live on the context's CUDA device")
        torch.cuda.current_stream(splats.device).synchronize()   # the packer reads it on the context's own stream
        desc.splats, desc.memory = splats.data_ptr(), N.GS_MEM_DEVICE
    n = int(splats.shape[0])
    desc.splat_count = n
    desc.pos_format, desc.scale_format, desc.color_format, desc.sh_format = int(pf), int(sf), int(cf), int(shf)
    sz = pack_sizes(n, (pf, sf, cf, shf))
    pos = np.zeros(sz.pos_bytes, np.uint8)
    other = np.zeros(sz.other_bytes, np.uint8)
    color = np.zeros(sz.color_bytes, np.uint8)
    sh = np.zeros(sz.sh_bytes, np.uint8)
    chunks = np.zeros(sz.chunk_bytes, np.uint8) if sz.chunk_bytes else None
    out = N.GsPackedAsset()
    out.pos, out.other, out.color, out.sh = pos.ctypes.data, other.ctypes.data, color.ctypes.data, sh.ctypes.data
    out.chunks = chunks.ctypes.data if chunks is not None else None
    out.memory = N.GS_MEM_HOST
    h = C.c_void_p()
    N.check(context.handle, context._lib.gs_pack_asset(context.handle, C.byref(desc), C.byref(out),
                                                       C.byref(h) if keep_on_device else None))
    asset = GaussianSplatAsset(n, VectorFormat(pf), VectorFormat(sf), ColorFormat(cf), SHFormat(shf), pos, other, color, sh, chunks,
                               np.array(out.bounds_min, np.float32), np.array(out.bounds_max, np.float32))
    if keep_on_device:
        return asset, GaussianSplatRenderer.from_device_asset(asset, h, context)
    return asset


def kmeans(data: np.ndarray, k: int, batch: int = 2048, passes: float = 1.2, context: Optional[GaussianSplatContext] = None):
    """gs_kmeans: the device twin of gsa_kmeans.  data (n, dim) float32 -> (means (k, dim) float32, labels (n,) int32)."""
    data = np.ascontiguousarray(data, np.float32)
    context = context or GaussianSplatContext(0)
    n, dim = data.shape
    means = np.zeros((k, dim), np.float32)
    labels = np.zeros(n, np.int32)
    N.check(context.handle, context._lib.gs_kmeans(context.handle, dim, data.ctypes.data, n, batch, passes, means.ctypes.data, k,
                                                   labels.ctypes.data))
    return means, labels


def pack_stats(context: GaussianSplatContext) -> np.ndarray:
    """gs_debug_pack_stats of the context's last pack: [pow values recomputed on the host, mini-batch iterations,
    k-means++ rounds, 0]."""
    out = np.zeros(4, np.uint64)
    N.check(context.handle, context._lib.gs_debug_pack_stats(context.handle, out.ctypes.data))
    return out
