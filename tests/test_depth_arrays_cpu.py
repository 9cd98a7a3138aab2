"""The host side of a scene depth buffer in a CUDA array (GS_MEM_ARRAY) or a layer of a layered one (GS_MEM_ARRAY_LAYER):
make_frame_params sets the memory kind and keeps the layer descriptor alive, and the ABI structs keep their sizes."""
import ctypes as C
import gc
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from util import camera

ROOT = Path(__file__).resolve().parents[1]


def test_frame_params_memory_kinds(g):
    from unitygaussiansplatting_b200 import _native as N
    cam = camera(g, 64, 32)
    fp, keep = g.make_frame_params(cam, scene_depth=g.CudaArrayDepth(0xABC000, 64, 32))
    assert (fp.scene_depth, fp.scene_depth_on_device) == (0xABC000, N.GS_MEM_ARRAY)
    fp, keep = g.make_frame_params(cam, scene_depth=g.CudaArrayDepth(0xABC000, 64, 32, layer=3))
    assert fp.scene_depth_on_device == N.GS_MEM_ARRAY_LAYER
    gc.collect()   # the descriptor lives as long as `keep`, not only as long as the CudaArrayDepth the caller made
    desc = N.GsArrayLayer.from_address(fp.scene_depth)
    assert (desc.array, desc.layer, desc.reserved) == (0xABC000, 3, 0)
    fp, keep = g.make_frame_params(cam, scene_depth=np.zeros((32, 64), np.float32))
    assert fp.scene_depth_on_device == N.GS_MEM_HOST


def test_cuda_array_depth_rejects_bad_shapes(g):
    cam = camera(g, 64, 32)
    with pytest.raises(ValueError):
        g.make_frame_params(cam, scene_depth=g.CudaArrayDepth(0xABC000, 32, 64))
    with pytest.raises(ValueError):
        g.CudaArrayDepth(0xABC000, 64, 32, layer=-1)
    with pytest.raises(ValueError):
        g.CudaArrayDepth(0xABC000, 0, 32)
    with pytest.raises(ValueError):
        g.CudaArrayDepth(0xABC000, 64, 32, layer=2 ** 32)


def test_abi_struct_sizes_are_unchanged():
    from unitygaussiansplatting_b200 import _native as N
    assert C.sizeof(N.GsFrameParams) == 344 and C.sizeof(N.GsArrayLayer) == 16
    assert C.sizeof(N.GsUnityFrameEvent) == 472 and C.sizeof(N.GsUnityFrameObjectsEvent) == 152
    text = (ROOT / "include" / "gsplat_b200.h").read_text()
    m = re.search(r"typedef struct GsFrameParams \{(.*?)\} GsFrameParams;", text, re.S)
    body = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S)
    assert re.findall(r"(\w+)(?:\[\d+\])?;", body)[-3:] == ["scene_depth", "scene_depth_on_device", "reserved1"]


CPP = r"""
#include "unitygaussiansplatting_b200/host/GaussianSplatRenderer.hpp"
int draw(GaussianSplatting::GaussianSplatRenderer &r, const GaussianSplatting::CameraState &cam, GsImage *rt, void *depth_array,
         GsArrayLayer *eye) {
  r.sceneDepth = static_cast<const float *>(depth_array);
  r.sceneDepthMemory = GS_MEM_ARRAY;
  if (!r.SortAndRenderSplats(cam, rt, nullptr)) return 1;
  r.SetSceneDepthLayer(eye);
  return r.SortAndRenderSplats(cam, rt, nullptr) ? 0 : 1;
}
"""


def test_cpp_mirror_takes_array_depth(tmp_path):
    src = tmp_path / "depth.cpp"
    src.write_text(CPP)
    r = subprocess.run(["/usr/bin/g++", "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I" + str(ROOT), str(src)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
