"""The host side of a rectangle of a CUDA array (GS_MEM_ARRAY_RECT): the header and the Python bindings agree on the kind and on
GsArrayRect, CudaArrayImage / CudaArrayDepth build and check the descriptor, the C++ mirror builds kind-5 images and depth, and
the ABI structs keep their sizes."""
import ctypes as C
import gc
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from util import camera

ROOT = Path(__file__).resolve().parents[1]


def test_header_and_python_agree_on_gs_mem_array_rect():
    from unitygaussiansplatting_b200 import _native as N
    text = (ROOT / "include" / "gsplat_b200.h").read_text()
    m = re.search(r"#define GS_MEM_ARRAY_RECT (\d+)u", text)
    assert m and int(m.group(1)) == N.GS_MEM_ARRAY_RECT == 5
    m = re.search(r"typedef struct GsArrayRect \{(.*?)\} GsArrayRect;", text, re.S)
    body = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S)
    assert re.findall(r"(\w+)(?:,\s*(\w+))?;", body) == [("array", ""), ("layer", ""), ("x", "y"), ("reserved", "")]
    assert [f[0] for f in N.GsArrayRect._fields_] == ["array", "layer", "x", "y", "reserved"]
    assert C.sizeof(N.GsArrayRect) == 24 and N.GsArrayRect.x.offset == 12 and N.GsArrayRect.reserved.offset == 20


def test_abi_struct_sizes_are_unchanged():
    from unitygaussiansplatting_b200 import _native as N
    assert C.sizeof(N.GsImage) == 32 and C.sizeof(N.GsFrameParams) == 344 and C.sizeof(N.GsArrayLayer) == 16
    assert C.sizeof(N.GsUnityFrameEvent) == 472 and C.sizeof(N.GsUnityFrameObjectsEvent) == 152


def test_cuda_array_image_origin_builds_a_rect_descriptor(g):
    from unitygaussiansplatting_b200 import _native as N
    from unitygaussiansplatting_b200.renderer import _image
    im = _image(g.CudaArrayImage(0x1234, 8, 4, np.float32, origin=(37, 19)), 8, 4)
    assert im.memory == N.GS_MEM_ARRAY_RECT and im.row_pitch_bytes == 0 and im.format == N.GS_PIX_RGBA32F
    assert (im.width, im.height) == (8, 4)   # the rectangle is the image
    gc.collect()   # the descriptor lives as long as the image that points to it
    d = N.GsArrayRect.from_address(im.data)
    assert (d.array, d.layer, d.x, d.y, d.reserved) == (0x1234, 0, 37, 19, 0)
    im = _image(g.CudaArrayImage(0x1234, 8, 4, layer=2, origin=(np.int64(0), 2 ** 32 - 1)), 8, 4)
    d = N.GsArrayRect.from_address(im.data)
    assert im.memory == N.GS_MEM_ARRAY_RECT and im.format == N.GS_PIX_RGBA16F and (d.layer, d.x, d.y) == (2, 0, 2 ** 32 - 1)
    # without an origin the kinds are those of before
    assert _image(g.CudaArrayImage(0x1234, 8, 4), 8, 4).memory == N.GS_MEM_ARRAY
    assert _image(g.CudaArrayImage(0x1234, 8, 4, layer=1), 8, 4).memory == N.GS_MEM_ARRAY_LAYER
    with pytest.raises(ValueError):   # the rectangle is the screen: its size must be the image's
        _image(g.CudaArrayImage(0x1234, 8, 4, origin=(0, 0)), 16, 4)


@pytest.mark.parametrize("origin", [(-1, 0), (0, -5), (1.5, 0), (0, 2.0), ("1", 0), (True, 0), (2 ** 32, 0), (1,), (1, 2, 3), 7,
                                    (1, None)])
def test_bad_origins_are_refused(g, origin):
    for make in (lambda: g.CudaArrayImage(0x1234, 8, 4, origin=origin), lambda: g.CudaArrayDepth(0x1234, 8, 4, origin=origin)):
        with pytest.raises(ValueError):
            make()


def test_frame_params_take_a_depth_rectangle(g):
    from unitygaussiansplatting_b200 import _native as N
    cam = camera(g, 64, 32)
    fp, keep = g.make_frame_params(cam, scene_depth=g.CudaArrayDepth(0xABC000, 64, 32, origin=(5, 7)))
    assert fp.scene_depth_on_device == N.GS_MEM_ARRAY_RECT
    gc.collect()   # the descriptor lives as long as `keep`
    d = N.GsArrayRect.from_address(fp.scene_depth)
    assert (d.array, d.layer, d.x, d.y, d.reserved) == (0xABC000, 0, 5, 7, 0)
    fp, keep = g.make_frame_params(cam, scene_depth=g.CudaArrayDepth(0xABC000, 64, 32, layer=3, origin=(0, 0)))
    assert fp.scene_depth_on_device == N.GS_MEM_ARRAY_RECT and N.GsArrayRect.from_address(fp.scene_depth).layer == 3
    with pytest.raises(ValueError):   # the rectangle is the screen
        g.make_frame_params(cam, scene_depth=g.CudaArrayDepth(0xABC000, 32, 64, origin=(0, 0)))


def test_header_documents_depth_kind_5():
    text = (ROOT / "include" / "gsplat_b200.h").read_text()
    m = re.search(r"uint32_t scene_depth_on_device; /\*(.*?)\*/", text, re.S)
    doc = " ".join(m.group(1).split())
    assert "GS_MEM_ARRAY_RECT (5)" in doc and "refuse 2, 4 and 5" in doc
    assert "Any other value (1, 3, 6, ...): device memory" in doc


CPP = r"""
#include "unitygaussiansplatting_b200/host/GaussianSplatRenderer.hpp"
static_assert(sizeof(GsArrayRect) == 24, "GsArrayRect is 24 bytes");
static_assert(sizeof(GsImage) == 32, "GsImage is 32 bytes");
static_assert(GS_MEM_ARRAY_RECT == 5u, "kind 5");
int draw(GaussianSplatting::GaussianSplatRenderer &r, const GaussianSplatting::CameraState &cam, void *colour, void *depth) {
  GsArrayRect tile{colour, 0, 37, 19, 0}, eye{depth, 1, 0, 0, 0};
  GsImage rt = GaussianSplatting::ArrayRectImage(&tile, 200, 120, GS_PIX_RGBA32F);
  if (rt.memory != GS_MEM_ARRAY_RECT || rt.data != &tile || rt.row_pitch_bytes != 0) return 2;
  r.SetSceneDepthRect(&eye);
  if (r.sceneDepthMemory != GS_MEM_ARRAY_RECT) return 3;
  return r.SortAndRenderSplats(cam, &rt, nullptr) ? 0 : 1;
}
"""


def test_cpp_mirror_builds_rect_images_and_depth(tmp_path):
    src = tmp_path / "rect.cpp"
    src.write_text(CPP)
    r = subprocess.run(["/usr/bin/g++", "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I" + str(ROOT), str(src)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
