"""gs_frame_objects without a device: the exported symbols, the Unity payload's layout and error path, the C++ mirror's
single-GPU SortAndRenderSplatsMulti, and the Python rule that picks one call or the per-object loop."""
import ctypes as C
import subprocess
from pathlib import Path
from types import SimpleNamespace

import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_new_symbols_are_exported():
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    for name in ("gs_frame_objects", "gs_unity_frame_objects_event_size"):
        assert hasattr(lib, name)


def test_frame_objects_event_layout_and_error_path():
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    assert lib.gs_unity_frame_objects_event_size() == C.sizeof(N.GsUnityFrameObjectsEvent)
    assert N.GsUnityFrameObjectsEvent.options.offset == 40 and N.GsUnityFrameObjectsEvent.rt.offset == 88
    ev = N.GsUnityFrameObjectsEvent()
    ev.status = -5
    lib.gs_unity_get_render_event_func()(N.GS_UNITY_EVENT_FRAME_OBJECTS, C.addressof(ev))   # null context: no CUDA call
    assert ev.status == -1
    assert lib.gs_frame_objects(None, 1, None, None, None, None, None, None) == -1


SRC = r'''
#include "unitygaussiansplatting_b200/host/GaussianSplatRenderer.hpp"
int main() {
  GaussianSplatting::GaussianSplatRenderer a, b;
  GaussianSplatting::CameraState cam{};
  b.OnEnable(GsAssetDesc{}, a.context());
  b.m_RenderOrder = 1;
  GsImage *rt = nullptr, *target = nullptr;
  return GaussianSplatting::GaussianSplatRenderer::SortAndRenderSplatsMulti(cam, {&a, &b}, rt, target) ? 0 : 1;
}
'''


def test_single_gpu_multi_object_mirror_compiles(tmp_path):
    src = tmp_path / "frame_objects.cpp"
    src.write_text(SRC)
    r = subprocess.run(["/usr/bin/g++", "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I" + str(ROOT), str(src)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout


def _stub(context, **kw):
    r = SimpleNamespace(context=context, blend_mode=0, async_readback=False, partition=(0, 0, 1), rows=(0, 0), band_packed=False)
    for k, v in kw.items():
        setattr(r, k, v)
    return r


@pytest.mark.parametrize("other, one_call", [
    (dict(), True),
    (dict(load_rt=True), True),              # the call clears the target itself; the flag is the loop's
    (dict(blend_mode=1), False),
    (dict(async_readback=True), False),
    (dict(partition=(1, 2, 1)), False),
    (dict(rows=(0, 4)), False),
    (dict(band_packed=True), False),
    (dict(context="another"), False),
])
def test_routing_rule(other, one_call):
    from unitygaussiansplatting_b200.renderer import draws_in_one_call
    ctx = "ctx"
    kw = dict(other)
    second = _stub(kw.pop("context", ctx), **kw)
    assert draws_in_one_call([_stub(ctx), second]) is one_call
    assert draws_in_one_call([_stub(ctx)]) is True
