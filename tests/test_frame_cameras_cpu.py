"""gs_frame_cameras without a device: the exported symbol, the NULL-context error, the C++ mirror's
SortAndRenderSplatsCameras, and the Python rule that picks one call or the per-camera loop."""
import subprocess
from pathlib import Path
from types import SimpleNamespace

import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_symbol_is_exported():
    from unitygaussiansplatting_b200 import _native as N
    assert hasattr(N.native(), "gs_frame_cameras")


def test_null_context_is_refused():
    from unitygaussiansplatting_b200 import _native as N
    assert N.native().gs_frame_cameras(None, 1, None, None, None, None, None, None, None) == -1


SRC = r'''
#include "unitygaussiansplatting_b200/host/GaussianSplatRenderer.hpp"
int main() {
  GaussianSplatting::GaussianSplatRenderer a, b;
  b.OnEnable(GsAssetDesc{}, a.context());
  b.m_RenderOrder = 1;
  std::vector<GaussianSplatting::CameraState> cams(2);
  std::vector<GsImage *> rts = {nullptr, nullptr}, targets = {nullptr, nullptr};
  return GaussianSplatting::GaussianSplatRenderer::SortAndRenderSplatsCameras(cams, {&a, &b}, rts, targets) ? 0 : 1;
}
'''


def test_camera_loop_mirror_compiles(tmp_path):
    src = tmp_path / "frame_cameras.cpp"
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
    (dict(load_rt=True), True),              # each camera's target is cleared by the call; the flag is the loop's
    (dict(blend_mode=1), False),             # a camera whose renderers differ in blend mode is drawn object by object
    (dict(async_readback=True), False),
    (dict(partition=(1, 2, 1)), False),
    (dict(rows=(0, 4)), False),
    (dict(band_packed=True), False),
    (dict(context="another"), False),
])
def test_routing_rule_within_a_camera(other, one_call):
    from unitygaussiansplatting_b200.renderer import cameras_in_one_call
    kw = dict(other)
    second = _stub(kw.pop("context", "ctx"), **kw)
    assert cameras_in_one_call([[_stub("ctx")], [_stub("ctx"), second]]) is one_call
    assert cameras_in_one_call([[_stub("ctx")], [_stub("ctx")]]) is True


@pytest.mark.parametrize("second, one_call", [
    (dict(), True),
    (dict(context="another"), False),        # cameras on two contexts
    (dict(async_readback=True), False),      # no per-camera asynchronous staging
    (dict(blend_mode=1), False),             # one blend mode for the call
])
def test_routing_rule_across_cameras(second, one_call):
    from unitygaussiansplatting_b200.renderer import cameras_in_one_call
    kw = dict(second)
    cam1 = [_stub(kw.pop("context", "ctx"), **kw)]
    assert cameras_in_one_call([[_stub("ctx")], cam1]) is one_call


def test_mirror_advances_the_frame_counter_per_camera(monkeypatch):
    """SortAndRenderCameras gathers per camera and advances each renderer's counter once per camera that draws it."""
    from unitygaussiansplatting_b200 import renderer as R
    calls = []
    monkeypatch.setattr(R, "_frame_cameras", lambda actives, cams, rts, tgts: calls.append([len(a) for a in actives]))
    monkeypatch.setattr(R, "GatherSplatsForCamera", lambda rs, cam: list(rs) if cam != "empty" else [])
    rs = [_stub("ctx"), _stub("ctx")]
    out = R.SortAndRenderCameras(rs, ["a", "empty", "b"], [None, None, None], ["t", None, "t"])
    assert calls == [[2, 2]] and [len(a) for a in out] == [2, 0, 2]
