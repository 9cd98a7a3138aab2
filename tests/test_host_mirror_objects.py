"""The C++ host mirror's multi-object group call (GaussianSplatRendererGroup::AddObject / SortAndRenderSplatsMulti) compiles
against the C ABI."""
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]

SRC = r'''
#include "unitygaussiansplatting_b200/host/GaussianSplatRenderer.hpp"
int main() {
  GaussianSplatting::GaussianSplatRendererGroup grp;
  GaussianSplatting::CameraState cam{};
  GaussianSplatting::GaussianSplatGroupObject *other = grp.AddObject(GsAssetDesc{});
  other = other ? other : &grp;
  other->m_RenderOrder = 1;
  GsImage *rts[1] = {nullptr}, *targets[1] = {nullptr};
  return grp.SortAndRenderSplatsMulti(cam, {&grp, other}, rts, targets) ? 0 : 1;
}
'''


def test_group_multi_object_mirror_compiles(tmp_path):
    src = tmp_path / "objects.cpp"
    src.write_text(SRC)
    r = subprocess.run(["/usr/bin/g++", "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I" + str(ROOT), str(src)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
