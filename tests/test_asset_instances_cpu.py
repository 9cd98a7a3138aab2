"""gs_asset_instance without a device: the library exports it, the header's declaration and the ctypes binding agree, null
arguments are refused before any CUDA call, and the C++ host mirror's instance entry points compile against the header (on
the GPU box the same program draws and compares its frames)."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import pytest

from conftest import has_cuda

ROOT = Path(__file__).resolve().parents[1]
INVALID = -1


def test_symbol_is_exported_and_bound(g):
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    assert hasattr(lib, "gs_asset_instance")
    res, args = N.NATIVE_SYMBOLS["gs_asset_instance"]
    assert res is C.c_int and args == [C.c_void_p, C.POINTER(C.c_void_p)]


def test_header_declaration_matches_the_binding():
    text = (ROOT / "include" / "gsplat_b200.h").read_text()
    decl = re.findall(r"GS_API\s+(\w+)\s+gs_asset_instance\s*\(([^)]*)\)\s*;", text)
    assert decl == [("int", "const GsAsset *source, GsAsset **out")]
    # gs_asset_device_ptr documents the blob pointers 3-7
    m = re.search(r"/\*([^*]|\*(?!/))*\*/\s*GS_API void \*gs_asset_device_ptr", text)
    assert m and all(w in m.group(0) for w in ("3 pos", "4 other", "5 sh", "6 color", "7 chunks"))


def test_null_arguments_are_refused_without_a_device(g):
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    h = C.c_void_p(1234)
    assert lib.gs_asset_instance(None, C.byref(h)) == INVALID
    assert not h.value, "*out must be NULL after a refused call"
    assert lib.gs_asset_instance(None, None) == INVALID
    assert b"null" in lib.gs_last_error(None)


def _build(tmp_path):
    exe = tmp_path / "asset_instance_test"
    lib = ROOT / "unitygaussiansplatting_b200"
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Werror", str(ROOT / "tests" / "asset_instance_test.cpp"), "-o", str(exe),
                    "-L" + str(lib), "-lgsplat_b200", "-Wl,-rpath," + str(lib)], check=True)
    return exe


@pytest.mark.skipif(has_cuda(), reason="CPU-only behaviour")
def test_host_mirror_instances_compile_and_fail_loudly_without_a_device(tmp_path):
    r = subprocess.run([str(_build(tmp_path))], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 3 and "no CUDA device" in r.stderr


@pytest.mark.gpu
def test_host_mirror_instances_draw_what_uploads_draw(tmp_path):
    r = subprocess.run([str(_build(tmp_path))], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
