"""In-tree native build of the two product libraries.

  libgsplat_b200.so   CUDA hot path + C ABI (include/gsplat_b200.h), sm_90a only
  libgsplat_asset.so  host-side asset packer / synthetic scenes (include/gsplat_asset.h)

(The CPU checker under the repo's test-infrastructure directory has its own Makefile and is
built by __graft_entry__.build() / the test session, never from here.)

Everything is compiled by explicit nvcc / g++ command lines (no JIT cache), so the
artefacts travel with the tree to the GPU box.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
CSRC = PKG / "csrc"
NATIVE_LIB = PKG / "libgsplat_b200.so"
ASSET_LIB = PKG / "libgsplat_asset.so"

CU_SOURCES = ["gs_api.cu", "gs_group.cu", "gs_view.cu", "gs_sort.cu", "gs_raster.cu", "gs_export.cu", "gs_pack.cu"]
CU_HEADERS = ["gs_common.cuh", "gs_kernels.cuh", "gs_internal.cuh", "gs_nccl.h", "gs_bc7.cuh", "bc7_tables.h", "../../include/gsplat_b200.h"]


def _host_cxx() -> str:
    for c in ("/usr/bin/g++", shutil.which("g++") or ""):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("no g++ found")


def _nvcc() -> str:
    for c in ("/usr/local/cuda/bin/nvcc", shutil.which("nvcc") or ""):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found: the CUDA extension cannot be built")


def _stale(target: Path, sources) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(s).stat().st_mtime > t for s in sources)


def _run(cmd, cwd=None):
    r = subprocess.run(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: %s\n%s" % (" ".join(map(str, cmd)), r.stdout))
    return r.stdout


def nvcc_flags(extra=()):
    return [
        "-gencode", "arch=compute_90a,code=sm_90a",
        "-O3", "-std=c++17", "-lineinfo",
        "-fmad=false",  # arithmetic contract: FMAs only where fmaf() is written
        "-diag-suppress", "186,128",  # "pointless comparison" / "loop not reachable" in template instantiations that compile a branch out
        "-Xcompiler", "-fPIC,-ffp-contract=off,-fvisibility=hidden",
        "-ccbin", _host_cxx(),
        *extra,
    ]


def build_native(force: bool = False, verbose: bool = False) -> Path:
    """Every .cu is compiled to its own object (in parallel, only when stale), then linked into the in-tree .so."""
    from concurrent.futures import ThreadPoolExecutor
    srcs = [CSRC / s for s in CU_SOURCES]
    hdrs = [CSRC / h for h in CU_HEADERS]
    objdir = PKG / "build"
    objdir.mkdir(exist_ok=True)
    extra = ["-Xptxas", "-v"] if verbose else []
    flag_stamp = objdir / "flags.txt"
    flags_text = " ".join(nvcc_flags(extra))
    if not flag_stamp.exists() or flag_stamp.read_text() != flags_text:
        force = True

    def compile_one(src: Path):
        obj = objdir / (src.stem + ".o")
        if force or _stale(obj, [src, *hdrs]):
            return _run([_nvcc(), *nvcc_flags(extra), "-c", "-o", str(obj), str(src)])
        return ""

    with ThreadPoolExecutor(max_workers=len(srcs)) as ex:
        outs = list(ex.map(compile_one, srcs))
    objs = [objdir / (s.stem + ".o") for s in srcs]
    if force or _stale(NATIVE_LIB, objs):
        _run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-ccbin", _host_cxx(), "-o", str(NATIVE_LIB),
              *map(str, objs), "-ldl"])
    flag_stamp.write_text(flags_text)
    if verbose:
        print("\n".join(o for o in outs if o))
    return NATIVE_LIB


def build_asset(force: bool = False) -> Path:
    srcs = [CSRC / "asset_creator.cpp", CSRC / "asset_cluster_bc7.cpp", CSRC / "asset_export.cpp"]
    if force or _stale(ASSET_LIB, [*srcs, ROOT / "include" / "gsplat_asset.h"]):
        # -mavx2: the k-means distance loops evaluate 16 candidate means side by side (no FMA: -ffp-contract=off)
        _run([_host_cxx(), "-O3", "-mavx2", "-std=c++17", "-fopenmp", "-fPIC", "-shared", "-ffp-contract=off", "-fvisibility=hidden",
              "-o", str(ASSET_LIB), *map(str, srcs), "-lz"])
    return ASSET_LIB


def build_all(force: bool = False, verbose: bool = False):
    return build_native(force, verbose), build_asset(force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built:", NATIVE_LIB, ASSET_LIB)
