"""The CPU restatement of GS_PIX_B10G11R11_UFLOAT camera targets (tests/packed_oracle.c), compiled once per process into a
temporary directory, with -ffp-contract=off as the CPU oracle is, and bound through ctypes."""
import atexit
import ctypes as C
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
_lib = None
_path = None


def path() -> Path:
    """The compiled libpacked_oracle.so."""
    global _path
    if _path is None:
        d = Path(tempfile.mkdtemp(prefix="packed_oracle_"))
        atexit.register(shutil.rmtree, d, True)
        so = d / "libpacked_oracle.so"
        cc = "/usr/bin/gcc" if Path("/usr/bin/gcc").exists() else "gcc"
        r = subprocess.run([cc, "-O2", "-ffp-contract=off", "-fno-math-errno", "-fPIC", "-shared", "-std=c11", "-Wall", "-Wextra",
                            "-o", str(so), str(HERE / "packed_oracle.c"), "-lm"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("packed_oracle.c does not compile:\n" + r.stdout)
        _path = so
    return _path


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(str(path()))
        for f in (L.gso_f32_to_uf11, L.gso_f32_to_uf10):
            f.restype, f.argtypes = C.c_uint32, [C.c_float]
        for f in (L.gso_uf11_to_f32, L.gso_uf10_to_f32):
            f.restype, f.argtypes = C.c_float, [C.c_uint32]
        L.gso_composite_b10g11r11.restype, L.gso_composite_b10g11r11.argtypes = None, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]
        _lib = L
    return _lib


def composite_b10g11r11(rt: np.ndarray, target: np.ndarray) -> np.ndarray:
    """(H, W, 4) render target onto (H, W) uint32 B10G11R11_UFLOAT texels; returns the new texels."""
    rt = np.ascontiguousarray(rt, np.float32)
    out = np.ascontiguousarray(target, np.uint32).copy()
    assert out.shape == rt.shape[:2]
    lib().gso_composite_b10g11r11(rt.ctypes.data, out.ctypes.data, rt.shape[1], rt.shape[0])
    return out
