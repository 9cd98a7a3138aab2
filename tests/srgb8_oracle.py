"""The CPU restatement of GS_PIX_R8G8B8A8_SRGB camera targets (tests/srgb8_oracle.c), compiled once per process into a
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
    """The compiled libsrgb8_oracle.so."""
    global _path
    if _path is None:
        d = Path(tempfile.mkdtemp(prefix="srgb8_oracle_"))
        atexit.register(shutil.rmtree, d, True)
        so = d / "libsrgb8_oracle.so"
        cc = "/usr/bin/gcc" if Path("/usr/bin/gcc").exists() else "gcc"
        r = subprocess.run([cc, "-O2", "-ffp-contract=off", "-fno-math-errno", "-fPIC", "-shared", "-std=c11", "-Wall", "-Wextra",
                            "-o", str(so), str(HERE / "srgb8_oracle.c"), "-lm"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("srgb8_oracle.c does not compile:\n" + r.stdout)
        _path = so
    return _path


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(str(path()))
        for f in (L.gso_srgb8_encode, L.gso_unorm8_encode):
            f.restype, f.argtypes = C.c_uint32, [C.c_float]
        for f in (L.gso_srgb8_decode, L.gso_unorm8_decode):
            f.restype, f.argtypes = C.c_float, [C.c_uint32]
        L.gso_composite_srgb8.restype, L.gso_composite_srgb8.argtypes = None, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]
        _lib = L
    return _lib


def encode(x: np.ndarray, alpha: bool = False) -> np.ndarray:
    """The oracle's encoder over an array of float32 values (RGB channels, or alpha)."""
    fn = lib().gso_unorm8_encode if alpha else lib().gso_srgb8_encode
    x = np.asarray(x, np.float32)
    return np.fromiter((fn(float(v)) for v in x.reshape(-1)), np.uint8, x.size).reshape(x.shape)


def composite_srgb8(rt: np.ndarray, target: np.ndarray) -> np.ndarray:
    """(H, W, 4) render target onto (H, W, 4) uint8 R8G8B8A8_SRGB texels; returns the new texels."""
    rt = np.ascontiguousarray(rt, np.float32)
    out = np.ascontiguousarray(target, np.uint8).copy()
    assert out.shape == rt.shape
    lib().gso_composite_srgb8(rt.ctypes.data, out.ctypes.data, rt.shape[1], rt.shape[0])
    return out
