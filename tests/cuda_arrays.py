"""CUDA arrays for the array-image tests: 2-D arrays (GS_MEM_ARRAY) and layered ones (GS_MEM_ARRAY_LAYER), made through the CUDA
runtime torch already loaded.  A runtime cudaArray_t is a driver CUarray in the device's primary context, so the library's own
runtime can use it."""
import ctypes as C

import numpy as np

# cudaChannelFormatKind / cudaArray flags / cudaMemcpyKind (cuda_runtime_api.h)
KIND_UNSIGNED, KIND_FLOAT = 1, 2
LAYERED, SURFACE_LOAD_STORE = 0x01, 0x02
H2D, D2H = 1, 2


class _Dim3(C.Structure):
    _fields_ = [("x", C.c_size_t), ("y", C.c_size_t), ("z", C.c_size_t)]   # cudaExtent and cudaPos


class _PitchedPtr(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("pitch", C.c_size_t), ("xsize", C.c_size_t), ("ysize", C.c_size_t)]


class _Memcpy3DParms(C.Structure):
    _fields_ = [("srcArray", C.c_void_p), ("srcPos", _Dim3), ("srcPtr", _PitchedPtr),
                ("dstArray", C.c_void_p), ("dstPos", _Dim3), ("dstPtr", _PitchedPtr), ("extent", _Dim3), ("kind", C.c_int)]


class _ChannelDesc(C.Structure):
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("z", C.c_int), ("w", C.c_int), ("f", C.c_int)]


class Cudart:
    """cudaMalloc3DArray / cudaMemcpy3D / cudaFreeArray through the runtime torch loaded."""

    def __init__(self):
        import torch
        torch.cuda.init()
        self.lib = C.CDLL("libcudart.so.12")   # resolves to the copy torch already loaded (same soname)
        self.lib.cudaMalloc3DArray.argtypes = [C.POINTER(C.c_void_p), C.POINTER(_ChannelDesc), _Dim3, C.c_uint]
        self.lib.cudaMemcpy3D.argtypes = [C.POINTER(_Memcpy3DParms)]
        self.lib.cudaFreeArray.argtypes = [C.c_void_p]
        self.live = []

    def array(self, w, h, depth=0, dtype=np.float16, flags=None, kind=KIND_FLOAT, fill=None):
        """A (depth, h, w) array of RGBA texels of `dtype`'s width (depth 0: a 2-D array), every texel set to `fill` unless it
        is None.  flags None: cudaArraySurfaceLoadStore, and cudaArrayLayered when depth > 0."""
        dtype = np.dtype(dtype)
        bits = 8 * dtype.itemsize
        if flags is None:
            flags = SURFACE_LOAD_STORE | (LAYERED if depth else 0)
        h_ = C.c_void_p()
        rc = self.lib.cudaMalloc3DArray(C.byref(h_), C.byref(_ChannelDesc(bits, bits, bits, bits, kind)), _Dim3(w, h, depth), flags)
        assert rc == 0, "cudaMalloc3DArray failed with CUDA error %d" % rc
        self.live.append(h_.value)
        if fill is not None:
            self.upload(h_.value, np.broadcast_to(np.asarray(fill, dtype), (max(depth, 1), h, w, 4)))
        return h_.value

    def _copy(self, handle, host, kind):
        host = host.reshape((-1,) + host.shape[-3:])   # (layers, h, w, 4): a 2-D array is one layer
        p = _Memcpy3DParms()
        pitched = _PitchedPtr(host.ctypes.data, host.shape[2] * 4 * host.itemsize, host.shape[2], host.shape[1])
        if kind == H2D:
            p.srcPtr, p.dstArray = pitched, handle
        else:
            p.srcArray, p.dstPtr = handle, pitched
        p.extent, p.kind = _Dim3(host.shape[2], host.shape[1], host.shape[0]), kind
        rc = self.lib.cudaMemcpy3D(C.byref(p))
        assert rc == 0, "cudaMemcpy3D failed with CUDA error %d" % rc

    def upload(self, handle, host):
        """host: (h, w, 4) texels of a 2-D array, or (layers, h, w, 4) of a layered one."""
        self._copy(handle, np.ascontiguousarray(host), H2D)

    def download(self, handle, shape, dtype):
        out = np.empty(shape, dtype)   # (h, w, 4), or (layers, h, w, 4)
        self._copy(handle, out, D2H)
        return out

    def free_all(self):
        for h in self.live:
            self.lib.cudaFreeArray(h)
        self.live = []
