"""Test images of every memory kind, in one place: CUDA arrays made through the CUDA runtime torch already loaded, an image of
one memory kind (host, device, a 2-D array, a layer of a layered array or a rectangle of a larger array) holding given texels,
several images in one shared array, and the bit-for-bit check of what a call wrote into an array and what it left alone.

A runtime cudaArray_t is a driver CUarray in the device's primary context, so the library's own runtime can use it.  The
library's stream does not synchronise with the legacy default stream the runtime copies run on: every read syncs the
library's stream first.  Test modules take the `ca` fixture with `from images import ca  # noqa: F401`."""
import ctypes as C

import numpy as np
import pytest

# cudaChannelFormatKind / cudaArray flags / cudaMemcpyKind (cuda_runtime_api.h)
KIND_UNSIGNED, KIND_FLOAT = 1, 2
LAYERED, SURFACE_LOAD_STORE = 0x01, 0x02
H2D, D2H = 1, 2

SENTINEL = -3.25   # exact in half and float
CHANNELS = {"colour": 4, "packed": 1, "depth": 1}   # an image's role: RGBA, a packed B10G11R11 camera target, a depth buffer


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
        self.live = {}   # handle -> (layers, (h, w[, channels]), dtype)

    def array(self, w, h, depth=0, dtype=np.float16, channels=4, fill=None, bits=None, kind=None, flags=None):
        """A (depth, h, w) array of `channels` channels of `dtype` (depth 0: a 2-D array), every texel set to `fill` unless it
        is None.  bits None: dtype's width; kind None: unsigned for an integer dtype, else float; flags None:
        cudaArraySurfaceLoadStore, and cudaArrayLayered when depth > 0."""
        dtype = np.dtype(dtype)
        bits = 8 * dtype.itemsize if bits is None else bits
        kind = (KIND_UNSIGNED if dtype.kind == "u" else KIND_FLOAT) if kind is None else kind
        if flags is None:
            flags = SURFACE_LOAD_STORE | (LAYERED if depth else 0)
        h_ = C.c_void_p()
        desc = _ChannelDesc(*[bits if i < channels else 0 for i in range(4)], kind)
        rc = self.lib.cudaMalloc3DArray(C.byref(h_), C.byref(desc), _Dim3(w, h, depth), flags)
        assert rc == 0, "cudaMalloc3DArray failed with CUDA error %d" % rc
        self.live[h_.value] = (depth, (h, w) + ((channels,) if channels > 1 else ()), dtype)
        if fill is not None:
            self.upload(h_.value, np.broadcast_to(np.asarray(fill, dtype), (max(depth, 1),) + self.live[h_.value][1]))
        return h_.value

    def _copy(self, handle, host, kind):
        host = host.reshape((-1,) + self.live[handle][1])   # (layers, h, w[, channels]): a 2-D array is one layer
        layers, h, w = host.shape[:3]
        p = _Memcpy3DParms()
        pitched = _PitchedPtr(host.ctypes.data, host[0, 0].nbytes, w, h)
        if kind == H2D:
            p.srcPtr, p.dstArray = pitched, handle
        else:
            p.srcArray, p.dstPtr = handle, pitched
        p.extent, p.kind = _Dim3(w, h, layers), kind
        rc = self.lib.cudaMemcpy3D(C.byref(p))
        assert rc == 0, "cudaMemcpy3D failed with CUDA error %d" % rc

    def upload(self, handle, host):
        """host: every texel of the array, in the shape download returns."""
        self._copy(handle, np.ascontiguousarray(host, self.live[handle][2]), H2D)

    def download(self, handle):
        """Every texel: (h, w[, channels]) of a 2-D array, (layers, h, w[, channels]) of a layered one."""
        layers, texels, dtype = self.live[handle]
        out = np.empty(((layers,) if layers else ()) + texels, dtype)
        self._copy(handle, out, D2H)
        return out

    def free_all(self):
        for h in self.live:
            self.lib.cudaFreeArray(h)
        self.live = {}


@pytest.fixture
def ca(ctx):
    c = Cudart()
    yield c
    ctx.sync()
    c.free_all()


def bits(a):
    """The words of an image: float16 as uint16, float32 and uint32 as uint32 (None stays None)."""
    if a is None:
        return None
    a = np.ascontiguousarray(a)
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


def to_device(host):
    """A CUDA tensor of host's texels; uint32 (packed) texels as the int32 tensor the library takes."""
    import torch
    host = np.ascontiguousarray(host)
    return torch.from_numpy(host.view(np.int32) if host.dtype == np.uint32 else host).cuda()


def to_host(ctx, t):
    """A tensor's texels once the library's stream and torch's are done; an int32 (packed) tensor as uint32."""
    import torch
    ctx.sync()
    torch.cuda.synchronize()
    out = t.cpu().numpy()
    return out.view(np.uint32) if out.dtype == np.int32 else out


def launches(ctx):
    return ctx.stage_times().kernel_launches


def background(h, w, dtype, seed):
    """A camera target's content: colours in [0, 1), alpha in [0, 0.5) (so that GS_FLAG_LOAD_RT draws still show)."""
    bg = np.random.default_rng(seed).random((h, w, 4), np.float32)
    bg[..., 3] *= 0.5
    return bg.astype(np.float16).astype(dtype)


def check_regions(got, start, regions, what):
    """got: every texel of an array, (layers, h, w[, channels]); start: what it held before the call (or one texel of it).
    regions: [(layer, x, y, want)]: each rectangle equals `want` word for word, and every other texel of every layer equals
    its start word for word."""
    expect = bits(np.broadcast_to(np.asarray(start, got.dtype), got.shape)).copy()
    got = bits(got)
    for layer, x, y, want in regions:
        want = bits(np.asarray(want))
        h, w = want.shape[:2]
        assert np.array_equal(got[layer or 0, y:y + h, x:x + w], want), \
            "%s: the rectangle at (%d, %d) of layer %d differs" % (what, x, y, layer or 0)
        expect[layer or 0, y:y + h, x:x + w] = want
    bad = got != expect
    assert not bad.any(), "%s: %d texels outside the rectangles were touched" % (what, int(bad.reshape(bad.shape[:3] + (-1,)).any(-1).sum()))


class SharedArray:
    """A (layers, h, w) array (layers 0: a 2-D array) of one role's texels, each starting as `start` (one texel, or all of
    them), that holds several images: .view() is one of them, .fill() gives a rectangle new start content and .check()
    compares the whole array with what the call should have left."""

    def __init__(self, g, ca, w, h, layers=0, dtype=np.float16, role="colour", start=SENTINEL):
        self.g, self.ca, self.w, self.h, self.layers, self.dtype, self.role = g, ca, w, h, layers, np.dtype(dtype), role
        shape = (max(layers, 1), h, w) + ((4,) if role == "colour" else ())
        self.start = np.array(np.broadcast_to(np.asarray(start, dtype), shape))
        self.handle = ca.array(w, h, layers, dtype, CHANNELS[role], fill=self.start)

    def view(self, layer=None, origin=None, size=None):
        """The image (or depth buffer) of `size` (default: the array's) at `origin` of `layer`; no origin: the whole layer."""
        w, h = size or (self.w, self.h)
        if self.role == "depth":
            return self.g.CudaArrayDepth(self.handle, w, h, layer=layer, origin=origin)
        return self.g.CudaArrayImage(self.handle, w, h, np.uint32 if self.role == "packed" else self.dtype, layer=layer, origin=origin)

    def fill(self, layer, x, y, host):
        self.start[layer or 0, y:y + host.shape[0], x:x + host.shape[1]] = host
        self.ca.upload(self.handle, self.start)

    def read(self, ctx):
        ctx.sync()
        return self.ca.download(self.handle).reshape(self.start.shape)

    def check(self, ctx, regions, what):
        """regions: [(layer, x, y, want)], as check_regions takes them."""
        check_regions(self.read(ctx), self.start, regions, what)


class Image:
    """An image of memory kind `kind` holding `content` (h x w texels of `role`): host (a numpy array), device (a tensor),
    array (a 2-D array), layer (layer `layer` of a `layers`-layer array) or rect (the rectangle at (x, y) of an aw x ah 2-D
    array, rect = (aw, ah, x, y)).  Every texel of an array outside the image starts as `start`.  .image is what the Python
    API or _image() takes; .read(ctx) returns the content after the call, having checked the texels outside it."""

    def __init__(self, g, ca, kind, content, role="colour", start=SENTINEL, layers=2, layer=1, rect=None):
        content = np.asarray(content)
        h, w = content.shape[:2]
        self.kind = kind
        if kind == "host":
            self.image = content.copy()
        elif kind == "device":
            self.image = to_device(content)
        else:
            aw, ah, x, y = rect if kind == "rect" else (w, h, 0, 0)
            self.array = SharedArray(g, ca, aw, ah, layers if kind == "layer" else 0, content.dtype, role, start)
            self.region = (layer if kind == "layer" else None, x, y, h, w)
            self.array.fill(self.region[0], x, y, content)
            self.image = self.array.view(layer=self.region[0], origin=(x, y) if kind == "rect" else None, size=(w, h))

    def read(self, ctx):
        if self.kind == "host":
            ctx.sync()
            return self.image.copy()
        if self.kind == "device":
            return to_host(ctx, self.image)
        layer, x, y, h, w = self.region
        got = self.array.read(ctx)
        inside = got[layer or 0, y:y + h, x:x + w]
        check_regions(got, self.array.start, [(layer, x, y, inside)], "%s image" % self.kind)
        return inside
