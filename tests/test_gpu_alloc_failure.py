"""A device allocation the library cannot make is reported by the call that asked for it, and by no later call: a refused
asset upload leaves no CUDA error behind for the next upload and frame on the same context."""
import ctypes as C

import numpy as np
import pytest

from util import camera

pytestmark = pytest.mark.gpu

GS_ERR_OUT_OF_MEMORY = -3


def _frame(g, context, asset, cam):
    r = g.GaussianSplatRenderer(asset, context)
    try:
        rt = np.zeros((cam.pixelHeight, cam.pixelWidth, 4), np.float16)
        r.SortAndRenderSplats(cam, rt=rt)
        context.sync()
        return rt, r.readback_order()
    finally:
        r.Dispose()


def test_refused_upload_leaves_no_error_for_the_next_frame(g, ctx):
    """A 2^50-byte position blob cannot be allocated: gs_asset_upload returns GS_ERR_OUT_OF_MEMORY and no asset.  The same
    asset, uploaded correctly on the same context, then renders the frame a fresh context renders, bit for bit."""
    asset = g.synthetic_asset(g.SCENE_CLUSTERED, 20000, 0x5EED0002, "Medium")
    cam = camera(g, 320, 200)
    refused = g.GaussianSplatContext(0)   # a fresh context (not the session's), whose next upload and frame are checked
    try:
        d = asset.desc()
        d.pos_bytes = 1 << 50
        h = C.c_void_p()
        assert refused._lib.gs_asset_upload(refused.handle, C.byref(d), C.byref(h)) == GS_ERR_OUT_OF_MEMORY
        assert not h.value
        rt, order = _frame(g, refused, asset, cam)
    finally:
        refused.close()
    fresh = g.GaussianSplatContext(0)
    try:
        rt_ref, order_ref = _frame(g, fresh, asset, cam)
    finally:
        fresh.close()
    assert rt_ref[..., 3].max() > 0
    assert np.array_equal(order, order_ref)
    assert np.array_equal(rt.view(np.uint16), rt_ref.view(np.uint16))
