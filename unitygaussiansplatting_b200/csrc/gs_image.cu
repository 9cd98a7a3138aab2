// gs_image.cu -- how the library reaches the pixels of a GsImage in each memory kind: validation, the device view a kernel
// draws into (the image itself, a surface of its CUDA array, or a staging image), and the copy of a linear device image into
// an image of any kind.  The same for the scene depth buffer a draw is tested against.
#include <cstring>
#include <string>

#include "gs_internal.cuh"

namespace gs {

uint32_t pix_bytes(uint32_t fmt) {
  return fmt == GS_PIX_RGBA16F ? 8u : (fmt == GS_PIX_B10G11R11_UFLOAT || fmt == GS_PIX_R8G8B8A8_SRGB) ? 4u : 16u;
}

// The rules every CUDA array the library reads or writes keeps: `a` (a GS_MEM_ARRAY, GS_MEM_ARRAY_LAYER or GS_MEM_ARRAY_RECT view:
// data and memory) is a W x H 2-D array, a layer below the layer count of a W x H layered one, or a W x H rectangle inside a
// 2-D array or inside a layer of a layered one, made with cudaArraySurfaceLoadStore, whose channels are `channels` x
// `bits`-bit of kind `kind` (else GS_ERR_UNSUPPORTED_FORMAT; everything else is GS_ERR_INVALID_ARGUMENT).  The messages start
// with `prefix`, and name the size `of` and the channels `format` expected.
static int array_ok(GsContext *ctx, const GsImage &a, uint32_t W, uint32_t H, cudaChannelFormatKind kind, int channels, int bits,
                    const char *prefix, const char *of, const char *format) {
  const std::string p(prefix);
  const bool layered = a.memory == GS_MEM_ARRAY_LAYER, rect = a.memory == GS_MEM_ARRAY_RECT;
  if (layered) {
    const GsArrayLayer *d = static_cast<const GsArrayLayer *>(a.data);
    if (!d->array || d->reserved) return fail(ctx, GS_ERR_INVALID_ARGUMENT, p + "GsArrayLayer: array is null or reserved is not 0");
  }
  if (rect) {
    const GsArrayRect *d = static_cast<const GsArrayRect *>(a.data);
    if (!d->array || d->reserved) return fail(ctx, GS_ERR_INVALID_ARGUMENT, p + "GsArrayRect: array is null or reserved is not 0");
  }
  int32_t layer = -1;
  uint32_t x = 0, y = 0;
  cudaChannelFormatDesc cd;
  cudaExtent ext;
  unsigned int flags = 0;
  const cudaError_t e = cudaArrayGetInfo(&cd, &ext, &flags, image_array(&a, &layer, &x, &y));
  if (e != cudaSuccess) { cudaGetLastError(); return fail(ctx, GS_ERR_INVALID_ARGUMENT, p + "not a CUDA array: " + cudaGetErrorString(e)); }
  const int want[4] = {bits, channels > 1 ? bits : 0, channels > 2 ? bits : 0, channels > 3 ? bits : 0};
  if (cd.f != kind || cd.x != want[0] || cd.y != want[1] || cd.z != want[2] || cd.w != want[3])
    return fail(ctx, GS_ERR_UNSUPPORTED_FORMAT, p + "the CUDA array's channel format does not match " + format);
  if (rect) {
    const bool is_layered = (flags & cudaArrayLayered) != 0;
    if (!is_layered && ext.depth != 0)
      return fail(ctx, GS_ERR_INVALID_ARGUMENT, p + "the CUDA array is a 3-D array, not a 2-D or layered one");
    if (!is_layered && layer != 0) return fail(ctx, GS_ERR_INVALID_ARGUMENT, p + "the layer of a 2-D CUDA array must be 0");
    if (is_layered && (uint32_t)layer >= ext.depth)
      return fail(ctx, GS_ERR_INVALID_ARGUMENT, p + "the layer is not below the CUDA array's layer count");
    if ((uint64_t)x + W > ext.width || (uint64_t)y + H > ext.height)   // 64-bit: a huge origin must not wrap around
      return fail(ctx, GS_ERR_INVALID_ARGUMENT, p + "the rectangle of " + of + " size does not lie inside the CUDA array");
  } else {
    if (!layered && (ext.width != W || ext.height != H || ext.depth != 0))
      return fail(ctx, GS_ERR_INVALID_ARGUMENT, p + "the CUDA array is not a 2-D array of " + of + " size");
    if (layered && (ext.width != W || ext.height != H || !(flags & cudaArrayLayered)))
      return fail(ctx, GS_ERR_INVALID_ARGUMENT, p + "the CUDA array is not a layered array of " + of + " size");
    if (layered && (uint32_t)layer >= ext.depth)
      return fail(ctx, GS_ERR_INVALID_ARGUMENT, p + "the layer is not below the CUDA array's layer count");
  }
  if (!(flags & cudaArraySurfaceLoadStore))
    return fail(ctx, GS_ERR_INVALID_ARGUMENT, p + "the CUDA array was not created with cudaArraySurfaceLoadStore");
  return GS_OK;
}

bool array_layered(cudaArray_t arr) {
  cudaChannelFormatDesc cd;
  cudaExtent ext;
  unsigned int flags = 0;
  if (cudaArrayGetInfo(&cd, &ext, &flags, arr) != cudaSuccess) { cudaGetLastError(); return false; }
  return (flags & cudaArrayLayered) != 0;
}

int image_ok(GsContext *ctx, const GsImage *im, uint32_t W, uint32_t H, ImageRole role, uint32_t *pitch) {
  if (!im || !im->data) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "image is null");
  const bool packed = im->format == GS_PIX_B10G11R11_UFLOAT, srgb8 = im->format == GS_PIX_R8G8B8A8_SRGB;
  if (im->format > GS_PIX_R8G8B8A8_SRGB) return fail(ctx, GS_ERR_UNSUPPORTED_FORMAT, "unsupported pixel format");
  if (packed && role != ImageRole::kCameraTarget)
    return fail(ctx, GS_ERR_UNSUPPORTED_FORMAT, "GS_PIX_B10G11R11_UFLOAT is a camera-target format, not a render-target one");
  if (srgb8 && role != ImageRole::kCameraTarget)
    return fail(ctx, GS_ERR_UNSUPPORTED_FORMAT, "GS_PIX_R8G8B8A8_SRGB is a camera-target format, not a render-target one");
  if (im->memory > GS_MEM_ARRAY_RECT || im->memory == 3)   // 3 is not a memory kind
    return fail(ctx, GS_ERR_INVALID_ARGUMENT, "unknown image memory kind");
  if (im->width != W || im->height != H) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "image size does not match screen size");
  if (is_array_image(im)) {   // a 2-D CUDA array (data is a cudaArray_t), a layer of a layered one (a GsArrayLayer *) or a
                              // rectangle of either (a GsArrayRect *)
    if (im->row_pitch_bytes) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "row_pitch_bytes must be 0 for a CUDA array image");
    const int rc = packed ? array_ok(ctx, *im, W, H, cudaChannelFormatKindUnsigned, 1, 32, "", "the image's", "one 32-bit unsigned channel")
                   : srgb8  ? array_ok(ctx, *im, W, H, cudaChannelFormatKindUnsigned, 4, 8, "", "the image's", "four 8-bit unsigned channels")
                            : array_ok(ctx, *im, W, H, cudaChannelFormatKindFloat, 4, im->format == GS_PIX_RGBA16F ? 16 : 32, "",
                                       "the image's", "the image's pixel format");
    if (rc) return rc;
    *pitch = 0;
    return GS_OK;
  }
  uint32_t p = im->row_pitch_bytes ? im->row_pitch_bytes : W * pix_bytes(im->format);
  if (p < W * pix_bytes(im->format) || (p % pix_bytes(im->format)) != 0) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "bad row pitch");
  *pitch = p;
  return GS_OK;
}

bool images_overlap(const GsImage *a, const GsImage *b) {
  if (!a || !b || is_array_image(a) != is_array_image(b)) return false;
  if (!is_array_image(a)) return a->data == b->data;
  int32_t la = -1, lb = -1;
  uint32_t ax = 0, ay = 0, bx = 0, by = 0;
  const cudaArray_t arr_a = image_array(a, &la, &ax, &ay), arr_b = image_array(b, &lb, &bx, &by);
  // a whole 2-D array (layer -1) and a rectangle of it (layer 0) are one layer
  if (arr_a != arr_b || std::max(la, 0) != std::max(lb, 0)) return false;
  if (a->memory != GS_MEM_ARRAY_RECT || b->memory != GS_MEM_ARRAY_RECT) return true;
  return (uint64_t)ax < (uint64_t)bx + b->width && (uint64_t)bx < (uint64_t)ax + a->width &&
         (uint64_t)ay < (uint64_t)by + b->height && (uint64_t)by < (uint64_t)ay + a->height;
}

// Destroys the held surface objects whose last use has completed; with `all`, every one, after waiting for its event.  The
// event, not the context stream, is what guards a batch: the group path composites onto CUDA-array camera targets on a
// member's transfer stream, which the context stream never waits for.
void release_surfaces(GsContext *ctx, bool all) {
  auto &held = ctx->held_surfaces;
  size_t keep = 0;
  for (size_t i = 0; i < held.size(); ++i) {
    bool done = all;
    if (all) {
      if (cudaEventSynchronize(held[i].done) != cudaSuccess) cudaGetLastError();   // failed: nothing will use the surfaces any more
    } else {
      const cudaError_t q = cudaEventQuery(held[i].done);
      done = q != cudaErrorNotReady;   // completed, or failed: either way nothing will use the surfaces any more
      if (!done && cudaPeekAtLastError() == cudaErrorNotReady) cudaGetLastError();
    }
    if (done) {
      for (cudaSurfaceObject_t so : held[i].surfs) cudaDestroySurfaceObject(so);
      ctx->spare_events.push_back(held[i].done);
    } else {
      if (keep != i) held[keep] = std::move(held[i]);
      ++keep;
    }
  }
  held.resize(keep);
}

int bind_image(GsContext *ctx, CallSurfaces &surfs, const GsImage *im, uint32_t pitch, uint32_t fmt, uint32_t W, uint32_t H, void *staging,
               StagingFill fill, cudaStream_t s, DeviceImage *out) {
  *out = DeviceImage{};
  if (im && im->memory == GS_MEM_DEVICE) { out->d_rt = im->data; out->pitch = pitch; return GS_OK; }
  if (im && is_array_image(im)) return surfs.make(im, &out->surf);
  out->d_rt = staging;
  out->pitch = W * pix_bytes(fmt);
  if (fill == StagingFill::kUpload)
    GS_CUDA_TRY(ctx, cudaMemcpy2DAsync(staging, out->pitch, im->data, pitch, out->pitch, H, cudaMemcpyHostToDevice, s));
  else if (fill == StagingFill::kZero)
    GS_CUDA_TRY(ctx, cudaMemsetAsync(staging, 0, (size_t)out->pitch * H, s));
  return GS_OK;
}

int copy_to_image(GsContext *ctx, const GsImage *im, uint32_t pitch, const void *src, uint32_t src_pitch, uint32_t W, uint32_t H,
                  cudaStream_t s) {
  const size_t row = (size_t)W * pix_bytes(im->format);
  if (is_array_image(im)) {
    int32_t layer = -1;
    uint32_t x = 0, y = 0;
    const cudaArray_t arr = image_array(im, &layer, &x, &y);
    if (im->memory == GS_MEM_ARRAY || (im->memory == GS_MEM_ARRAY_RECT && !array_layered(arr))) {
      // wOffset is in bytes
      GS_CUDA_TRY(ctx, cudaMemcpy2DToArrayAsync(arr, (size_t)x * pix_bytes(im->format), y, src, src_pitch, row, H, cudaMemcpyDeviceToDevice, s));
    } else {
      cudaMemcpy3DParms cp;
      memset(&cp, 0, sizeof(cp));
      cp.srcPtr = make_cudaPitchedPtr(const_cast<void *>(src), src_pitch, W, H);
      cp.dstArray = arr;
      cp.dstPos = make_cudaPos(x, y, (size_t)(uint32_t)layer);   // in texels: the destination is an array
      cp.extent = make_cudaExtent(W, H, 1);
      cp.kind = cudaMemcpyDeviceToDevice;
      GS_CUDA_TRY(ctx, cudaMemcpy3DAsync(&cp, s));
    }
  } else {
    const cudaMemcpyKind kind = im->memory == GS_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    GS_CUDA_TRY(ctx, cudaMemcpy2DAsync(im->data, pitch, src, src_pitch, row, H, kind, s));
  }
  return GS_OK;
}

int depth_ok(GsContext *ctx, const GsFrameParams *fp) {
  if (!depth_in_array(fp)) return GS_OK;
  return array_ok(ctx, depth_view(fp), (uint32_t)fp->screen_w, (uint32_t)fp->screen_h, cudaChannelFormatKindFloat, 1, 32, "scene depth: ",
                  "the screen's", "one 32-bit float channel");
}

std::tuple<const void *, int32_t, uint32_t, uint32_t, uint32_t> depth_id(const GsFrameParams *fp) {
  if (!fp->scene_depth) return {nullptr, -1, 0, 0, 0};
  if (fp->scene_depth_on_device == GS_MEM_ARRAY_LAYER) {
    const GsArrayLayer *d = reinterpret_cast<const GsArrayLayer *>(fp->scene_depth);
    return {d->array, (int32_t)d->layer, GS_MEM_ARRAY_LAYER, 0, 0};
  }
  if (fp->scene_depth_on_device == GS_MEM_ARRAY_RECT) {
    const GsArrayRect *d = reinterpret_cast<const GsArrayRect *>(fp->scene_depth);
    return {d->array, (int32_t)d->layer, GS_MEM_ARRAY_RECT, d->x, d->y};
  }
  return {fp->scene_depth, -1, fp->scene_depth_on_device, 0, 0};
}

int bind_depth(GsContext *ctx, CallSurfaces *surfs, const GsFrameParams *fp, float *staging, cudaStream_t s, SceneDepth *out) {
  *out = SceneDepth{};
  if (!fp->scene_depth) return GS_OK;
  if (depth_in_array(fp)) {
    if (!surfs) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "a scene depth buffer in a CUDA array needs the call's surfaces");
    const GsImage a = depth_view(fp);
    out->on_surface = true;
    return surfs->make(&a, &out->surf);
  }
  if (!depth_on_host(fp)) { out->ptr = fp->scene_depth; return GS_OK; }
  const size_t pixels = (size_t)(uint32_t)fp->screen_w * (uint32_t)fp->screen_h;
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(staging, fp->scene_depth, pixels * sizeof(float), cudaMemcpyHostToDevice, s));
  out->ptr = staging;
  return GS_OK;
}

}  // namespace gs
