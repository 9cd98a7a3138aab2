// gs_internal.cuh -- what gs_api.cu (single GPU) and gs_group.cu (several GPUs) share behind the C ABI:
// the context / asset objects and the per-stage drivers.
#pragma once
#include <algorithm>
#include <atomic>
#include <cstring>
#include <string>
#include <tuple>
#include <vector>

#include <nvtx3/nvToolsExt.h>   // header-only; costs one predicted-not-taken branch per range when no tool is attached

#include "gs_buffer.cuh"
#include "gs_kernels.cuh"

// Host-side ranges named as the reference's profiler markers (R/GaussianSplatRenderer.cs:20-22,287): an Nsight timeline of a
// host using this library shows GaussianSplat.Sort / CalcView / Draw / Compose like Unity's profiler does.
struct GsNvtxRange {
  explicit GsNvtxRange(const char *name) { nvtxRangePushA(name); }
  ~GsNvtxRange() { nvtxRangePop(); }
  GsNvtxRange(const GsNvtxRange &) = delete;
  GsNvtxRange &operator=(const GsNvtxRange &) = delete;
};

struct GsContext;
namespace gs {
class CallSurfaces;
int fail(GsContext *ctx, int code, const std::string &msg);
int fail_cuda(GsContext *ctx, cudaError_t e, const char *expr, const char *file, int line);

// The bin list (DESIGN §2, "Overflow across a call"), entry_count = [entries within the capacity, overflow flag, total]: its rules
// inline, its buffers and CUDA calls in gs_bins.cu.  A call starts with begin_call; each draw is begin_draw, builds, end_draw.
constexpr uint32_t kBinListMax = 768u << 20;
constexpr uint32_t kRuleBins = 128;   // the capacity rule was set for screens of at most this many bins per axis (8160 px)
class BinList {
 public:
  static uint32_t capacity_for(uint32_t splats) {
    return (uint32_t)std::min<uint64_t>(std::max<uint64_t>((uint64_t)splats * 8, 4u << 20), kBinListMax);
  }
  void begin_call() { flag_ = kFirst; }
  bool clears() const { return flag_ == kFirst; }   // the draw's first build
  // One camera above kRuleBins bins on an axis reads back and may rebuild: it first reads the flag the last draw did not read.
  int begin_draw(GsContext *ctx, uint32_t cameras, const FrameConsts &fc) {
    reads_ = cameras == 1 && (fc.binsX > kRuleBins || fc.binsY > kRuleBins);
    if (!reads_ || flag_ != kUnknown) return GS_OK;
    uint32_t ec[2] = {0, 0};
    GS_CUDA_TRY(ctx, read(ctx, ec, 2));
    flag_ = ec[1] ? kSet : kClear;
    return GS_OK;
  }
  // After the first build, an overflowed list grows to its total + 1/4, at most kBinListMax, and *again asks to rebuild it with
  // *clear: the grown list fits, so only a truncated earlier draw of the call keeps the flag set.
  int end_draw(GsContext *ctx, uint32_t n, uint32_t bins, bool *again, bool *clear) {
    uint32_t ec[3] = {0, 0, 0};   // clamped count, overflow flag, total (of this run, for gs_frame_objects)
    if (reads_) GS_CUDA_TRY(ctx, read(ctx, ec, 3));
    *again = reads_ && ec[2] > capacity() && ec[2] <= kBinListMax;
    *clear = flag_ != kSet;
    if (!reads_) flag_ = kUnknown;
    else flag_ = (*again ? *clear : ec[1] == 0) ? kClear : kSet;
    return *again ? reserve(ctx, n, bins, (uint32_t)std::min<uint64_t>((uint64_t)ec[2] + ec[2] / 4, kBinListMax)) : GS_OK;
  }
  int reserve(GsContext *ctx, uint32_t n, uint32_t bins, uint32_t min_capacity = 0);   // with the bin sort's sort scratch
  cudaError_t read(GsContext *ctx, uint32_t *ec, uint32_t words);   // entry_count[0, words), once the stream is done
  uint32_t capacity() const;   // the smaller buffer: after a failed growth one of them may still hold the larger, older size
  int check(GsContext *ctx);   // at a host sync point: ctx->times.tile_entries, and GS_ERR_OUT_OF_MEMORY for a truncated list
  Buffer<uint32_t> keys, vals, block_sums, entry_count;   // launchers take the view bin_scratch(ctx)
  Buffer<uint2> ranges;

 private:
  enum { kFirst, kClear, kSet, kUnknown } flag_ = kFirst;   // the flag as the host knows it (kFirst: the next build clears it)
  bool reads_ = false;   // the current draw reads its list back
};
}  // namespace gs

enum { EV_BEGIN = 0, EV_DIST, EV_SORT0, EV_SORT1, EV_SORT2, EV_SORT3, EV_SORT4, EV_VIEW0, EV_VIEW1, EV_BIN1, EV_RASTER1, EV_COMP1, EV_COUNT };

struct GsContext {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  std::string err;
  bool timing = false;
  GsStageTimes times{};
  cudaEvent_t ev[EV_COUNT]{};
  bool ev_valid[EV_COUNT]{};
  // sort scratch (launchers take the view sort_scratch(ctx))
  gs::Buffer<uint32_t> sort_alt_keys, sort_alt_vals;   // ping-pong buffers, as many elements as the largest sort so far
  gs::Buffer<uint32_t> sort_ghist, sort_lookback, sort_tickets;
  gs::Buffer<uint32_t> d_scalar;  // small device scalars (standalone sorter count)
  gs::BinList bins;
  gs::Buffer<uint32_t> tile_cost, tile_order;   // the single-grid raster-tile history, and the launch order of every draw
  uint32_t raster_tiles_cur = 0;   // the tile count tile_cost's history was kept for
  // gs_frame_cameras: the tile-cost histories of the camera layouts seen ((raster tiles per row, rows) per camera of a run,
  // each history at its base in cams_tile_cost), the digit histograms of a camera run's bin list (the depth sorts between its
  // emits use sort_ghist), and one scratch buffer for a run's record slabs, staging images and host depth buffers
  std::vector<std::vector<uint32_t>> cams_layouts;
  std::vector<size_t> cams_layout_base;
  gs::Buffer<uint32_t> cams_tile_cost;
  size_t cams_cost_used = 0;
  gs::Buffer<uint32_t> cams_ghist;
  gs::Buffer<uint8_t> cams_scratch;
  // image scratch
  gs::Buffer<uint8_t> rt_scratch, tgt_scratch;
  // asynchronous read-back (GS_FLAG_ASYNC_READBACK): two device staging images, a copy stream, and the events that order
  // "raster k -> copy k" and "copy k -> raster k+2 may reuse the staging image"
  cudaStream_t copy_stream = nullptr;
  gs::Buffer<uint8_t> rt_async[2];
  cudaEvent_t ev_rt_ready[2]{}, ev_copy_done[2]{};
  bool copy_pending[2] = {false, false};
  int rt_flip = 0;
  // per-frame optional inputs
  gs::Buffer<GsCutout> d_cutouts;
  gs::Buffer<uint32_t> d_deleted, d_selected;
  gs::Buffer<float> d_depth;   // the frame's scene depth buffer when it was handed over in host memory
  uint32_t launches = 0;
  uint64_t pack_stats[4] = {0, 0, 0, 0};   // gs_debug_pack_stats
  // surface objects of GS_MEM_ARRAY / GS_MEM_ARRAY_LAYER images, one per array per call: each batch is destroyed once `done` (recorded behind the
  // call's last use on `stream`) has completed, or at gs_sync / gs_destroy
  struct HeldSurfaces {
    cudaEvent_t done;
    std::vector<cudaSurfaceObject_t> surfs;
  };
  std::vector<HeldSurfaces> held_surfaces;
  std::vector<cudaEvent_t> spare_events;
};

// The five blobs of an asset in HBM, 16 bytes of slack each.  Nothing writes them after gs_asset_upload / gs_pack_asset, so an
// asset and its instances (gs_asset_instance), all on one context, hold one GsBlobs; the last of them to be destroyed frees it.
struct GsBlobs {
  gs::Buffer<uint8_t> pos, other, sh, color, chunks;
  std::atomic<uint32_t> refs{1};   // the assets holding it
};

// Its buffers are freed by gs_asset_destroy, with the context's device current and its stream drained; so is its GsBlobs when
// no other asset holds it.
struct GsAsset {
  GsContext *ctx = nullptr;
  gs::AssetView av{};
  GsBlobs *blobs = nullptr;   // av points into them
  gs::Buffer<uint32_t> order, keys, key_table, view, rect, d_n;
  gs::Buffer<uint32_t> block_bits;  // bit j: some splat of block j (256 splats) got a bin rectangle from the last view-calc
  // group path only (allocated by gs_group_*): slab membership (bit per splat, byte per 128), compaction output / sort ping-pong payload
  gs::Buffer<uint32_t> slab_mask, order_tmp;
  gs::Buffer<float> zndc;           // per-splat quad depth clip.z / clip.w, written by view-calc when a scene depth buffer is bound
  bool zndc_valid = false;
  gs::Buffer<uint32_t> order_alt;   // peer-to-peer order exchange: `order` and `order_alt` alternate as last / new draw order
  gs::Buffer<uint32_t> slab_group_bits;
  gs::Buffer<float4> draw;  // raster-ready 48-byte records of the drawable splats (3 float4 each)
  bool view_valid = false;   // the full 40-byte _SplatViewData buffer is current (gs_calc_view)
  bool draw_valid = false;   // draw records + bin rects are current (gs_calc_view or gs_frame)
  uint32_t draw_part[3] = {0, 0, 1};   // the tile partition those records were culled for (count <= 1: complete)
  uint32_t view_w = 0, view_h = 0;

  GsAsset() = default;
  GsAsset(const GsAsset &) = delete;
  GsAsset &operator=(const GsAsset &) = delete;
  ~GsAsset() {
    if (blobs && blobs->refs.fetch_sub(1) == 1) delete blobs;
  }
};

namespace gs {
// The launchers' views of the context's scratch.
inline SortScratch sort_scratch(const GsContext *ctx) {
  return {ctx->sort_alt_keys.get(), ctx->sort_alt_vals.get(), ctx->sort_ghist.get(), ctx->sort_lookback.get(), ctx->sort_tickets.get(),
          ctx->sort_lookback.size()};
}
inline BinScratch bin_scratch(const GsContext *ctx) {
  return {ctx->bins.block_sums.get(), ctx->bins.entry_count.get(), ctx->bins.keys.get(), ctx->bins.vals.get(),
          reinterpret_cast<uint32_t *>(ctx->bins.ranges.get()), ctx->tile_cost.get(), ctx->tile_order.get(), ctx->bins.capacity()};
}
FrameConsts make_frame_consts(const GsFrameParams *fp);
int check_params(GsContext *ctx, GsAsset *as, const GsFrameParams *fp);
int check_options(GsContext *ctx, const FrameConsts &fc, GsRenderOptions &opt);
int ensure_sort_scratch(GsContext *ctx, uint32_t capacity);
// Grows the context's cutout / deleted / selected buffers to what fp needs for `as`; `users`: the streams whose view-calcs may
// still read them (Buffer::reserve).  Uploads nothing.
int reserve_frame_inputs(GsContext *ctx, GsAsset *as, const GsFrameParams *fp, std::initializer_list<cudaStream_t> users);
int upload_frame_inputs(GsContext *ctx, GsAsset *as, const GsFrameParams *fp, cudaStream_t stream);
// draw / zndc (optional): where the raster records and quad depths go instead of the asset's own buffers (gs_frame_cameras'
// record slabs); the asset's draw state is then left as it was.  after_sort: the last thing on `stream` is do_sort of `as`
// (launch_calc_view)
int do_view(GsContext *ctx, GsAsset *as, const GsFrameParams *fp, const FrameConsts &fc, bool cull, const GsRenderOptions &opt,
            cudaStream_t stream, float4 *draw = nullptr, float *zndc = nullptr, bool after_sort = false);
// Bins and rasterizes one object `as`, drawn with the uniforms *fp, into a device image (d_rt == nullptr: the CUDA array behind
// `surf`) on ctx->stream with gs_frame's kernels; its scene depth buffer is bound here, a CUDA array through `surfs` (nullptr:
// the caller takes no CUDA-array depth).  A run of several objects or cameras is gs_api.cu's draw_run.  bin_done (optional) is
// recorded on ctx->stream when binning ends.
int do_draw(GsContext *ctx, CallSurfaces *surfs, const FrameConsts &fc, const GsRenderOptions &opt, GsAsset *as, const GsFrameParams *fp,
            void *d_rt, uint32_t pitch, uint32_t fmt, Surface surf = Surface{}, cudaEvent_t bin_done = nullptr);
// The composite pass (gs_composite) of a linear device render target onto `tgt` (host, device or CUDA-array memory, already
// validated as W x H), enqueued on `s`.  A host target is uploaded and read back, and the call waits for `s`.
int composite_device_rt(GsContext *ctx, const void *d_rt, uint32_t rt_pitch, uint32_t rt_fmt, GsImage *tgt, uint32_t W, uint32_t H,
                        cudaStream_t s);

// ---- images (gs_image.cu) -------------------------------------------------------------------------------------------------
// What an image is to the call: a render target (also gs_composite's source, band_packed and gs_unshuffle_bands output), which
// is RGBA16F or RGBA32F, or a camera target, which may also be GS_PIX_B10G11R11_UFLOAT or GS_PIX_R8G8B8A8_SRGB.
enum class ImageRole { kRenderTarget, kCameraTarget };
int image_ok(GsContext *ctx, const GsImage *im, uint32_t W, uint32_t H, ImageRole role, uint32_t *pitch);
uint32_t pix_bytes(uint32_t fmt);
inline bool is_array_image(const GsImage *im) {
  return im->memory == GS_MEM_ARRAY || im->memory == GS_MEM_ARRAY_LAYER || im->memory == GS_MEM_ARRAY_RECT;
}
// The CUDA array of a GS_MEM_ARRAY / GS_MEM_ARRAY_LAYER / GS_MEM_ARRAY_RECT image, in *layer the layer it names (-1: a whole
// 2-D array; a GS_MEM_ARRAY_RECT image names its descriptor's layer, 0 on a 2-D array), and in *x / *y (optional) the texel
// that holds its pixel (0, 0).
inline cudaArray_t image_array(const GsImage *im, int32_t *layer, uint32_t *x = nullptr, uint32_t *y = nullptr) {
  uint32_t ox = 0, oy = 0;
  cudaArray_t arr = static_cast<cudaArray_t>(im->data);
  *layer = -1;
  if (im->memory == GS_MEM_ARRAY_LAYER) {
    const GsArrayLayer *d = static_cast<const GsArrayLayer *>(im->data);
    *layer = (int32_t)d->layer;
    arr = static_cast<cudaArray_t>(d->array);
  } else if (im->memory == GS_MEM_ARRAY_RECT) {
    const GsArrayRect *d = static_cast<const GsArrayRect *>(im->data);
    *layer = (int32_t)d->layer;
    ox = d->x; oy = d->y;
    arr = static_cast<cudaArray_t>(d->array);
  }
  if (x) *x = ox;
  if (y) *y = oy;
  return arr;
}
// Whether `arr` (a valid CUDA array) is a layered one, as cudaArrayGetInfo reports it.
bool array_layered(cudaArray_t arr);
// Whether two images of a call share pixels: linear images by pointer; CUDA-array images when they name the same array and
// layer and their rectangles intersect (a whole array or layer intersects every rectangle of it; the layers of one array are
// separate images).  A null image shares nothing.
bool images_overlap(const GsImage *a, const GsImage *b);
void release_surfaces(GsContext *ctx, bool all);

// The surface objects one call creates for its CUDA-array images, one per array: the layers and rectangles of one array share
// it, and each image's Surface carries its own layer and origin.  When the call returns they are handed to the context behind an event recorded on the stream that used them (the context's,
// unless another is named) after their last use.  They are never cached by cudaArray_t value beyond the call: a freed array's
// handle can be reused by the next allocation.
class CallSurfaces {
 public:
  explicit CallSurfaces(GsContext *ctx, cudaStream_t stream = nullptr) : ctx_(ctx), stream_(stream ? stream : ctx->stream) {}
  CallSurfaces(const CallSurfaces &) = delete;
  CallSurfaces &operator=(const CallSurfaces &) = delete;
  ~CallSurfaces() {
    if (made_.empty()) return;
    cudaEvent_t ev = nullptr;
    if (!ctx_->spare_events.empty()) { ev = ctx_->spare_events.back(); ctx_->spare_events.pop_back(); }
    else if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) ev = nullptr;
    if (ev && cudaEventRecord(ev, stream_) == cudaSuccess) {
      ctx_->held_surfaces.push_back({ev, std::move(made_)});
      return;
    }
    cudaStreamSynchronize(stream_);   // no event to wait for: wait for the stream itself
    for (cudaSurfaceObject_t so : made_) cudaDestroySurfaceObject(so);
    if (ev) ctx_->spare_events.push_back(ev);
  }
  // `im` has passed image_ok as a GS_MEM_ARRAY, GS_MEM_ARRAY_LAYER or GS_MEM_ARRAY_RECT image
  int make(const GsImage *im, Surface *out) {
    const cudaArray_t arr = image_array(im, &out->layer, &out->x, &out->y);
    size_t i = 0;
    while (i < arrays_.size() && arrays_[i] != arr) ++i;
    if (i == arrays_.size()) {
      if (made_.empty()) release_surfaces(ctx_, false);
      cudaResourceDesc rd;
      memset(&rd, 0, sizeof(rd));
      rd.resType = cudaResourceTypeArray;
      rd.res.array.array = arr;
      cudaSurfaceObject_t so = 0;
      GS_CUDA_TRY(ctx_, cudaCreateSurfaceObject(&so, &rd));
      made_.push_back(so);
      arrays_.push_back(arr);
      layered_.push_back(im->memory == GS_MEM_ARRAY_LAYER || (im->memory == GS_MEM_ARRAY_RECT && array_layered(arr)));
    }
    out->obj = made_[i];
    if (!layered_[i]) out->layer = -1;   // a rectangle of a 2-D array is drawn with the 2-D surface calls
    return GS_OK;
  }

 private:
  GsContext *ctx_;
  cudaStream_t stream_;
  std::vector<cudaSurfaceObject_t> made_;
  std::vector<cudaArray_t> arrays_;   // made_[i] is the surface of arrays_[i]
  std::vector<bool> layered_;         // arrays_[i] is a layered array
};

// The device view of an image a kernel reads and writes: linear memory at d_rt / pitch, or (d_rt == nullptr) the CUDA array
// (layer) behind `surf`.
struct DeviceImage {
  void *d_rt = nullptr;
  uint32_t pitch = 0;
  Surface surf;
};
// What a staging image holds before the kernel runs: the host image's pixels, zeros, or whatever it held.
enum class StagingFill { kUpload, kZero, kNone };
// The device view of `im` (passed image_ok with `pitch`), on `s`: device memory is the image itself, a CUDA array (layer) a
// surface made through `surfs`.  A host image, or none (im == nullptr, whose fill must not be kUpload), is the tight W x H
// image of pixel format `fmt` at `staging`, which the caller has grown, filled as `fill` says.
int bind_image(GsContext *ctx, CallSurfaces &surfs, const GsImage *im, uint32_t pitch, uint32_t fmt, uint32_t W, uint32_t H, void *staging,
               StagingFill fill, cudaStream_t s, DeviceImage *out);
// Copies W x H pixels of linear device memory (src / src_pitch) into `im` (passed image_ok with `pitch`), of any memory kind,
// on `s`.
int copy_to_image(GsContext *ctx, const GsImage *im, uint32_t pitch, const void *src, uint32_t src_pitch, uint32_t W, uint32_t H,
                  cudaStream_t s);

// ---- the scene depth buffer (gs_image.cu) --------------------------------------------------------------------------------
// GsFrameParams.scene_depth_on_device is the GsMemory of scene_depth: 0 host memory, GS_MEM_ARRAY a 2-D float32 CUDA array,
// GS_MEM_ARRAY_LAYER a GsArrayLayer naming a layer of a layered one, GS_MEM_ARRAY_RECT a GsArrayRect naming a rectangle of
// either, any other value linear device memory.
inline bool depth_on_host(const GsFrameParams *fp) { return fp->scene_depth && fp->scene_depth_on_device == GS_MEM_HOST; }
inline bool depth_in_array(const GsFrameParams *fp) {
  return fp->scene_depth && (fp->scene_depth_on_device == GS_MEM_ARRAY || fp->scene_depth_on_device == GS_MEM_ARRAY_LAYER ||
                             fp->scene_depth_on_device == GS_MEM_ARRAY_RECT);
}
// The array (layer, rectangle) of a depth_in_array buffer as an image view (data and memory), as image_array and CallSurfaces
// take it.
inline GsImage depth_view(const GsFrameParams *fp) {
  GsImage a{};
  a.data = const_cast<float *>(fp->scene_depth);
  a.memory = fp->scene_depth_on_device;
  return a;
}
// A CUDA-array depth buffer must be a screen_w x screen_h array (layer), or a rectangle of that size inside one, of one 32-bit
// float channel made with cudaArraySurfaceLoadStore: GS_ERR_UNSUPPORTED_FORMAT for another channel format,
// GS_ERR_INVALID_ARGUMENT for anything else.
int depth_ok(GsContext *ctx, const GsFrameParams *fp);
// What makes two objects' depth buffers one buffer: the same pointer and memory kind, or the same array, layer and origin
// (GS_MEM_ARRAY_LAYER / GS_MEM_ARRAY_RECT: two descriptors of one layer and rectangle are one buffer, the layers of one array
// and its other rectangles are not).  (nullptr, ...): none.
std::tuple<const void *, int32_t, uint32_t, uint32_t, uint32_t> depth_id(const GsFrameParams *fp);
// The kernels' view of fp's depth buffer (passed depth_ok), on `s`: device memory in place, a CUDA array (layer) through a
// surface made by `surfs` (nullptr: none may be made, and a CUDA array is GS_ERR_INVALID_ARGUMENT), or a host buffer uploaded
// into `staging`, W x H floats that the caller has grown.
int bind_depth(GsContext *ctx, CallSurfaces *surfs, const GsFrameParams *fp, float *staging, cudaStream_t s, SceneDepth *out);
// The per-asset work buffers (order, keys, view data, ...) of an asset whose blobs as->blobs are already in HBM, the format
// fields of as->av, and CSSetIndices: what gs_asset_upload, gs_pack_asset and gs_asset_instance share.
cudaError_t asset_init_work(GsContext *ctx, GsAsset *as, uint32_t n, uint32_t pos_fmt, uint32_t scale_fmt, uint32_t sh_fmt,
                            uint32_t col_fmt, uint32_t chunk_count);
void rec(GsContext *ctx, int e);
// The render-thread events of the group calls (gs_group.cu), which gs_api.cu's event callback dispatches to: each runs its
// entry point on the payload and stores the GsStatus in the payload's `status`.
void unity_group_frame_objects_event(GsUnityGroupFrameObjectsEvent *ev);
void unity_group_sync_event(GsUnityGroupSyncEvent *ev);
void launch_row_costs(const uint32_t *cost, uint32_t ntx, uint32_t t0, uint32_t t1, uint32_t *row_cost, cudaStream_t s,
                      bool accumulate = false);   // gs_raster.cu
}  // namespace gs
