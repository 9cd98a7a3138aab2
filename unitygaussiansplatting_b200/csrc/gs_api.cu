// gs_api.cu -- the C ABI of libgsplat_b200.so (include/gsplat_b200.h): context, asset
// residency in HBM, per-frame uniform derivation and stage sequencing on one CUDA stream.
//
// This file is the native counterpart of the C# frame driver: CreateResourcesForAsset /
// InitSortBuffers (R/GaussianSplatRenderer.cs:373-445), CalcViewData (:579-610), SortPoints
// (:612-639) and SortAndRenderSplats (:108-169).  There is no CPU fallback anywhere: without
// a CUDA device gs_create fails with GS_ERR_NO_DEVICE.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>

#include "gs_internal.cuh"

namespace gs {
static thread_local std::string g_last_error;
}  // namespace gs

namespace gs {

int fail(GsContext *ctx, int code, const std::string &msg) {
  g_last_error = msg;
  if (ctx) ctx->err = msg;
  return code;
}
int fail_cuda(GsContext *ctx, cudaError_t e, const char *expr, const char *file, int line) {
  char buf[512];
  snprintf(buf, sizeof(buf), "CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, expr);
  return fail(ctx, e == cudaErrorMemoryAllocation ? GS_ERR_OUT_OF_MEMORY : GS_ERR_CUDA, buf);
}

#define M_(m, r, c) ((m)[(c)*4 + (r)])
// Matrix4x4 operator* as Unity evaluates it (plain float ops, no contraction: this TU is
// compiled with -Xcompiler -ffp-contract=off).
static void mat_mul(const float *a, const float *b, float *o) {
  for (int c = 0; c < 4; ++c)
    for (int r = 0; r < 4; ++r)
      M_(o, r, c) = M_(a, r, 0) * M_(b, 0, c) + M_(a, r, 1) * M_(b, 1, c) + M_(a, r, 2) * M_(b, 2, c) + M_(a, r, 3) * M_(b, 3, c);
}

// Uniform derivation of CalcViewData (R/GaussianSplatRenderer.cs:586-606) and SortPoints (:617-629),
// plus the CalcCovariance2D constants that depend only on the camera (S/GaussianSplatting.hlsl:62-70).
FrameConsts make_frame_consts(const GsFrameParams *fp) {
  FrameConsts fc;
  memset(&fc, 0, sizeof(fc));
  float mv[16], vp[16], w2c[16], mvs[16];
  mat_mul(fp->mat_view, fp->mat_object_to_world, mv);
  mat_mul(fp->mat_proj_gpu, fp->mat_view, vp);
  memcpy(w2c, fp->mat_view, 64);
  M_(w2c, 2, 0) *= -1.0f; M_(w2c, 2, 1) *= -1.0f; M_(w2c, 2, 2) *= -1.0f;
  mat_mul(w2c, fp->mat_object_to_world, mvs);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) {
      fc.o2w[r * 4 + c] = M_(fp->mat_object_to_world, r, c);
      fc.mv[r * 4 + c] = M_(mv, r, c);
    }
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) fc.w2o[r * 3 + c] = M_(fp->mat_world_to_object, r, c);
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) fc.vp[r * 4 + c] = M_(vp, r, c);
  for (int c = 0; c < 4; ++c) fc.sort_row[c] = M_(mvs, 2, c);
  for (int k = 0; k < 3; ++k) fc.cam_pos[k] = fp->cam_pos_world[k];
  const float p00 = M_(fp->mat_proj_gpu, 0, 0), p11 = M_(fp->mat_proj_gpu, 1, 1);
  const float aspect = p00 / p11;
  const float tanFovX = 1.0f / p00;
  const float tanFovY = 1.0f / (p11 * aspect);  // == tanFovX: reference quirk, kept
  fc.limX = 1.3f * tanFovX;
  fc.limY = 1.3f * tanFovY;
  fc.focal = fp->screen_w * p00 / 2.0f;
  fc.splatScale2 = fp->splat_scale * fp->splat_scale;
  fc.opacityScale = fp->opacity_scale;
  {
    // Bound behind the fused kernel's cheap culls.  CalcCovariance2D (S/GaussianSplatting.hlsl:56-90): cov2d = T S T^t + 0.3 I with
    // T = J W, J = (focal/tz) [I2 | -u], |u|^2 <= limX^2 + limY^2 (the clamp), W = MV 3x3, S = R diag(s^2) R^t splatScale^2.
    // So lambda1 <= |J|_2^2 |W|_2^2 smax^2 splatScale^2 + 0.3 with |J|_2^2 = (focal/tz)^2 (1 + |u|^2); the quad reaches at most
    // 2 (|a1x| + |a2x|) <= 2 sqrt(2) sqrt(2 lambda1) pixels from its centre.  |W|_2^2 is bounded by the smaller of the Frobenius
    // norm and the Gershgorin bound of W^t W (exact for rotation x uniform scale, the usual transform).
    double a[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, fro = 0.0;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        for (int k = 0; k < 3; ++k) a[i][j] += (double)M_(mv, k, i) * (double)M_(mv, k, j);
        fro += (double)M_(mv, i, j) * (double)M_(mv, i, j);
      }
    double gersh = 0.0;
    for (int i = 0; i < 3; ++i) {
      double row = 0.0;
      for (int j = 0; j < 3; ++j) row += a[i][j] < 0 ? -a[i][j] : a[i][j];
      if (row > gersh) gersh = row;
    }
    const double w2 = (gersh < fro ? gersh : fro) * 1.0001;
    fc.extentK = (float)((double)fc.focal * fc.focal * (1.0 + (double)fc.limX * fc.limX + (double)fc.limY * fc.limY) * w2 * fc.splatScale2);
  }
  fc.screenW = fp->screen_w;
  fc.screenH = fp->screen_h;
  fc.shOrder = fp->sh_order;
  fc.shOnly = fp->sh_only;
  fc.cutoutCount = fp->cutouts ? fp->cutout_count : 0;
  fc.bitsValid = fp->deleted_bits ? 1u : 0u;
  fc.selValid = fp->selected_bits ? 1u : 0u;
  fc.binsX = ((uint32_t)fp->screen_w + kBin - 1) / kBin;
  fc.binsY = ((uint32_t)fp->screen_h + kBin - 1) / kBin;
  return fc;
}

int ensure_sort_scratch(GsContext *ctx, uint32_t capacity) {
  GS_CUDA_TRY(ctx, ctx->sort_alt_keys.reserve(capacity, {ctx->stream}));
  GS_CUDA_TRY(ctx, ctx->sort_alt_vals.reserve(capacity, {ctx->stream}));
  GS_CUDA_TRY(ctx, ctx->sort_lookback.reserve(sort_lookback_words(capacity, 4), {ctx->stream}));
  return GS_OK;
}

void rec(GsContext *ctx, int e) {
  if (ctx->timing) { cudaEventRecord(ctx->ev[e], ctx->stream); ctx->ev_valid[e] = true; }
}
static float ev_ms(GsContext *ctx, int a, int b) {
  if (!ctx->ev_valid[a] || !ctx->ev_valid[b]) return 0.0f;
  float ms = 0.0f;
  if (cudaEventElapsedTime(&ms, ctx->ev[a], ctx->ev[b]) != cudaSuccess) { cudaGetLastError(); return 0.0f; }
  return ms;
}

// GS_FLAG_ASYNC_READBACK plumbing, created on first use
static int ensure_async_readback(GsContext *ctx) {
  if (ctx->copy_stream) return GS_OK;
  GS_CUDA_TRY(ctx, cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
  for (int i = 0; i < 2; ++i) {
    GS_CUDA_TRY(ctx, cudaEventCreateWithFlags(&ctx->ev_rt_ready[i], cudaEventDisableTiming));
    GS_CUDA_TRY(ctx, cudaEventCreateWithFlags(&ctx->ev_copy_done[i], cudaEventDisableTiming));
  }
  return GS_OK;
}

int reserve_frame_inputs(GsContext *ctx, GsAsset *as, const GsFrameParams *fp, std::initializer_list<cudaStream_t> users) {
  if (fp->cutouts && fp->cutout_count) GS_CUDA_TRY(ctx, ctx->d_cutouts.reserve(fp->cutout_count, users));
  const size_t words = ((size_t)as->av.n + 31) / 32;
  if (fp->deleted_bits) GS_CUDA_TRY(ctx, ctx->d_deleted.reserve(words, users));
  if (fp->selected_bits) GS_CUDA_TRY(ctx, ctx->d_selected.reserve(words, users));
  return GS_OK;
}

int upload_frame_inputs(GsContext *ctx, GsAsset *as, const GsFrameParams *fp, cudaStream_t stream) {
  int rc = reserve_frame_inputs(ctx, as, fp, {ctx->stream});
  if (rc) return rc;
  const size_t words = ((size_t)as->av.n + 31) / 32;
  if (fp->cutouts && fp->cutout_count)
    GS_CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_cutouts.get(), fp->cutouts, sizeof(GsCutout) * fp->cutout_count, cudaMemcpyHostToDevice, stream));
  if (fp->deleted_bits) GS_CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_deleted.get(), fp->deleted_bits, words * 4, cudaMemcpyHostToDevice, stream));
  if (fp->selected_bits) GS_CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_selected.get(), fp->selected_bits, words * 4, cudaMemcpyHostToDevice, stream));
  return GS_OK;
}

int check_params(GsContext *ctx, GsAsset *as, const GsFrameParams *fp) {
  if (!ctx || !as || !fp) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null context/asset/params");
  if (as->ctx != ctx) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "asset belongs to another context");
  GS_CUDA_TRY(ctx, cudaSetDevice(ctx->device));   // the caller's current device may be another one
  if (!(fp->screen_w >= 1.0f) || !(fp->screen_h >= 1.0f) || fp->screen_w > 16384.0f || fp->screen_h > 16384.0f)
    return fail(ctx, GS_ERR_INVALID_ARGUMENT, "screen size must be in [1,16384] (8-bit indices of 64-pixel bins)");
  if (fp->sh_order > 3) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "sh_order must be 0..3");
  return depth_ok(ctx, fp);
}

static int do_sort(GsContext *ctx, GsAsset *as, const FrameConsts &fc) {
  GsNvtxRange nvtx("GaussianSplat.Sort");
  int rc = ensure_sort_scratch(ctx, as->av.n);
  if (rc) return rc;
  rec(ctx, EV_BEGIN);
  // one clear for the whole sort: the digit histograms k_calc_distances counts into, the four passes' look-back rows and
  // their tickets.  It releases before it waits, so that k_calc_distances computes the keys beside the previous call's
  // last kernel and waits only to count them into the cleared histograms
  const SortScratch sc = sort_scratch(ctx);
  ClearSpans cl = {};
  cl.ptr[0] = sc.ghist; cl.words[0] = 4 * 256;
  cl.ptr[1] = sc.lookback; cl.words[1] = sort_lookback_words(as->av.n, 4);
  cl.ptr[2] = sc.tickets; cl.words[2] = 4;
  launch_clear(cl, ctx->stream, /*release_first=*/true);
  launch_calc_distances(as->av, fc, as->key_table.get(), sc.ghist, ctx->stream);
  rec(ctx, EV_DIST);
  cudaEvent_t pe[5] = {ctx->ev[EV_SORT0], ctx->ev[EV_SORT1], ctx->ev[EV_SORT2], ctx->ev[EV_SORT3], ctx->ev[EV_SORT4]};
  GS_CUDA_TRY(ctx, launch_sort_pairs(as->keys.get(), as->order.get(), as->d_n.get(), as->av.n, 4, 8, true, sc, ctx->stream,
                                     ctx->timing ? pe : nullptr, as->key_table.get(), true, nullptr, nullptr, /*scratch_clear=*/true));
  if (ctx->timing) for (int e = EV_SORT0; e <= EV_SORT4; ++e) ctx->ev_valid[e] = true;
  ctx->launches += 1 + 4;
  GS_CUDA_TRY(ctx, cudaGetLastError());
  return GS_OK;
}

static GsRenderOptions default_opts() {
  GsRenderOptions o;
  memset(&o, 0, sizeof(o));
  return o;
}

int do_view(GsContext *ctx, GsAsset *as, const GsFrameParams *fp, const FrameConsts &fc, bool cull, const GsRenderOptions &opt,
            cudaStream_t stream, float4 *draw, float *zndc, bool after_sort) {
  GsNvtxRange nvtx("GaussianSplat.CalcView");
  int rc = upload_frame_inputs(ctx, as, fp, stream);
  if (rc) return rc;
  const bool own = stream == ctx->stream;   // the group path runs view-calc beside the sort on a second stream and times it itself
  if (own) rec(ctx, EV_VIEW0);
  if (draw) {   // a record slab: the asset's own records stay as they are
    launch_calc_view(as->av, fc, ctx->d_cutouts.get(), ctx->d_deleted.get(), ctx->d_selected.get(), as->view.get(), as->rect.get(), draw,
                     as->block_bits.get(), fp->scene_depth ? zndc : nullptr, cull, make_partition(opt), stream, after_sort);
    if (own) rec(ctx, EV_VIEW1);
    ctx->launches += 1;
    GS_CUDA_TRY(ctx, cudaGetLastError());
    return GS_OK;
  }
  if (fp->scene_depth) GS_CUDA_TRY(ctx, as->zndc.reserve((size_t)as->av.n + 4, {ctx->stream}));   // 16 bytes of slack
  as->zndc_valid = fp->scene_depth != nullptr;
  launch_calc_view(as->av, fc, ctx->d_cutouts.get(), ctx->d_deleted.get(), ctx->d_selected.get(), as->view.get(), as->rect.get(), as->draw.get(),
                   as->block_bits.get(), as->zndc_valid ? as->zndc.get() : nullptr, cull, make_partition(opt), stream, after_sort);
  if (own) rec(ctx, EV_VIEW1);
  ctx->launches += 1;
  as->view_valid = !cull;
  as->draw_valid = true;
  {
    const gs::Partition p = make_partition(opt);
    as->draw_part[0] = p.range ? p.t0 : p.index; as->draw_part[1] = cull ? (p.range ? 0xFFFFFFFFu : p.count) : 0; as->draw_part[2] = p.range ? p.t1 : p.band;
  }
  as->view_w = (uint32_t)fp->screen_w;
  as->view_h = (uint32_t)fp->screen_h;
  GS_CUDA_TRY(ctx, cudaGetLastError());
  return GS_OK;
}

// The raster-tile cost history (launch order) of a draw of `tiles` tiles, in *cost.  layout == nullptr: the single-grid history
// of gs_frame, gs_render, the group path and the one-camera runs, indexed by the tile's id in the whole image and reset when
// the tile count changes.  Otherwise a run of several cameras, whose layout ((raster tiles per row, rows) of each camera) keeps
// its own history in cams_tile_cost, so that the runs of one call and the single-grid draws between calls do not reset each
// other's.  At most kCameraLayouts layouts are kept; one more starts that cache afresh.  The launch-order scratch
// tile_order serves both.
constexpr size_t kCameraLayouts = 16;
static int tile_history(GsContext *ctx, uint32_t tiles, const std::vector<uint32_t> *layout, uint32_t **cost) {
  if (tiles > ctx->tile_cost.size()) ctx->raster_tiles_cur = 0;   // a new buffer holds no history
  GS_CUDA_TRY(ctx, ctx->tile_cost.reserve(tiles, {ctx->stream}));
  GS_CUDA_TRY(ctx, ctx->tile_order.reserve(tiles, {ctx->stream}));
  if (!layout) {
    if (tiles != ctx->raster_tiles_cur) {
      GS_CUDA_TRY(ctx, cudaMemsetAsync(ctx->tile_cost.get(), 0, (size_t)tiles * 4, ctx->stream));
      ctx->raster_tiles_cur = tiles;
    }
    *cost = ctx->tile_cost.get();
    return GS_OK;
  }
  for (size_t i = 0; i < ctx->cams_layouts.size(); ++i)
    if (ctx->cams_layouts[i] == *layout) { *cost = ctx->cams_tile_cost.get() + ctx->cams_layout_base[i]; return GS_OK; }
  if (ctx->cams_layouts.size() >= kCameraLayouts) { ctx->cams_layouts.clear(); ctx->cams_layout_base.clear(); ctx->cams_cost_used = 0; }
  const size_t need = ctx->cams_cost_used + tiles;
  if (need > ctx->cams_tile_cost.size()) {   // grown with the histories kept
    Buffer<uint32_t> grown;
    GS_CUDA_TRY(ctx, grown.reserve(std::max(need, 2 * ctx->cams_tile_cost.size()), {ctx->stream}));
    if (ctx->cams_cost_used)
      GS_CUDA_TRY(ctx, cudaMemcpyAsync(grown.get(), ctx->cams_tile_cost.get(), ctx->cams_cost_used * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    cudaStreamSynchronize(ctx->stream);
    std::swap(ctx->cams_tile_cost, grown);   // the old buffer is freed with `grown`
  }
  GS_CUDA_TRY(ctx, cudaMemsetAsync(ctx->cams_tile_cost.get() + ctx->cams_cost_used, 0, (size_t)tiles * 4, ctx->stream));
  ctx->cams_layouts.push_back(*layout);
  ctx->cams_layout_base.push_back(ctx->cams_cost_used);
  *cost = ctx->cams_tile_cost.get() + ctx->cams_cost_used;
  ctx->cams_cost_used = need;
  return GS_OK;
}

int do_draw(GsContext *ctx, CallSurfaces *surfs, const FrameConsts &fc, const GsRenderOptions &opt, GsAsset *as, const GsFrameParams *fp,
            void *d_rt, uint32_t pitch, uint32_t fmt, Surface surf, cudaEvent_t bin_done) {
  GsNvtxRange nvtx("GaussianSplat.Draw");
  const uint32_t n = as->av.n, bins = fc.binsX * fc.binsY;
  int rc = GS_OK;
  if ((rc = ctx->bins.begin_draw(ctx, 1, fc)) || (rc = ctx->bins.reserve(ctx, n, bins))) return rc;
  uint32_t *tile_cost = nullptr;
  const uint32_t rtiles = (((uint32_t)fc.screenW + kTile - 1) / kTile) * fc.binsY * (kBin / kTile);   // of the whole image
  if ((rc = tile_history(ctx, rtiles, nullptr, &tile_cost))) return rc;
  if (depth_on_host(fp)) GS_CUDA_TRY(ctx, ctx->d_depth.reserve((size_t)(uint32_t)fp->screen_w * (uint32_t)fp->screen_h, {ctx->stream}));
  SceneDepth depth;
  if ((rc = bind_depth(ctx, surfs, fp, ctx->d_depth.get(), ctx->stream, &depth))) return rc;
  BinScratch lists;
  int bin_launches = 0, more = 0;
  GS_CUDA_TRY(ctx, launch_binning(fc, opt, as->order.get(), as->rect.get(), as->block_bits.get(), n, ctx->bins.clears(), bin_scratch(ctx),
                                  sort_scratch(ctx), ctx->stream, &lists, &bin_launches));
  bool again = false, clear = false;
  if ((rc = ctx->bins.end_draw(ctx, n, bins, &again, &clear))) return rc;
  if (again) {
    GS_CUDA_TRY(ctx, launch_binning(fc, opt, as->order.get(), as->rect.get(), as->block_bits.get(), n, clear, bin_scratch(ctx), sort_scratch(ctx),
                                    ctx->stream, &lists, &more));
    bin_launches += more;
  }
  rec(ctx, EV_BIN1);
  if (bin_done) cudaEventRecord(bin_done, ctx->stream);
  launch_raster(fc, opt, as->draw.get(), fp->scene_depth ? as->zndc.get() : nullptr, fp->selected_bits != nullptr || fp->scene_depth != nullptr,
                lists, d_rt, pitch, fmt, surf, ctx->stream, depth);
  rec(ctx, EV_RASTER1);
  ctx->launches += bin_launches + 3;  // look-back clear + bin_emit, 1-2 sort passes; bin_ranges, tile_order, raster
  GS_CUDA_TRY(ctx, cudaGetLastError());
  return GS_OK;
}

// options shared by gs_render / gs_frame: validated copy
int check_options(GsContext *ctx, const FrameConsts &fc, GsRenderOptions &opt) {
  if (opt.blend_mode > GS_BLEND_FP32) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "bad blend mode");
  if (opt.row_end > opt.row_begin) {
    const uint32_t rows = ((uint32_t)fc.screenH + kTile - 1) / kTile;
    if (opt.row_end > rows) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "row_end beyond the last 16-pixel row of the screen");
    opt.band_packed = 0; opt.partition_count = 0; opt.partition_index = 0;
  } else {
    opt.row_begin = opt.row_end = 0;
  }
  return GS_OK;
}

cudaError_t asset_init_work(GsContext *ctx, GsAsset *as, uint32_t n, uint32_t pos_fmt, uint32_t scale_fmt, uint32_t sh_fmt,
                            uint32_t col_fmt, uint32_t chunk_count) {
  const cudaStream_t s = ctx->stream;
  cudaError_t e = cudaSuccess;
  // view: 16 bytes of slack; block_bits: 64
  if ((e = as->order.reserve(n, {s})) != cudaSuccess || (e = as->keys.reserve(n, {s})) != cudaSuccess ||
      (e = as->key_table.reserve(n, {s})) != cudaSuccess || (e = as->draw.reserve((size_t)n * 3, {s})) != cudaSuccess ||
      (e = as->view.reserve((size_t)n * kViewStride / 4 + 4, {s})) != cudaSuccess || (e = as->rect.reserve(n, {s})) != cudaSuccess ||
      (e = as->d_n.reserve(1, {s})) != cudaSuccess || (e = as->block_bits.reserve(block_bits_words(n) + 16, {s})) != cudaSuccess)
    return e;
  if ((e = cudaMemcpyAsync(as->d_n.get(), &n, 4, cudaMemcpyHostToDevice, s)) != cudaSuccess) return e;
  as->av.n = n;
  as->av.posFmt = pos_fmt; as->av.scaleFmt = scale_fmt; as->av.shFmt = sh_fmt; as->av.colFmt = col_fmt;
  as->av.chunkCount = chunk_count;
  const GsBlobs &b = *as->blobs;
  as->av.pos = b.pos.get(); as->av.other = b.other.get(); as->av.sh = b.sh.get();
  as->av.color = b.color.get(); as->av.chunks = (const Chunk *)b.chunks.get();
  launch_set_indices(as->order.get(), as->av.n, s);  // CSSetIndices
  ctx->launches += 1;
  // `n` is a stack value: the copy above must have left it before this returns
  return cudaStreamSynchronize(s);
}

// d_rt == nullptr: the render target is the CUDA array (layer) behind rt_surf.  Enqueued on `s`: the context's stream, or the group
// path's transfer stream (surfs must then hand its surfaces over on `s` as well).
static int composite_impl(GsContext *ctx, CallSurfaces &surfs, const void *d_rt, uint32_t rt_pitch, Surface rt_surf,
                          uint32_t rt_fmt, GsImage *tgt, uint32_t W, uint32_t H, cudaStream_t s) {
  GsNvtxRange nvtx("GaussianSplat.Compose");
  uint32_t tp = 0;
  int rc = image_ok(ctx, tgt, W, H, ImageRole::kCameraTarget, &tp);
  if (rc) return rc;
  const bool host = tgt->memory == GS_MEM_HOST;
  if (host) GS_CUDA_TRY(ctx, ctx->tgt_scratch.reserve((size_t)W * pix_bytes(tgt->format) * H, {ctx->stream}));
  DeviceImage t;
  if ((rc = bind_image(ctx, surfs, tgt, tp, tgt->format, W, H, ctx->tgt_scratch.get(), StagingFill::kUpload, s, &t))) return rc;
  launch_composite(d_rt, rt_pitch, rt_surf, rt_fmt, t.d_rt, t.pitch, t.surf, tgt->format, W, H, s);
  if (host && (rc = copy_to_image(ctx, tgt, tp, t.d_rt, t.pitch, W, H, s))) return rc;
  if (s == ctx->stream) rec(ctx, EV_COMP1);
  ctx->launches += 1;
  GS_CUDA_TRY(ctx, cudaGetLastError());
  if (host) GS_CUDA_TRY(ctx, cudaStreamSynchronize(s));
  return GS_OK;
}
int composite_device_rt(GsContext *ctx, const void *d_rt, uint32_t rt_pitch, uint32_t rt_fmt, GsImage *tgt, uint32_t W, uint32_t H,
                        cudaStream_t s) {
  CallSurfaces surfs(ctx, s);
  return composite_impl(ctx, surfs, d_rt, rt_pitch, Surface{}, rt_fmt, tgt, W, H, s);
}

// The device image a frame draws into (DeviceImage): `rt` itself when it is device or array memory, else library scratch (or,
// with GS_FLAG_ASYNC_READBACK, one of the two asynchronous staging images) that a host `rt` is read back from.
struct FrameImage : DeviceImage {
  bool async_rb = false;
  int slot = 0;
};

// what a frame does between its view-calcs and its draw; rt (when given) has passed image_ok.  staging (optional): where a
// staging image goes instead of rt_scratch (one slice per camera of a run of several cameras).  A staging image starts from
// the host rt's content (GS_FLAG_LOAD_RT; zeros without an rt), or from zeros where a partition leaves rows untouched.
static int begin_frame_image(GsContext *ctx, CallSurfaces &surfs, const GsRenderOptions &opt, GsImage *rt, uint32_t rt_pitch,
                             uint32_t rt_fmt, const GsImage *tgt, uint32_t W, uint32_t H, FrameImage *fi, void *staging = nullptr) {
  int rc = GS_OK;
  const bool staged = !rt || rt->memory == GS_MEM_HOST;
  const size_t bytes = (size_t)W * pix_bytes(rt_fmt) * H;
  fi->async_rb = rt && staged && !tgt && (opt.flags & GS_FLAG_ASYNC_READBACK) != 0;
  if (fi->async_rb) {
    if ((rc = ensure_async_readback(ctx))) return rc;
    const int slot = fi->slot = ctx->rt_flip;
    ctx->rt_flip ^= 1;
    // the staging image of two frames ago: its copy must have left the device before this frame's raster overwrites it
    if (ctx->copy_pending[slot]) GS_CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_copy_done[slot], 0));
    GS_CUDA_TRY(ctx, ctx->rt_async[slot].reserve(bytes, {ctx->stream, ctx->copy_stream}));
    staging = ctx->rt_async[slot].get();
  } else if (staged && !staging) {
    GS_CUDA_TRY(ctx, ctx->rt_scratch.reserve(bytes, {ctx->stream}));
    staging = ctx->rt_scratch.get();
  }
  const StagingFill fill = (opt.flags & GS_FLAG_LOAD_RT) ? (rt ? StagingFill::kUpload : StagingFill::kZero)
                           : (opt.partition_count > 1 || opt.row_end > opt.row_begin) ? StagingFill::kZero : StagingFill::kNone;
  return bind_image(ctx, surfs, rt, rt_pitch, rt_fmt, W, H, staging, fill, ctx->stream, fi);
}

// what follows the draw: the read-back of a host `rt` (enqueued only, with GS_FLAG_ASYNC_READBACK) and the composite onto the
// camera target.  The caller checks the bin list once, after its last draw.
static int end_frame_image(GsContext *ctx, CallSurfaces &surfs, GsImage *rt, uint32_t rt_pitch, uint32_t rt_fmt, GsImage *tgt, uint32_t W,
                           uint32_t H, const FrameImage &fi) {
  int rc = GS_OK;
  if (fi.async_rb) {
    const int slot = fi.slot;
    GS_CUDA_TRY(ctx, cudaEventRecord(ctx->ev_rt_ready[slot], ctx->stream));
    GS_CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_rt_ready[slot], 0));
    if ((rc = copy_to_image(ctx, rt, rt_pitch, fi.d_rt, fi.pitch, W, H, ctx->copy_stream))) return rc;
    GS_CUDA_TRY(ctx, cudaEventRecord(ctx->ev_copy_done[slot], ctx->copy_stream));
    ctx->copy_pending[slot] = true;
    return GS_OK;   // completion and the bin-list check: gs_sync
  }
  if (rt && rt->memory == GS_MEM_HOST && (rc = copy_to_image(ctx, rt, rt_pitch, fi.d_rt, fi.pitch, W, H, ctx->stream))) return rc;
  return tgt ? composite_impl(ctx, surfs, fi.d_rt, fi.pitch, fi.surf, rt_fmt, tgt, W, H, ctx->stream) : GS_OK;
}

}  // namespace gs

using namespace gs;

extern "C" {

const char *gs_version(void) { return "gsplat_b200 0.1 (sm_90a)"; }

const char *gs_last_error(GsContext *ctx) { return ctx ? ctx->err.c_str() : g_last_error.c_str(); }

int gs_create(int cuda_device, void *stream_handle, GsContext **out) {
  if (!out) return fail(nullptr, GS_ERR_INVALID_ARGUMENT, "out is null");
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    cudaGetLastError();
    return fail(nullptr, GS_ERR_NO_DEVICE, "no CUDA device: libgsplat_b200 has no CPU fallback");
  }
  if (cuda_device < 0 || cuda_device >= count) return fail(nullptr, GS_ERR_INVALID_ARGUMENT, "bad device index");
  GsContext *ctx = new (std::nothrow) GsContext();
  if (!ctx) return fail(nullptr, GS_ERR_OUT_OF_MEMORY, "host allocation failed");
  ctx->device = cuda_device;
  auto init = [&]() -> int {
    GS_CUDA_TRY(ctx, cudaSetDevice(cuda_device));
    if (stream_handle) ctx->stream = (cudaStream_t)stream_handle;
    else {
      // own stream: highest priority, so that the group path's helper stream (view-calc, lowest priority) only fills what the
      // sort / compositing chain on this stream leaves idle
      int least = 0, greatest = 0;
      GS_CUDA_TRY(ctx, cudaDeviceGetStreamPriorityRange(&least, &greatest));
      GS_CUDA_TRY(ctx, cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, greatest));
      ctx->own_stream = true;
    }
    for (int i = 0; i < EV_COUNT; ++i) GS_CUDA_TRY(ctx, cudaEventCreate(&ctx->ev[i]));
    GS_CUDA_TRY(ctx, ctx->sort_ghist.reserve(4 * 256, {ctx->stream}));
    GS_CUDA_TRY(ctx, ctx->sort_tickets.reserve(4, {ctx->stream}));
    GS_CUDA_TRY(ctx, ctx->d_scalar.reserve(16, {ctx->stream}));
    GS_CUDA_TRY(ctx, ctx->bins.entry_count.reserve(4, {ctx->stream}));
    GS_CUDA_TRY(ctx, cudaMemsetAsync(ctx->bins.entry_count.get(), 0, 16, ctx->stream));
    return GS_OK;
  };
  const int rc = init();
  if (rc != GS_OK) {
    g_last_error = ctx->err;   // keep the text reachable through gs_last_error(NULL)
    gs_destroy(ctx);
    return rc;
  }
  *out = ctx;
  return GS_OK;
}

void gs_destroy(GsContext *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  if (ctx->copy_stream) { cudaStreamSynchronize(ctx->copy_stream); cudaStreamDestroy(ctx->copy_stream); }
  for (int i = 0; i < 2; ++i) {
    if (ctx->ev_rt_ready[i]) cudaEventDestroy(ctx->ev_rt_ready[i]);
    if (ctx->ev_copy_done[i]) cudaEventDestroy(ctx->ev_copy_done[i]);
  }
  for (int i = 0; i < EV_COUNT; ++i) if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
  release_surfaces(ctx, true);   // waits for each batch's event (a group's transfer stream may still hold one)
  for (cudaEvent_t e : ctx->spare_events) cudaEventDestroy(e);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;   // frees the scratch buffers, on the context's device
}

int gs_sync(GsContext *ctx) {
  if (!ctx) return fail(nullptr, GS_ERR_INVALID_ARGUMENT, "null context");
  GS_CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  // frames rendered into device images are not checked when they are enqueued: surface a truncated bin list here
  const int rc = ctx->bins.check(ctx);
  if (ctx->copy_stream) {   // asynchronous read-backs in flight complete here
    GS_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->copy_stream));
    ctx->copy_pending[0] = ctx->copy_pending[1] = false;
  }
  GS_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  release_surfaces(ctx, true);   // also waits for surfaces a group's transfer stream still uses (camera targets)
  return rc;
}

int gs_set_timing(GsContext *ctx, int enabled) {
  if (!ctx) return fail(nullptr, GS_ERR_INVALID_ARGUMENT, "null context");
  ctx->timing = enabled != 0;
  return GS_OK;
}

int gs_get_stage_times(GsContext *ctx, GsStageTimes *out) {
  if (!ctx || !out) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null argument");
  GS_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  GsStageTimes t = ctx->times;
  t.distances_ms = ev_ms(ctx, EV_BEGIN, EV_DIST);
  t.sort_ms = ev_ms(ctx, EV_SORT0, EV_SORT4);
  for (int p = 0; p < 4; ++p) t.sort_pass_ms[p] = ev_ms(ctx, EV_SORT0 + p, EV_SORT1 + p);
  t.view_ms = ev_ms(ctx, EV_VIEW0, EV_VIEW1);
  t.bin_ms = ev_ms(ctx, EV_VIEW1, EV_BIN1);
  t.raster_ms = ev_ms(ctx, EV_BIN1, EV_RASTER1);
  t.composite_ms = ev_ms(ctx, EV_RASTER1, EV_COMP1);
  int first = ctx->ev_valid[EV_BEGIN] ? EV_BEGIN : EV_VIEW0, last = EV_VIEW1;
  for (int e = EV_VIEW1; e < EV_COUNT; ++e) if (ctx->ev_valid[e]) last = e;
  t.total_ms = ev_ms(ctx, first, last);
  uint32_t ec[2] = {0, 0};
  ctx->bins.read(ctx, ec, 2);   // a failed read reports no entries
  t.tile_entries = ec[0];
  t.kernel_launches = ctx->launches;
  *out = t;
  return GS_OK;
}

int gs_asset_upload(GsContext *ctx, const GsAssetDesc *d, GsAsset **out) {
  if (!ctx || !d || !out) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  // HasValidAsset, R/GaussianSplatRenderer.cs:361-368
  if (d->splat_count == 0 || !d->pos || !d->other || !d->sh || !d->color) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "asset has no splats or a null blob");
  if (d->pos_format > 3 || d->scale_format > 3) return fail(ctx, GS_ERR_UNSUPPORTED_FORMAT, "unknown vector format");
  if (d->color_format > GS_COL_BC7) return fail(ctx, GS_ERR_UNSUPPORTED_FORMAT, "unknown colour format");
  if (d->sh_format > GS_SH_CLUSTER4K) return fail(ctx, GS_ERR_UNSUPPORTED_FORMAT, "unknown SH format");
  const uint64_t n = d->splat_count;
  // clustered SH (R/GaussianSplatAsset.cs:135-150,187-198): the blob is a palette of 64k..4k Float16 entries and every
  // splat carries a u16 palette index at the end of its `other` record (S/GaussianSplatting.hlsl:447-448,467-470)
  const bool clustered = d->sh_format > GS_SH_NORM6;
  if (d->pos_bytes < n * vec_stride(d->pos_format) || d->other_bytes < n * other_stride(d->scale_format, d->sh_format) ||
      d->sh_bytes < (uint64_t)sh_count(d->sh_format, d->splat_count) * sh_stride(d->sh_format) ||
      d->color_bytes < (uint64_t)kTexWidth * tex_height(n) * color_size(d->color_format))
    return fail(ctx, GS_ERR_INVALID_ARGUMENT, "asset blob smaller than its format requires");
  const uint32_t chunk_count = (d->chunks && d->chunk_bytes) ? (uint32_t)(d->chunk_bytes / 64) : 0;
  GS_CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  GsAsset *as = new (std::nothrow) GsAsset();
  if (as) as->blobs = new (std::nothrow) GsBlobs();
  if (!as || !as->blobs) {
    delete as;
    return fail(ctx, GS_ERR_OUT_OF_MEMORY, "host allocation failed");
  }
  as->ctx = ctx;
  GsBlobs &b = *as->blobs;
  auto up = [&](gs::Buffer<uint8_t> &dst, const void *src, uint64_t bytes, uint64_t min_bytes = 0) -> cudaError_t {
    // +16 bytes of slack: the widest vector load of the last splat may read past a tightly sized blob
    const uint64_t alloc = (bytes > min_bytes ? bytes : min_bytes) + 16;
    cudaError_t e = dst.reserve(alloc, {ctx->stream});
    if (e != cudaSuccess) return e;
    e = cudaMemsetAsync(dst.get() + bytes, 0, alloc - bytes, ctx->stream);
    if (e != cudaSuccess) return e;
    return cudaMemcpyAsync(dst.get(), src, bytes, cudaMemcpyHostToDevice, ctx->stream);
  };
  // a u16 palette index can name any of 65536 entries whatever the palette's nominal size: back all of them (zeros)
  const uint64_t sh_min = clustered ? 65536ull * 96ull : 0ull;
  cudaError_t e = cudaSuccess;
  if ((e = up(b.pos, d->pos, d->pos_bytes)) != cudaSuccess || (e = up(b.other, d->other, d->other_bytes)) != cudaSuccess ||
      (e = up(b.sh, d->sh, d->sh_bytes, sh_min)) != cudaSuccess || (e = up(b.color, d->color, d->color_bytes)) != cudaSuccess ||
      (chunk_count && (e = up(b.chunks, d->chunks, (uint64_t)chunk_count * 64)) != cudaSuccess) ||
      (e = asset_init_work(ctx, as, d->splat_count, d->pos_format, d->scale_format, d->sh_format, d->color_format, chunk_count)) != cudaSuccess) {
    gs_asset_destroy(as);
    cudaGetLastError();   // a failed copy or launch leaves its error behind: the next call on the context must not report it
    return fail_cuda(ctx, e, "asset upload", __FILE__, __LINE__);
  }
  GS_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));  // host blobs are only borrowed for this call
  *out = as;
  return GS_OK;
}

void gs_asset_destroy(GsAsset *as) {
  if (!as) return;
  if (as->ctx) { cudaSetDevice(as->ctx->device); cudaStreamSynchronize(as->ctx->stream); }
  delete as;
}

int gs_asset_instance(const GsAsset *source, GsAsset **out) {
  if (out) *out = nullptr;
  if (!source || !out) return fail(source ? source->ctx : nullptr, GS_ERR_INVALID_ARGUMENT, "null argument");
  GsContext *ctx = source->ctx;
  GS_CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  GsAsset *as = new (std::nothrow) GsAsset();
  if (!as) return fail(ctx, GS_ERR_OUT_OF_MEMORY, "host allocation failed");
  as->ctx = ctx;
  as->blobs = source->blobs;
  as->blobs->refs.fetch_add(1);
  const AssetView &sv = source->av;
  const cudaError_t e = asset_init_work(ctx, as, sv.n, sv.posFmt, sv.scaleFmt, sv.shFmt, sv.colFmt, sv.chunkCount);
  if (e != cudaSuccess) {
    gs_asset_destroy(as);   // gives its reference back: the source's blobs stay
    cudaGetLastError();
    return fail_cuda(ctx, e, "asset instance", __FILE__, __LINE__);
  }
  *out = as;
  return GS_OK;
}

int gs_asset_reset_order(GsAsset *as) {
  if (!as) return fail(nullptr, GS_ERR_INVALID_ARGUMENT, "null asset");
  launch_set_indices(as->order.get(), as->av.n, as->ctx->stream);
  as->ctx->launches += 1;
  GS_CUDA_TRY(as->ctx, cudaGetLastError());
  return GS_OK;
}

uint32_t gs_asset_splat_count(const GsAsset *as) { return as ? as->av.n : 0; }

int gs_sort(GsContext *ctx, GsAsset *as, const GsFrameParams *fp) {
  int rc = check_params(ctx, as, fp);
  if (rc) return rc;
  for (int e = 0; e < EV_COUNT; ++e) ctx->ev_valid[e] = false;
  FrameConsts fc = make_frame_consts(fp);
  return do_sort(ctx, as, fc);
}

int gs_calc_view(GsContext *ctx, GsAsset *as, const GsFrameParams *fp) {
  int rc = check_params(ctx, as, fp);
  if (rc) return rc;
  for (int e = 0; e < EV_COUNT; ++e) ctx->ev_valid[e] = false;
  FrameConsts fc = make_frame_consts(fp);
  return do_view(ctx, as, fp, fc, false, default_opts(), ctx->stream);
}

int gs_render(GsContext *ctx, GsAsset *as, const GsFrameParams *fp, const GsRenderOptions *opt_in, GsImage *rt) {
  int rc = check_params(ctx, as, fp);
  if (rc) return rc;
  if (!as->draw_valid || as->view_w != (uint32_t)fp->screen_w || as->view_h != (uint32_t)fp->screen_h)
    return fail(ctx, GS_ERR_NOT_READY, "gs_render needs gs_calc_view for the same screen size first");
  const uint32_t W = (uint32_t)fp->screen_w;
  uint32_t pitch = 0;
  GsRenderOptions opt = opt_in ? *opt_in : default_opts();
  FrameConsts fc = make_frame_consts(fp);
  if ((rc = check_options(ctx, fc, opt))) return rc;
  {
    const gs::Partition p = make_partition(opt);
    const uint32_t want[3] = {p.range ? p.t0 : p.index, p.range ? 0xFFFFFFFFu : p.count, p.range ? p.t1 : p.band};
    if (as->draw_part[1] > 1 && (as->draw_part[0] != want[0] || as->draw_part[1] != want[1] || as->draw_part[2] != want[2]))
      return fail(ctx, GS_ERR_NOT_READY, "the last gs_frame prepared draw records for another tile partition; run gs_calc_view");
  }
  const uint32_t H = opt.band_packed ? partition_own_bin_rows(opt, fc.binsY) * kBin : (uint32_t)fp->screen_h;
  if (opt.band_packed && rt && is_array_image(rt))
    return fail(ctx, GS_ERR_INVALID_ARGUMENT, "band_packed output is the send buffer of an all-gather: it must be linear memory, not a CUDA array");
  if ((rc = image_ok(ctx, rt, W, H, ImageRole::kRenderTarget, &pitch))) return rc;
  if (fp->scene_depth && !as->zndc_valid) return fail(ctx, GS_ERR_NOT_READY, "a scene depth buffer needs the quad depths: run gs_calc_view with scene_depth set");
  for (int e = EV_BIN1; e < EV_COUNT; ++e) ctx->ev_valid[e] = false;
  rec(ctx, EV_VIEW1);
  opt.flags &= ~(uint32_t)GS_FLAG_ASYNC_READBACK;   // a host rt is read back before gs_render returns
  CallSurfaces surfs(ctx);
  FrameImage fi;
  if ((rc = begin_frame_image(ctx, surfs, opt, rt, pitch, rt->format, nullptr, W, H, &fi))) return rc;
  ctx->bins.begin_call();
  if ((rc = do_draw(ctx, &surfs, fc, opt, as, fp, fi.d_rt, fi.pitch, rt->format, fi.surf)) ||
      (rc = end_frame_image(ctx, surfs, rt, pitch, rt->format, nullptr, W, H, fi)))
    return rc;
  return rt->memory == GS_MEM_HOST ? ctx->bins.check(ctx) : GS_OK;
}

int gs_composite(GsContext *ctx, const GsImage *rt, GsImage *tgt) {
  if (!ctx || !rt || !tgt) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null argument");
  GS_CUDA_TRY(ctx, cudaSetDevice(ctx->device));   // array images are inspected and bound on the context's device
  uint32_t rp = 0;
  int rc = image_ok(ctx, rt, rt->width, rt->height, ImageRole::kRenderTarget, &rp);
  if (rc) return rc;
  const uint32_t W = rt->width, H = rt->height;
  ctx->ev_valid[EV_COMP1] = false;
  rec(ctx, EV_RASTER1);
  CallSurfaces surfs(ctx);
  if (rt->memory == GS_MEM_HOST) GS_CUDA_TRY(ctx, ctx->rt_scratch.reserve((size_t)W * pix_bytes(rt->format) * H, {ctx->stream}));
  DeviceImage r;
  if ((rc = bind_image(ctx, surfs, rt, rp, rt->format, W, H, ctx->rt_scratch.get(), StagingFill::kUpload, ctx->stream, &r))) return rc;
  return composite_impl(ctx, surfs, r.d_rt, r.pitch, r.surf, rt->format, tgt, W, H, ctx->stream);
}

}  // extern "C"

namespace gs {
// One camera of gs_frame_objects / gs_frame_cameras: its objects' arguments assets / fps / do_sort_flags [off, off + K), and
// its images.
struct CameraArgs {
  uint32_t off, K, W, H, rt_pitch = 0, rt_fmt = GS_PIX_RGBA16F;
  std::vector<FrameConsts> fcs;
  GsImage *rt, *tgt;
  FrameImage fi;     // set up by the camera's first run
};

// What gs_frame_objects checks of one camera's arguments: the objects, the options (validated into *opt) and the images.
// Out: the objects' uniforms, the screen size, and the render target's pitch and pixel format (RGBA16F without one).
static int check_camera(GsContext *ctx, GsAsset *const *assets, const GsFrameParams *fps, GsRenderOptions *opt, CameraArgs *a) {
  int rc = GS_OK;
  const uint32_t K = a->K;
  for (uint32_t k = 0; k < K; ++k) {
    if (!assets[k]) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null asset");
    if ((rc = check_params(ctx, assets[k], &fps[k]))) return rc;
    if (fps[k].screen_w != fps[0].screen_w || fps[k].screen_h != fps[0].screen_h)
      return fail(ctx, GS_ERR_INVALID_ARGUMENT, "the objects of one call must share screen_w / screen_h");
  }
  {
    std::vector<GsAsset *> sorted(assets, assets + K);
    std::sort(sorted.begin(), sorted.end());
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end())
      return fail(ctx, GS_ERR_INVALID_ARGUMENT, "an asset is listed for two objects (its draw order would be sorted twice)");
  }
  if (!a->rt && !a->tgt) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "gs_frame_objects needs rt and/or camera_target");
  if (opt->flags & GS_FLAG_LOAD_RT) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "GS_FLAG_LOAD_RT is not accepted: the call clears the target once itself");
  if (opt->partition_count > 1 || opt->partition_index || opt->row_begin || opt->row_end || opt->band_packed)
    return fail(ctx, GS_ERR_INVALID_ARGUMENT, "gs_frame_objects draws the whole screen: no partition, row range or band packing");
  a->fcs.resize(K);
  for (uint32_t k = 0; k < K; ++k) a->fcs[k] = make_frame_consts(&fps[k]);
  if ((rc = check_options(ctx, a->fcs[0], *opt))) return rc;
  a->W = (uint32_t)fps[0].screen_w; a->H = (uint32_t)fps[0].screen_h;
  uint32_t tgt_pitch = 0;
  if (a->rt) { if ((rc = image_ok(ctx, a->rt, a->W, a->H, ImageRole::kRenderTarget, &a->rt_pitch))) return rc; a->rt_fmt = a->rt->format; }
  if (a->tgt && (rc = image_ok(ctx, a->tgt, a->W, a->H, ImageRole::kCameraTarget, &tgt_pitch))) return rc;
  return GS_OK;
}

// ---- runs ---------------------------------------------------------------------------------------------
// A run (see DrawCameras) is a list of camera segments: the camera's pairs [k0, k0 + K), and load = 1 where an earlier run of
// the call drew the camera's first pairs.  A run holds at most kRunObjects pairs, each object of fewer than 2^kSlotShift splats
// (the slot tag), at most one scene depth buffer per camera, whole cameras of at most kMaxRunScreen px per axis when it holds
// several, and at most kMaxRunBins bins (the largest bin space the bin sort's digit plans cover).
constexpr uint32_t kMaxRunScreen = 8160, kMaxRunBins = 65536;
struct Segment {
  uint32_t cam, k0, K, load;
};
using Run = std::vector<Segment>;

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// The end of the longest run of the objects [k, K) that starts at k: at most kRunObjects objects, each of fewer than
// 2^kSlotShift splats, binding at most one scene depth buffer.
static uint32_t run_end(GsAsset *const *assets, const GsFrameParams *fps, uint32_t k, uint32_t K) {
  const GsFrameParams *depth = nullptr;
  uint32_t e = k;
  for (; e < K && e - k < kRunObjects && assets[e]->av.n <= kLocalIdMask; ++e) {
    const GsFrameParams &f = fps[e];
    if (!f.scene_depth) continue;
    if (!depth) depth = &f;
    else if (depth_id(&f) != depth_id(depth)) break;
  }
  return e;
}

// The call's cameras as runs, in order.  Consecutive whole cameras share a run while each fits it, the run's totals hold, they
// have one pixel format, and no camera's image shares pixels with another's render target (two cameras rasterizing into one
// image at once would race, where the loop draws one after the other; disjoint rectangles of one array do not).  A camera
// alone is split into runs of run_end, each later one loading what the earlier ones drew.
static std::vector<Run> form_runs(const std::vector<CameraArgs> &cams, GsAsset *const *assets, const GsFrameParams *fps) {
  auto whole = [&](uint32_t c) {
    const CameraArgs &a = cams[c];
    return a.W <= kMaxRunScreen && a.H <= kMaxRunScreen && run_end(assets + a.off, fps + a.off, 0, a.K) == a.K;
  };
  auto joins = [&](uint32_t c0, uint32_t c, uint32_t run_pairs, uint32_t run_bins) {
    const CameraArgs &a = cams[c];
    if (run_pairs + a.K > kRunObjects || run_bins + a.fcs[0].binsX * a.fcs[0].binsY > kMaxRunBins || a.rt_fmt != cams[c0].rt_fmt) return false;
    for (uint32_t j = c0; j < c; ++j)
      if (images_overlap(a.rt, cams[j].rt) || images_overlap(a.rt, cams[j].tgt) || images_overlap(a.tgt, cams[j].rt)) return false;
    return true;
  };
  std::vector<Run> runs;
  const uint32_t count = (uint32_t)cams.size();
  for (uint32_t c = 0; c < count;) {
    uint32_t e = c, run_pairs = 0, run_bins = 0;
    while (e < count && whole(e) && (e == c || joins(c, e, run_pairs, run_bins))) {
      run_pairs += cams[e].K;
      run_bins += cams[e].fcs[0].binsX * cams[e].fcs[0].binsY;
      ++e;
    }
    if (e - c >= 2) {
      runs.emplace_back();
      for (uint32_t j = c; j < e; ++j) runs.back().push_back({j, 0, cams[j].K, 0});
      c = e;
      continue;
    }
    const CameraArgs &a = cams[c];
    for (uint32_t k = 0; k < a.K;) {
      const uint32_t ke = std::max(run_end(assets + a.off, fps + a.off, k, a.K), k + 1);
      runs.push_back({{c, k, ke - k, k ? 1u : 0u}});
      k = ke;
    }
    ++c;
  }
  return runs;
}

// Draws one run.  Pair by pair the sort and the view-calc; a pair's bin entries are emitted before a later pair of the run
// sorts or view-calculates the same asset, and otherwise after the last view-calc.  A run of one pair is then drawn by
// do_draw; a longer one by one bin sort and one MULTI raster over every camera's tiles.  Each camera's image is set up by its
// first run (a camera of a run of several stages a host image in the run's scratch, every other camera in rt_scratch) and read
// back / composited after its last.
static int draw_run(GsContext *ctx, CallSurfaces &surfs, std::vector<CameraArgs> &cams, const Run &run, GsAsset *const *assets,
                    const GsFrameParams *fps, const int32_t *do_sort_flags, const GsRenderOptions &opt) {
  GsNvtxRange nvtx("GaussianSplat.DrawRun");
  int rc = ctx->bins.begin_draw(ctx, (uint32_t)run.size(), cams[run[0].cam].fcs[0]);   // any wait: before the run's sorts
  if (rc) return rc;
  std::vector<uint32_t> pair_at, seg_of;   // each pair's argument index and segment, in draw order
  for (uint32_t i = 0; i < run.size(); ++i)
    for (uint32_t k = run[i].k0; k < run[i].k0 + run[i].K; ++k) { pair_at.push_back(cams[run[i].cam].off + k); seg_of.push_back(i); }
  const uint32_t count = (uint32_t)pair_at.size();
  const bool multi = count > 1, cams_run = run.size() > 1;
  DrawCameras dc;
  memset(&dc, 0, sizeof(dc));
  DepthSurfaces depth_surfs{};
  dc.count = (uint32_t)run.size();
  std::vector<uint32_t> layout;
  uint32_t tiles = 0, bins = 0;
  uint64_t total = 0;
  size_t bytes = 0;
  std::vector<size_t> slab_at(count, 0), depth_at(run.size(), 0), stage_at(run.size(), 0);
  std::vector<const GsFrameParams *> depth_fp(run.size(), nullptr);
  for (uint32_t i = 0, q = 0; i < run.size(); ++i) {
    const CameraArgs &c = cams[run[i].cam];
    RasterCamera &r = dc.cam[i];
    r.W = c.W; r.H = c.H;
    r.binsX = c.fcs[0].binsX;
    r.ntx = (c.W + kTile - 1) / kTile;
    r.load = run[i].load;
    const uint32_t rows = c.fcs[0].binsY * (kBin / kTile);
    r.tile_base = tiles; r.bin_base = bins;
    tiles += r.ntx * rows;
    bins += r.binsX * c.fcs[0].binsY;
    layout.push_back(r.ntx); layout.push_back(rows);
    for (uint32_t k = 0; k < run[i].K; ++k, ++q) {
      const GsAsset *as = assets[pair_at[q]];
      const GsFrameParams &f = fps[pair_at[q]];
      total += as->av.n;
      if (f.scene_depth && !depth_fp[i]) depth_fp[i] = &f;
      // every appearance of an asset but its last in the run draws from a record slab: a later view-calc overwrites its own
      bool later = false;
      for (uint32_t m = q + 1; m < count; ++m) later |= assets[pair_at[m]] == as;
      slab_at[q] = later ? bytes + 1 : 0;   // 0: the asset's own buffers (offsets are stored + 1)
      if (later) bytes += align256((size_t)as->av.n * 48) + (f.scene_depth ? align256((size_t)as->av.n * 4 + 16) : 0);
    }
    if (multi && depth_fp[i] && depth_on_host(depth_fp[i])) { depth_at[i] = bytes; bytes += align256((size_t)c.W * c.H * 4); }
    if (cams_run && (!c.rt || c.rt->memory == GS_MEM_HOST)) { stage_at[i] = bytes; bytes += align256((size_t)c.W * pix_bytes(c.rt_fmt) * c.H); }
  }
  GS_CUDA_TRY(ctx, ctx->cams_scratch.reserve(bytes, {ctx->stream}));
  uint8_t *scratch = ctx->cams_scratch.get();
  const uint32_t n = (uint32_t)std::min<uint64_t>(total, 0xFFFFFFFFu);
  uint32_t *tile_cost = nullptr;
  if (multi) {
    GS_CUDA_TRY(ctx, ctx->cams_ghist.reserve(4 * 256, {ctx->stream}));
    if ((rc = ctx->bins.reserve(ctx, n, bins))) return rc;
    if ((rc = tile_history(ctx, tiles, cams_run ? &layout : nullptr, &tile_cost))) return rc;
    for (uint32_t i = 0; i < run.size(); ++i) {
      SceneDepth d;
      if (depth_fp[i] && (rc = bind_depth(ctx, &surfs, depth_fp[i], reinterpret_cast<float *>(scratch + depth_at[i]), ctx->stream, &d)))
        return rc;
      dc.cam[i].depth = d.ptr;
      if (d.on_surface) { depth_surfs.surf[i] = d.surf; depth_surfs.on_surface |= 1u << i; }
    }
    launch_bin_list_begin(bin_scratch(ctx), ctx->cams_ghist.get(), ctx->stream);
  }

  DrawObjects objs;
  memset(&objs, 0, sizeof(objs));
  objs.count = count;
  uint32_t emitted = 0;   // the pairs [emitted, p) are view-calculated and not yet emitted
  auto emit_to = [&](uint32_t end, bool clear) {
    for (; emitted < end; ++emitted) {
      const GsAsset *as = assets[pair_at[emitted]];
      const RasterCamera &r = dc.cam[seg_of[emitted]];
      launch_bin_emit_pair(as->order.get(), as->rect.get(), as->block_bits.get(), as->av.n, r.binsX, r.bin_base, emitted, clear && emitted == 0, bins,
                           bin_scratch(ctx), ctx->cams_ghist.get(), ctx->stream);
      ctx->launches += 2;   // look-back clear, bin_emit
    }
  };
  for (uint32_t p = 0; p < count; ++p) {
    GsAsset *as = assets[pair_at[p]];
    const GsFrameParams &f = fps[pair_at[p]];
    const CameraArgs &c = cams[run[seg_of[p]].cam];
    for (uint32_t q = emitted; q < p; ++q)
      if (assets[pair_at[q]] == as) { emit_to(p, ctx->bins.clears()); break; }
    float4 *draw = nullptr;
    float *zndc = nullptr;
    if (slab_at[p]) {
      draw = reinterpret_cast<float4 *>(scratch + slab_at[p] - 1);
      zndc = reinterpret_cast<float *>(scratch + slab_at[p] - 1 + align256((size_t)as->av.n * 48));
    }
    const bool sorted = do_sort_flags[pair_at[p]] != 0;
    if (sorted && (rc = do_sort(ctx, as, c.fcs[pair_at[p] - c.off]))) return rc;
    if ((rc = do_view(ctx, as, &f, c.fcs[pair_at[p] - c.off], true, opt, ctx->stream, draw, zndc, sorted))) return rc;
    objs.draw[p] = draw ? draw : as->draw.get();
    if (f.scene_depth) {
      objs.zndc[p] = draw ? zndc : as->zndc.get();
      objs.depth_mask |= 1u << p;
    }
    objs.extras |= f.selected_bits != nullptr || f.scene_depth != nullptr;
  }
  for (uint32_t i = 0; i < run.size(); ++i) {
    CameraArgs &c = cams[run[i].cam];
    if (!run[i].load && (rc = begin_frame_image(ctx, surfs, opt, c.rt, c.rt_pitch, c.rt_fmt, c.tgt, c.W, c.H, &c.fi,
                                                cams_run ? scratch + stage_at[i] : nullptr)))
      return rc;
    dc.cam[i].rt = static_cast<uint8_t *>(c.fi.d_rt); dc.cam[i].pitch = c.fi.pitch; dc.cam[i].surf = c.fi.surf;
  }
  if (!multi) {
    const CameraArgs &c = cams[run[0].cam];
    GsRenderOptions o = opt;
    if (run[0].load) o.flags |= GS_FLAG_LOAD_RT;
    if ((rc = do_draw(ctx, &surfs, c.fcs[run[0].k0], o, assets[pair_at[0]], &fps[pair_at[0]], c.fi.d_rt, c.fi.pitch, c.rt_fmt, c.fi.surf)))
      return rc;
  } else {
    emit_to(count, ctx->bins.clears());
    BinScratch lists;
    int sort_launches = 0, more = 0;
    GS_CUDA_TRY(ctx, launch_bin_list_sort(bins, bin_scratch(ctx), sort_scratch(ctx), ctx->cams_ghist.get(), ctx->stream, &lists, &sort_launches));
    bool again = false, clear = false;
    if ((rc = ctx->bins.end_draw(ctx, n, bins, &again, &clear))) return rc;
    if (again) {
      launch_bin_list_begin(bin_scratch(ctx), ctx->cams_ghist.get(), ctx->stream);
      emitted = 0;
      emit_to(count, clear);
      GS_CUDA_TRY(ctx, launch_bin_list_sort(bins, bin_scratch(ctx), sort_scratch(ctx), ctx->cams_ghist.get(), ctx->stream, &lists, &more));
      sort_launches += more;
    }
    lists.tile_cost = tile_cost;
    rec(ctx, EV_BIN1);
    launch_raster_cameras(objs, dc, depth_surfs, bins, tiles, opt.blend_mode, cams[run[0].cam].rt_fmt, lists, ctx->stream);
    rec(ctx, EV_RASTER1);
    ctx->launches += sort_launches + 3;   // bin sort passes; bin_ranges, tile_order, raster
    GS_CUDA_TRY(ctx, cudaGetLastError());
  }
  for (const Segment &sg : run) {
    CameraArgs &c = cams[sg.cam];
    if (sg.k0 + sg.K == c.K && (rc = end_frame_image(ctx, surfs, c.rt, c.rt_pitch, c.rt_fmt, c.tgt, c.W, c.H, c.fi))) return rc;
  }
  return GS_OK;
}

// The work of gs_frame_objects and gs_frame_cameras once every camera has passed check_camera: the runs in order, and the bin
// list's overflow reported here when some image was read back to the host, else at gs_sync.
static int draw_cameras(GsContext *ctx, std::vector<CameraArgs> &cams, GsAsset *const *assets, const GsFrameParams *fps,
                        const int32_t *do_sort_flags, const GsRenderOptions &opt) {
  int rc = GS_OK;
  // the objects' cutouts / bits share the context's buffers: sized for all of them before the first view-calc is queued
  const uint32_t pairs = cams.back().off + cams.back().K;
  for (uint32_t p = 0; p < pairs; ++p)
    if ((rc = reserve_frame_inputs(ctx, assets[p], &fps[p], {ctx->stream}))) return rc;
  for (int e = 0; e < EV_COUNT; ++e) ctx->ev_valid[e] = false;
  CallSurfaces surfs(ctx);
  ctx->bins.begin_call();
  for (const Run &run : form_runs(cams, assets, fps))
    if ((rc = draw_run(ctx, surfs, cams, run, assets, fps, do_sort_flags, opt))) return rc;
  bool host = false;
  for (const CameraArgs &c : cams)
    host |= (c.rt && c.rt->memory == GS_MEM_HOST && !c.fi.async_rb) || (c.tgt && c.tgt->memory == GS_MEM_HOST);
  return host ? ctx->bins.check(ctx) : GS_OK;
}
}  // namespace gs

extern "C" {

int gs_frame(GsContext *ctx, GsAsset *as, const GsFrameParams *fp, const GsRenderOptions *opt_in, int do_sort_flag, GsImage *rt,
             GsImage *tgt) {
  int rc = check_params(ctx, as, fp);
  if (rc) return rc;
  if (!rt && !tgt) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "gs_frame needs rt and/or camera_target");
  GsRenderOptions opt = opt_in ? *opt_in : default_opts();
  std::vector<CameraArgs> cams(1);
  CameraArgs &a = cams[0];
  a.off = 0; a.K = 1; a.rt = rt; a.tgt = tgt;
  a.fcs.assign(1, make_frame_consts(fp));
  if ((rc = check_options(ctx, a.fcs[0], opt))) return rc;
  a.W = (uint32_t)fp->screen_w;
  a.H = opt.band_packed ? partition_own_bin_rows(opt, a.fcs[0].binsY) * kBin : (uint32_t)fp->screen_h;
  if (opt.band_packed && tgt) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "band_packed output cannot be composited before the gather");
  if (opt.band_packed && rt && is_array_image(rt))
    return fail(ctx, GS_ERR_INVALID_ARGUMENT, "band_packed output is the send buffer of an all-gather: it must be linear memory, not a CUDA array");
  if (rt) { if ((rc = image_ok(ctx, rt, a.W, a.H, ImageRole::kRenderTarget, &a.rt_pitch))) return rc; a.rt_fmt = rt->format; }
  return draw_cameras(ctx, cams, &as, fp, &do_sort_flag, opt);
}

int gs_frame_objects(GsContext *ctx, uint32_t object_count, GsAsset *const *assets, const GsFrameParams *fps, const int32_t *do_sort_flags,
                     const GsRenderOptions *opt_in, GsImage *rt, GsImage *tgt) {
  if (!ctx || !assets || !fps || !do_sort_flags) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null context / assets / fps / do_sort");
  if (object_count == 0) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "object_count is 0");
  GsRenderOptions opt = opt_in ? *opt_in : default_opts();
  std::vector<CameraArgs> cams(1);
  cams[0].off = 0; cams[0].K = object_count; cams[0].rt = rt; cams[0].tgt = tgt;
  const int rc = check_camera(ctx, assets, fps, &opt, &cams[0]);
  if (rc) return rc;
  return draw_cameras(ctx, cams, assets, fps, do_sort_flags, opt);
}

int gs_frame_cameras(GsContext *ctx, uint32_t camera_count, const uint32_t *object_counts, GsAsset *const *assets, const GsFrameParams *fps,
                     const int32_t *do_sort_flags, const GsRenderOptions *opt_in, GsImage *const *rts, GsImage *const *camera_targets) {
  if (!ctx || !object_counts || !assets || !fps || !do_sort_flags || !rts || !camera_targets)
    return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null context / object_counts / assets / fps / do_sort / rts / camera_targets");
  if (camera_count == 0) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "camera_count is 0");
  GsRenderOptions opt = opt_in ? *opt_in : default_opts();
  if (opt.flags & GS_FLAG_ASYNC_READBACK)
    return fail(ctx, GS_ERR_INVALID_ARGUMENT, "GS_FLAG_ASYNC_READBACK is not accepted by gs_frame_cameras: its host images are read back before it returns");
  std::vector<CameraArgs> cams(camera_count);
  uint64_t pairs = 0;
  for (uint32_t c = 0; c < camera_count; ++c) {
    CameraArgs &a = cams[c];
    if (object_counts[c] == 0) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "a camera has no objects (leave it out: the reference draws nothing for it)");
    a.off = (uint32_t)pairs; a.K = object_counts[c]; a.rt = rts[c]; a.tgt = camera_targets[c];
    pairs += a.K;
    if (pairs > 0xFFFFFFFFu) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "more than 2^32 - 1 objects in all");
    GsRenderOptions o = opt;
    const int rc = check_camera(ctx, assets + a.off, fps + a.off, &o, &a);
    if (rc) return rc;
  }
  return draw_cameras(ctx, cams, assets, fps, do_sort_flags, opt);
}

// GS_UNITY_EVENT_FRAME_CAMERAS: the payload's by-value images as the GsImage * arrays gs_frame_cameras takes, on the stack
static void unity_frame_cameras_event(GsUnityFrameCamerasEvent *ev) {
  if (ev->camera_count > GS_UNITY_EVENT_MAX_CAMERAS) {
    ev->status = fail(ev->ctx, GS_ERR_INVALID_ARGUMENT, "more than GS_UNITY_EVENT_MAX_CAMERAS cameras in one event: issue one event per 64 cameras");
    return;
  }
  GsImage *rts[GS_UNITY_EVENT_MAX_CAMERAS], *tgts[GS_UNITY_EVENT_MAX_CAMERAS];
  for (uint32_t c = 0; c < ev->camera_count; ++c) {
    rts[c] = ev->rts && ev->rts[c].data ? const_cast<GsImage *>(&ev->rts[c]) : nullptr;
    tgts[c] = ev->camera_targets && ev->camera_targets[c].data ? const_cast<GsImage *>(&ev->camera_targets[c]) : nullptr;
  }
  ev->status = gs_frame_cameras(ev->ctx, ev->camera_count, ev->object_counts, ev->assets, ev->fps, ev->do_sort, &ev->options,
                                ev->rts ? rts : nullptr, ev->camera_targets ? tgts : nullptr);
}

int gs_unshuffle_bands(GsContext *ctx, const void *gathered, uint32_t parts, uint32_t band_rows, uint32_t rows_pp, uint32_t fmt,
                       GsImage *out) {
  if (!ctx || !gathered || !out || parts == 0) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null argument");
  if (is_array_image(out)) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "gs_unshuffle_bands writes host or linear device memory, not a CUDA array");
  uint32_t pitch = 0;
  int rc = image_ok(ctx, out, out->width, out->height, ImageRole::kRenderTarget, &pitch);
  if (rc) return rc;
  if (out->format != fmt) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "gathered and output pixel formats differ");
  const uint32_t W = out->width, H = out->height;
  const bool host = out->memory == GS_MEM_HOST;
  if (host) GS_CUDA_TRY(ctx, ctx->rt_scratch.reserve((size_t)W * pix_bytes(fmt) * H, {ctx->stream}));
  CallSurfaces surfs(ctx);
  DeviceImage o;
  if ((rc = bind_image(ctx, surfs, out, pitch, fmt, W, H, ctx->rt_scratch.get(), StagingFill::kNone, ctx->stream, &o))) return rc;
  launch_unshuffle(gathered, parts, band_rows, rows_pp, fmt, o.d_rt, o.pitch, W, H, ctx->stream);
  ctx->launches += 1;
  GS_CUDA_TRY(ctx, cudaGetLastError());
  if (host && (rc = copy_to_image(ctx, out, pitch, o.d_rt, o.pitch, W, H, ctx->stream))) return rc;
  if (host) GS_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return GS_OK;
}

// ---- stand-alone sorter ---------------------------------------------------------------------------
int gs_sort_pairs_device(GsContext *ctx, uint32_t *d_keys, uint32_t *d_payload, uint32_t count) {
  if (!ctx || (count && (!d_keys || !d_payload))) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null argument");
  if (count == 0) return GS_OK;
  if (count >= (1u << 30)) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "count must be < 2^30");
  int rc = ensure_sort_scratch(ctx, count);
  if (rc) return rc;
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_scalar.get(), &count, 4, cudaMemcpyHostToDevice, ctx->stream));
  for (int e = 0; e < EV_COUNT; ++e) ctx->ev_valid[e] = false;
  cudaEvent_t pe[5] = {ctx->ev[EV_SORT0], ctx->ev[EV_SORT1], ctx->ev[EV_SORT2], ctx->ev[EV_SORT3], ctx->ev[EV_SORT4]};
  rec(ctx, EV_BEGIN);
  GS_CUDA_TRY(ctx, launch_sort_pairs(d_keys, d_payload, ctx->d_scalar.get(), count, 4, 8, false, sort_scratch(ctx), ctx->stream, ctx->timing ? pe : nullptr));
  if (ctx->timing) for (int e = EV_SORT0; e <= EV_SORT4; ++e) ctx->ev_valid[e] = true;
  ctx->launches += 5;
  GS_CUDA_TRY(ctx, cudaGetLastError());
  return GS_OK;
}

int gs_sort_pairs_host(GsContext *ctx, uint32_t *keys, uint32_t *payload, uint32_t count) {
  if (!ctx || (count && (!keys || !payload))) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null argument");
  if (count == 0) return GS_OK;
  gs::Buffer<uint32_t> dk, dv;
  GS_CUDA_TRY(ctx, dk.reserve(count, {ctx->stream}));
  GS_CUDA_TRY(ctx, dv.reserve(count, {ctx->stream}));
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(dk.get(), keys, (size_t)count * 4, cudaMemcpyHostToDevice, ctx->stream));
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(dv.get(), payload, (size_t)count * 4, cudaMemcpyHostToDevice, ctx->stream));
  int rc = gs_sort_pairs_device(ctx, dk.get(), dv.get(), count);
  if (rc) return rc;
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(keys, dk.get(), (size_t)count * 4, cudaMemcpyDeviceToHost, ctx->stream));
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(payload, dv.get(), (size_t)count * 4, cudaMemcpyDeviceToHost, ctx->stream));
  GS_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return GS_OK;
}

// ---- test hooks -------------------------------------------------------------------------------------
static int readback(GsAsset *as, void *dst, const void *src, size_t bytes) {
  if (!as || !dst) return fail(as ? as->ctx : nullptr, GS_ERR_INVALID_ARGUMENT, "null argument");
  GsContext *ctx = as->ctx;
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  GS_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return GS_OK;
}
int gs_readback_order(GsAsset *as, uint32_t *dst) { return readback(as, dst, as ? as->order.get() : nullptr, as ? (size_t)as->av.n * 4 : 0); }
int gs_readback_keys(GsAsset *as, uint32_t *dst) { return readback(as, dst, as ? as->keys.get() : nullptr, as ? (size_t)as->av.n * 4 : 0); }
int gs_readback_view(GsAsset *as, void *dst) {
  if (as && !as->view_valid) return fail(as->ctx, GS_ERR_NOT_READY, "_SplatViewData is only materialised by gs_calc_view (gs_frame hands the draw its own records)");
  return readback(as, dst, as ? as->view.get() : nullptr, as ? (size_t)as->av.n * kViewStride : 0);
}
int gs_export_splats(GsContext *ctx, GsAsset *as, const GsCutout *cutouts, uint32_t cutout_count, uint32_t bake_transform, void *dst) {
  if (!ctx || !as || !dst || (cutout_count && !cutouts)) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null argument");
  if (as->ctx != ctx) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "asset belongs to another context");
  if (bake_transform) return fail(ctx, GS_ERR_UNSUPPORTED_FORMAT, "the baked export is a host pass over these records: call with bake_transform = 0, then gsa_bake_transform (gsplat_asset.h)");
  GS_CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  GsFrameParams fp;
  memset(&fp, 0, sizeof(fp));
  fp.cutouts = cutouts; fp.cutout_count = cutout_count;
  int rc = upload_frame_inputs(ctx, as, &fp, ctx->stream);
  if (rc != GS_OK) return rc;
  gs::Buffer<float> d_out;
  const size_t floats = (size_t)as->av.n * 62;
  GS_CUDA_TRY(ctx, d_out.reserve(floats, {ctx->stream}));
  launch_export_data(as->av, cutout_count, ctx->d_cutouts.get(), d_out.get(), ctx->stream);
  ctx->launches += 1;
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(dst, d_out.get(), floats * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  GS_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return GS_OK;
}

int gs_upload_order(GsAsset *as, const uint32_t *src) {
  if (!as || !src) return fail(as ? as->ctx : nullptr, GS_ERR_INVALID_ARGUMENT, "null argument");
  GS_CUDA_TRY(as->ctx, cudaMemcpyAsync(as->order.get(), src, (size_t)as->av.n * 4, cudaMemcpyHostToDevice, as->ctx->stream));
  GS_CUDA_TRY(as->ctx, cudaStreamSynchronize(as->ctx->stream));
  return GS_OK;
}

// ---- Unity render-thread entry: IssuePluginEventAndData -> gs_frame / gs_sync / gs_frame_objects / gs_frame_cameras / the
// group calls (gs_group.cu) ----
static void gs_unity_on_render_event(int event_id, void *data) {
  if (!data) return;
  switch (event_id) {
    case GS_UNITY_EVENT_FRAME_OBJECTS: {
      GsUnityFrameObjectsEvent *ev = static_cast<GsUnityFrameObjectsEvent *>(data);
      ev->status = gs_frame_objects(ev->ctx, ev->object_count, ev->assets, ev->fps, ev->do_sort, &ev->options, ev->has_rt ? &ev->rt : nullptr,
                                    ev->has_camera_target ? &ev->camera_target : nullptr);
      return;
    }
    case GS_UNITY_EVENT_FRAME_CAMERAS: unity_frame_cameras_event(static_cast<GsUnityFrameCamerasEvent *>(data)); return;
    case GS_UNITY_EVENT_GROUP_FRAME_OBJECTS: unity_group_frame_objects_event(static_cast<GsUnityGroupFrameObjectsEvent *>(data)); return;
    case GS_UNITY_EVENT_GROUP_SYNC: unity_group_sync_event(static_cast<GsUnityGroupSyncEvent *>(data)); return;
    default: break;
  }
  GsUnityFrameEvent *ev = static_cast<GsUnityFrameEvent *>(data);
  switch (event_id) {
    case GS_UNITY_EVENT_FRAME:
      ev->status = gs_frame(ev->ctx, ev->asset, &ev->params, &ev->options, ev->do_sort, ev->has_rt ? &ev->rt : nullptr,
                            ev->has_camera_target ? &ev->camera_target : nullptr);
      break;
    case GS_UNITY_EVENT_SYNC:
      ev->status = gs_sync(ev->ctx);
      break;
    default:
      ev->status = fail(ev->ctx, GS_ERR_INVALID_ARGUMENT, "unknown render event id");
  }
}
GsUnityRenderEventAndDataFunc gs_unity_get_render_event_func(void) { return gs_unity_on_render_event; }
uint32_t gs_unity_frame_event_size(void) { return (uint32_t)sizeof(GsUnityFrameEvent); }
uint32_t gs_unity_frame_objects_event_size(void) { return (uint32_t)sizeof(GsUnityFrameObjectsEvent); }
uint32_t gs_unity_frame_cameras_event_size(void) { return (uint32_t)sizeof(GsUnityFrameCamerasEvent); }
uint32_t gs_unity_group_frame_objects_event_size(void) { return (uint32_t)sizeof(GsUnityGroupFrameObjectsEvent); }
uint32_t gs_unity_group_sync_event_size(void) { return (uint32_t)sizeof(GsUnityGroupSyncEvent); }

int gs_debug_raster_stats(GsContext *ctx, uint64_t out[8]) {
  if (!ctx || !out) return GS_ERR_INVALID_ARGUMENT;
  memset(out, 0, 64);
  if (!g_raster_stats) return GS_ERR_NOT_READY;
  GS_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  GS_CUDA_TRY(ctx, cudaMemcpy(out, g_raster_stats, 64, cudaMemcpyDeviceToHost));
  return GS_OK;
}

int gs_debug_sort_phases(GsContext *ctx, uint64_t *out, uint32_t max_words, uint32_t *tiles) {
  if (!ctx || !tiles) return GS_ERR_INVALID_ARGUMENT;
  *tiles = g_sort_phase_tiles;
  if (!g_sort_phases) return GS_ERR_NOT_READY;
  const size_t all = (size_t)4 * g_sort_phase_tiles * 8, words = max_words < all ? max_words : all;
  if (words && !out) return GS_ERR_INVALID_ARGUMENT;
  GS_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (words) GS_CUDA_TRY(ctx, cudaMemcpy(out, g_sort_phases, words * 8, cudaMemcpyDeviceToHost));
  return GS_OK;
}

void *gs_context_stream(GsContext *ctx) { return ctx ? (void *)ctx->stream : nullptr; }
void *gs_asset_device_ptr(GsAsset *as, int which) {
  if (!as) return nullptr;
  const GsBlobs &b = *as->blobs;
  switch (which) {
    case 0: return as->order.get();
    case 1: return as->keys.get();
    case 2: return as->view.get();
    case 3: return b.pos.get();
    case 4: return b.other.get();
    case 5: return b.sh.get();
    case 6: return b.color.get();
    case 7: return b.chunks.get();
    default: return nullptr;
  }
}

}  // extern "C"
