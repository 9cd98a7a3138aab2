// gs_internal.cuh -- what gs_api.cu (single GPU) and gs_group.cu (several GPUs) share behind the C ABI:
// the context / asset objects and the per-stage drivers.
#pragma once
#include <string>

#include <nvtx3/nvToolsExt.h>   // header-only; costs one predicted-not-taken branch per range when no tool is attached

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
int fail(GsContext *ctx, int code, const std::string &msg);
int fail_cuda(GsContext *ctx, cudaError_t e, const char *expr, const char *file, int line);
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
  // sort scratch
  gs::SortScratch sort{};
  uint32_t sort_capacity = 0;
  size_t lookback_words = 0;
  uint32_t *d_scalar = nullptr;  // small device scalars (standalone sorter count)
  // bin scratch
  gs::BinScratch bin{};
  uint32_t bin_blocks_cap = 0, tiles_cap = 0, raster_tiles_cap = 0, raster_tiles_cur = 0;
  // image scratch
  void *rt_scratch = nullptr;
  size_t rt_bytes = 0;
  void *tgt_scratch = nullptr;
  size_t tgt_bytes = 0;
  // asynchronous read-back (GS_FLAG_ASYNC_READBACK): two device staging images, a copy stream, and the events that order
  // "raster k -> copy k" and "copy k -> raster k+2 may reuse the staging image"
  cudaStream_t copy_stream = nullptr;
  void *rt_async[2] = {nullptr, nullptr};
  size_t rt_async_bytes[2] = {0, 0};
  cudaEvent_t ev_rt_ready[2]{}, ev_copy_done[2]{};
  bool copy_pending[2] = {false, false};
  int rt_flip = 0;
  // per-frame optional inputs
  GsCutout *d_cutouts = nullptr;
  uint32_t cutout_cap = 0;
  uint32_t *d_deleted = nullptr;
  size_t deleted_words = 0;
  uint32_t *d_selected = nullptr;
  size_t selected_words = 0;
  float *d_depth = nullptr;          // the frame's scene depth buffer when it was handed over in host memory
  size_t depth_bytes = 0;
  const float *cur_depth = nullptr;  // what the compositor tests against this frame (nullptr: no depth test)
  uint32_t launches = 0;
  uint64_t pack_stats[4] = {0, 0, 0, 0};   // gs_debug_pack_stats
};

struct GsAsset {
  GsContext *ctx = nullptr;
  gs::AssetView av{};
  void *d_pos = nullptr, *d_other = nullptr, *d_sh = nullptr, *d_color = nullptr, *d_chunks = nullptr;
  uint32_t *order = nullptr, *keys = nullptr, *key_table = nullptr, *view = nullptr, *rect = nullptr, *d_n = nullptr;
  uint32_t *block_bits = nullptr;  // bit j: some splat of block j (256 splats) got a bin rectangle from the last view-calc
  // group path only (allocated by gs_group_*): slab membership (bit per splat, byte per 128), compaction output / sort ping-pong payload
  uint32_t *slab_mask = nullptr, *order_tmp = nullptr;
  float *zndc = nullptr;           // per-splat quad depth clip.z / clip.w, written by view-calc when a scene depth buffer is bound
  bool zndc_valid = false;
  uint32_t *order_alt = nullptr;   // peer-to-peer order exchange: `order` and `order_alt` alternate as last / new draw order
  uint32_t *slab_group_bits = nullptr;
  float4 *draw = nullptr;  // raster-ready 48-byte records of the drawable splats
  bool view_valid = false;   // the full 40-byte _SplatViewData buffer is current (gs_calc_view)
  bool draw_valid = false;   // draw records + bin rects are current (gs_calc_view or gs_frame)
  uint32_t draw_part[3] = {0, 0, 1};   // the tile partition those records were culled for (count <= 1: complete)
  uint32_t view_w = 0, view_h = 0;
};

namespace gs {
FrameConsts make_frame_consts(const GsFrameParams *fp);
int check_params(GsContext *ctx, GsAsset *as, const GsFrameParams *fp);
int check_options(GsContext *ctx, const FrameConsts &fc, GsRenderOptions &opt);
int ensure_sort_scratch(GsContext *ctx, uint32_t capacity);
int upload_frame_inputs(GsContext *ctx, GsAsset *as, const GsFrameParams *fp, cudaStream_t stream);
int bind_depth(GsContext *ctx, const GsFrameParams *fp, cudaStream_t stream);   // sets ctx->cur_depth for the draw that follows
int do_view(GsContext *ctx, GsAsset *as, const GsFrameParams *fp, const FrameConsts &fc, bool cull, const GsRenderOptions &opt,
            cudaStream_t stream);
int do_render(GsContext *ctx, GsAsset *as, const FrameConsts &fc, const GsRenderOptions &opt, void *d_rt, uint32_t pitch, uint32_t fmt);
int image_ok(GsContext *ctx, const GsImage *im, uint32_t W, uint32_t H, uint32_t *pitch);
uint32_t pix_bytes(uint32_t fmt);
// The per-asset work buffers (order, keys, view data, ...) of an asset whose blobs as->d_* are already in HBM, the format
// fields of as->av, and CSSetIndices: what gs_asset_upload and gs_pack_asset share.
cudaError_t asset_init_work(GsContext *ctx, GsAsset *as, uint32_t n, uint32_t pos_fmt, uint32_t scale_fmt, uint32_t sh_fmt,
                            uint32_t col_fmt, uint32_t chunk_count);
void rec(GsContext *ctx, int e);
void launch_row_costs(const uint32_t *cost, uint32_t ntx, uint32_t t0, uint32_t t1, uint32_t *row_cost, cudaStream_t s);   // gs_raster.cu
}  // namespace gs
