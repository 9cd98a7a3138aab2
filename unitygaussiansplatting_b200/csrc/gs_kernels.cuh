// gs_kernels.cuh -- declarations shared between the .cu translation units.
#pragma once
#include <utility>

#include "gs_common.cuh"

namespace gs {

// Bin rect sentinel: x0 = 255 > x1 = 0, which no rectangle footprint_tile_rect makes can be.  (All ones would be the
// one-bin rectangle at bin (255, 255), which exists on screens wider and taller than 16320 px.)
constexpr uint32_t kRectEmpty = 0x000000FFu;

// Screen-space footprint of one splat, derived from its SplatViewData exactly the way the
// draw stage defines it (S/RenderGaussianSplats.shader:35-77; DESIGN.md "Raster rule").
struct SplatFootprint {
  float cx, cy;              // centre, pixels (D3D viewport: x right, y down)
  float i1x, i1y, i2x, i2y;  // axis / |axis|^2 : quad coordinates q = (dot(d,i1), dot(d,i2))
  float hx, hy;              // conservative half extents of the visible part, pixels
  float ca;                  // opacity (half -> float)
};

// `selected`: the splat's bit is set in _SplatSelectedBits, so the vertex shader hands the pixel shader col.a = -1 (:63-73)
// and the fragment's alpha comes from the gaussian alone (:87-101): the footprint is that of opacity 1, and the record
// carries ca = -1 as the marker.
__device__ __forceinline__ bool splat_footprint(float4 clip, float a1x, float a1y, float a2x, float a2y, float ca, float W,
                                                float H, SplatFootprint &fp, bool selected = false) {
  if (!(clip.w > 0.0f)) return false;  // behindCam -> NaN vertex -> primitive dropped (shader :41-45)
  if (!(ca >= 0.0f)) return false;     // CSCalcViewData never emits a negative opacity; NaN draws nothing
  const float ca_rec = selected ? -1.0f : ca;
  if (selected) ca = 1.0f;
  float ndx = __fdiv_rn(clip.x, clip.w), ndy = __fdiv_rn(clip.y, clip.w);
  float cx = fmaf(ndx, 0.5f, 0.5f) * W, cy = fmaf(ndy, -0.5f, 0.5f) * H;
  float ex = 2.0f * (fabsf(a1x) + fabsf(a2x)), ey = 2.0f * (fabsf(a1y) + fabsf(a2y));
  if (!(ex < 1.0e6f) || !(ey < 1.0e6f) || !(fabsf(cx) < 1.0e7f) || !(fabsf(cy) < 1.0e7f)) return false;
  // alpha = sat(exp(-r2) * ca) can only reach 1/255 if ca does (exp_neg(0) = 1.00000012)
  if (ca < 0.00392f) return false;
  float n1 = a1x * a1x + a1y * a1y, n2 = a2x * a2x + a2y * a2y;
  fp.cx = cx; fp.cy = cy;
  fp.i1x = __fdiv_rn(a1x, n1); fp.i1y = __fdiv_rn(a1y, n1);
  fp.i2x = __fdiv_rn(a2x, n2); fp.i2y = __fdiv_rn(a2y, n2);
  fp.ca = ca_rec;
  // visible part: the +-2 quad intersected with {r2 <= ln(255*ca)} (discard at alpha < 1/255)
  float r2 = fminf(__logf(ca * 255.0f) * 1.001f + 2.0e-3f, 8.0f);
  float rq = sqrtf(fmaxf(r2, 0.0f));
  float exE = rq * sqrtf(a1x * a1x + a2x * a2x), eyE = rq * sqrtf(a1y * a1y + a2y * a2y);
  fp.hx = fminf(ex, exE) * 1.0001f + 0.01f;
  fp.hy = fminf(ey, eyE) * 1.0001f + 0.01f;
  return true;
}

// ---- screen-tile partition helpers (multi-GPU, SURVEY 8e.1) ----------------------------------
// Two ways of giving one GPU a part of the screen:
//   interleaved (count > 1): 64-pixel bin rows r with (r / band) % count == index (GsRenderOptions.partition_*);
//   range       (range != 0): the contiguous 16-pixel raster-tile rows [t0, t1) (GsRenderOptions.row_begin/row_end) --
//                what the group path uses, with boundaries moved every frame by last frame's measured row costs.
struct Partition {
  uint32_t index, count, band;  // interleaved; count <= 1 and !range: everything is ours
  uint32_t range, t0, t1;       // range mode: own raster-tile rows
  __host__ __device__ uint32_t b0() const { return t0 / (kBin / kTile); }                          // first own bin row
  __host__ __device__ uint32_t b1() const { return (t1 + (kBin / kTile) - 1) / (kBin / kTile); }   // one past the last
  __host__ __device__ uint32_t own_rows_below(uint32_t y) const {  // # own bin rows in [0, y)
    if (range) { const uint32_t lo = b0(), hi = b1(); return y <= lo ? 0u : (y < hi ? y : hi) - lo; }
    if (count <= 1) return y;
    uint32_t cyc = band * count, q = y / cyc, r = y % cyc;
    uint32_t lo = index * band;
    uint32_t in = r > lo ? (r - lo < band ? r - lo : band) : 0u;
    return q * band + in;
  }
  __host__ __device__ bool owns(uint32_t y) const {
    if (range) return y >= b0() && y < b1();
    return count <= 1 || (y / band) % count == index;
  }
  __host__ __device__ uint32_t kth_own_row(uint32_t k) const {
    if (range) return b0() + k;
    if (count <= 1) return k;
    return ((k / band) * count + index) * band + (k % band);
  }
  // raster-tile rows: how many are ours, and the k-th of them
  __host__ __device__ uint32_t own_tile_rows(uint32_t binsY) const {
    return range ? t1 - t0 : own_rows_below(binsY) * (kBin / kTile);
  }
  __host__ __device__ uint32_t kth_own_tile_row(uint32_t k) const {
    if (range) return t0 + k;
    return kth_own_row(k / (kBin / kTile)) * (kBin / kTile) + (k % (kBin / kTile));
  }
};
inline Partition make_partition(const GsRenderOptions &o) {
  Partition p;
  p.count = o.partition_count;
  p.index = o.partition_count > 1 ? o.partition_index : 0;
  p.band = o.band_rows ? o.band_rows : 1;
  p.range = o.row_end > o.row_begin ? 1u : 0u;
  p.t0 = o.row_begin; p.t1 = o.row_end;
  if (p.range) { p.count = 0; p.index = 0; }
  return p;
}

// Pixel rows/cols whose centres can be touched -> inclusive rectangle of kBin-pixel bins packed x0|y0<<8|x1<<16|y1<<24
// (8 bits per index: 256 bins = 16384 px per axis, the largest screen check_params accepts).
// Range partitions clip the rows to their own pixel band first, so the rectangle holds own bin rows only.
__device__ __forceinline__ uint32_t footprint_tile_rect(const SplatFootprint &fp, const FrameConsts &fc, const Partition &part) {
  float x0 = fmaxf(ceilf(fp.cx - fp.hx - 0.5f), 0.0f), x1 = fminf(floorf(fp.cx + fp.hx - 0.5f), fc.screenW - 1.0f);
  float y0 = fmaxf(ceilf(fp.cy - fp.hy - 0.5f), 0.0f), y1 = fminf(floorf(fp.cy + fp.hy - 0.5f), fc.screenH - 1.0f);
  if (part.range) {
    y0 = fmaxf(y0, (float)(part.t0 * kTile));
    y1 = fminf(y1, (float)(part.t1 * kTile) - 1.0f);
  }
  if (!(x0 <= x1) || !(y0 <= y1)) return kRectEmpty;
  uint32_t tx0 = (uint32_t)x0 / kBin, tx1 = (uint32_t)x1 / kBin, ty0 = (uint32_t)y0 / kBin, ty1 = (uint32_t)y1 / kBin;
  return tx0 | (ty0 << 8) | (tx1 << 16) | (ty1 << 24);
}

__device__ __forceinline__ uint32_t rect_entries(uint32_t r, const Partition &p) {
  if (r == kRectEmpty) return 0;
  uint32_t x0 = r & 255u, y0 = (r >> 8) & 255u, x1 = (r >> 16) & 255u, y1 = r >> 24;
  uint32_t rows = p.own_rows_below(y1 + 1) - p.own_rows_below(y0);
  return rows * (x1 - x0 + 1);
}


// ---- launchers (each enqueues on `s`, returns nothing; errors surface via cudaGetLastError) ----
// A launch in the frame's chain: the kernel may be placed while its predecessor on `s` drains (programmatic stream
// serialization); it must keep the rules beside chain_wait() in gs_common.cuh.
template <typename... KArgs, typename... Args>
inline void chain_launch(void (*kern)(KArgs...), uint32_t grid, uint32_t block, size_t smem, cudaStream_t s, Args &&...args) {
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}
// Zeroes up to kClearSpans word ranges in one chained kernel: the per-frame clears of scratch that the frame's kernels count
// or tick into, without a memset node in the chain.  Spans with a null pointer or no words are skipped.
constexpr int kClearSpans = 4;
struct ClearSpans {
  uint32_t *ptr[kClearSpans];
  size_t words[kClearSpans];
};
// release_first: the successor is placed before the clear waits for its own predecessor (see k_calc_distances)
void launch_clear(const ClearSpans &spans, cudaStream_t s, bool release_first = false);
uint32_t sm_count();   // multiprocessors of the current device (queried once per device): sizes grid-stride and persistent grids
void launch_set_indices(uint32_t *order, uint32_t n, cudaStream_t s);
void launch_export_data(const AssetView &a, uint32_t cutoutCount, const GsCutout *cutouts, float *out, cudaStream_t s);  // gs_export.cu

// Key-range sharding of the depth sort over the GPUs of a group (SURVEY 8e.2); see k_calc_distances.
constexpr int kMaxSlabs = 16;
struct SlabArgs {
  uint32_t count, index;          // G slabs, and the one this GPU sorts
  const uint32_t *order_prev;     // last frame's draw order (replicated)
  uint32_t qpos[kMaxSlabs - 1];   // positions in order_prev whose splats' current keys are the G-1 splitters
  uint32_t *mask;                 // out: bit i = splat i belongs to slab `index`
  uint32_t *group_bits;           // out: bit j = some splat of [128 j, 128 j + 128) belongs to slab `index` (group_bits_words(n) words)
  uint32_t *info;                 // out (zeroed by the caller): [0, kMaxSlabs) ascending splitters, [kMaxSlabs, 2 kMaxSlabs) #{key >= splitter j}
};
void launch_calc_distances(const AssetView &a, const FrameConsts &fc, uint32_t *key_table, uint32_t *ghist, cudaStream_t s,
                           const SlabArgs *slabs = nullptr);
// block_bits: block_bits_words(n) words, bit j = some splat of [256 j, 256 j + 256) got a bin rectangle
inline size_t block_bits_words(uint32_t n) { return ((size_t)(n + 255) / 256 + 31) / 32 + 1; }
inline size_t group_bits_words(uint32_t n) { return ((size_t)(n + 127) / 128 + 31) / 32 + 1; }
void launch_calc_view(const AssetView &a, const FrameConsts &fc, const GsCutout *cutouts, const uint32_t *deleted, const uint32_t *selected, uint32_t *view,
                      uint32_t *rect, float4 *draw, uint32_t *block_bits, float *zndc /* per-splat quad depth, or nullptr */, bool cull_undrawable,
                      const Partition &part, cudaStream_t s, bool after_sort = false);
// (after_sort: the kernel before it on `s` is the depth sort of this asset, and the view-calc runs beside its last pass)

// Radix sort (gs_sort.cu).  Scratch layout is owned by the caller (gs_api.cu).
struct SortScratch {
  uint32_t *alt_keys, *alt_vals;  // ping-pong buffers, >= capacity elements each
  uint32_t *ghist;                // 4*256 digit counts (one row of 256 per pass; a single 9-bit pass uses the first 512)
  uint32_t *lookback;             // 1024 status words per tile: 4 passes x 256 digits or 1 pass x 512
  uint32_t *tickets;              // passes counters
  size_t lookback_words;          // size of `lookback`
};
constexpr uint32_t kSortTileItems = 8192;  // 512 threads x 16 keys
size_t sort_lookback_words(uint32_t capacity, int passes);
extern unsigned long long *g_sort_phases;   // diagnostics, see GS_SORT_PHASES
extern uint32_t g_sort_phase_tiles;
// Stable ascending LSD sort of (key,val) pairs on bits [0, bits*passes), bits in {5..8}, or one pass of 9 bits.  The count
// is read from d_count (device).  count_is_capacity: the host passes the exact count as `capacity` (exact grid); otherwise
// `capacity` only bounds the buffers and a persistent grid serves whatever d_count holds.
// ghist must already hold the per-pass digit counts when hist_ready, otherwise it is computed (4 x 8 or 1..2 x 5..8 bits
// only: a 9-bit pass needs hist_ready).  Each pass of a tile publishes 2^bits status words; `lookback` must hold
// passes * 2^bits words per 8192-pair tile.  An unsupported request launches nothing and returns cudaErrorInvalidValue.
// After an even number of passes the result is back in keys/vals -- unless final_keys/final_vals name where the last pass
// writes.  key_table != nullptr: the input keys are key_table[vals[i]] (gathered inside pass 0; `keys` is then output only).
// scratch_clear (count_is_capacity only): the caller has zeroed the passes' look-back rows and the 4 tickets.
cudaError_t launch_sort_pairs(uint32_t *keys, uint32_t *vals, const uint32_t *d_count, uint32_t capacity, int passes, int bits, bool hist_ready,
                       const SortScratch &sc, cudaStream_t s, cudaEvent_t *pass_events = nullptr, const uint32_t *key_table = nullptr,
                       bool count_is_capacity = true, uint32_t *final_keys = nullptr, uint32_t *final_vals = nullptr,
                       bool scratch_clear = false);
// (out_ids, out_keys) = (id, key_table[id]) of the ids of order[0..n) whose mask bit is set, order kept; *count_out = how many.
// group_bits (one bit per 128 ids, kept in shared memory) lets whole groups be skipped without reading their mask words.
// status: compact_status_words(n) words of scratch.
size_t compact_status_words(uint32_t n);
void launch_compact_order(const uint32_t *order, uint32_t n, const uint32_t *mask, const uint32_t *group_bits, const uint32_t *key_table,
                          uint32_t *out_ids, uint32_t *out_keys, uint32_t *status, uint32_t *count_out, cudaStream_t s);

// Binning + raster + composite (gs_raster.cu)
struct BinScratch {
  uint32_t *block_sums;    // [0] block ticket, [1..] look-back status of the fused count+scan+emit kernel
  uint32_t *entry_count;   // [0] = (tile,splat) entries clamped to capacity, [1] = overflow flag, [2] = unclamped total
  uint32_t *tile_keys, *tile_vals;  // capacity entries each
  uint32_t *bin_ranges;    // uint2 [start,end) per bin
  uint32_t *tile_cost, *tile_order;   // per raster tile: last frame's cost, this frame's launch order
  uint32_t capacity;
};
// A run: several (camera, object) pairs, at most kRunObjects, drawn by one bin list, one bin sort and one k_raster<..., MULTI>
// pass.  Each pair's object has fewer than 2^kSlotShift splats; its entries are tagged (slot << kSlotShift) | splat id, slot
// being the pair's index in the run.  A single object is drawn by gs_frame's kernels instead (launch_binning, launch_raster).
constexpr uint32_t kRunObjects = 16, kSlotShift = 28, kLocalIdMask = (1u << kSlotShift) - 1u;
// What the MULTI raster reads of the run's pairs (a kernel parameter).
struct DrawObjects {
  const float4 *draw[kRunObjects];   // raster records
  const float *zndc[kRunObjects];    // quad depths, where the pair is depth-tested
  uint32_t depth_mask;               // bit k: pair k is depth-tested against its camera's scene depth buffer
  uint32_t count;
  bool extras;                       // some pair has a selection or is depth-tested: the raster's SEL instantiation
};
struct NoRasterObjects {};
// One object's (bin id, splat id) list, sorted by bin id.  *sorted: the scratch view whose tile_keys / tile_vals hold it
// (launch_raster's input).  clear_overflow: the list sets the flag entry_count[1], else only ever sets it (BinList decides).
cudaError_t launch_binning(const FrameConsts &fc, const GsRenderOptions &opt, const uint32_t *order, const uint32_t *rect,
                           const uint32_t *block_bits, uint32_t n, bool clear_overflow, const BinScratch &bs, const SortScratch &sc,
                           cudaStream_t s, BinScratch *sorted, int *launches);

// The surface of a CUDA-array image: a 2-D array (GS_MEM_ARRAY, layer -1), read and written with surf2Dread / surf2Dwrite, or
// one layer of a layered array (GS_MEM_ARRAY_LAYER), read and written with surf2DLayeredread / surf2DLayeredwrite.  Pixel
// (px, py) of the image is texel (x + px, y + py): the rectangle's origin of a GS_MEM_ARRAY_RECT image, 0 for a whole array.
struct Surface {
  cudaSurfaceObject_t obj = 0;
  int32_t layer = -1;
  uint32_t x = 0, y = 0;
};
// The scene depth buffer a draw is tested against, W x H float32 texels, texel (x, y) the depth of pixel (x, y): linear device
// memory at `ptr` (rows tightly packed), or, with `on_surface`, a one-channel float32 CUDA array (layer) behind `surf`.  Neither:
// no depth test.
struct SceneDepth {
  const float *ptr = nullptr;
  Surface surf;
  bool on_surface = false;
  __host__ __device__ bool bound() const { return ptr != nullptr || on_surface; }
};

// The cameras of a run, in shared memory in the MULTI raster.  A run is a list of camera segments: camera c's pairs of the run
// own the bin ids [bin_base, bin_base + its bins) and the raster tiles [tile_base, tile_base + its tiles).  A run of one camera
// has bin_base = tile_base = 0.
struct RasterCamera {
  uint8_t *rt;                 // linear device image, or nullptr: the CUDA array behind `surf`
  Surface surf;
  const float *depth;          // the camera's scene depth buffer in linear device memory, or nullptr (see DepthSurfaces)
  uint32_t pitch, tile_base, bin_base, ntx, binsX, W, H;
  uint32_t load;               // 1: blend under what the image holds (the camera's earlier run drew it); 0: the image starts cleared
};
struct DrawCameras {
  RasterCamera cam[kRunObjects];
  uint32_t count;
};
// The run's scene depth buffers that are CUDA arrays (layers): with bit c of on_surface, camera c's depth is the array behind
// surf[c] rather than cam[c].depth.  A parameter of the MULTI raster's SEL instantiations only, after the camera table, so that
// the others keep their parameter layout and code.
struct DepthSurfaces {
  Surface surf[kRunObjects];
  uint32_t on_surface;
};
// The run's binning, in three steps around its pairs' sorts and view-calcs (a pair's emit must come before a later sort or
// view-calc of the same asset overwrites order / rect / block_bits):
//   launch_bin_list_begin: empties the list and zeroes `ghist`, the digit histograms the emits count into;
//   launch_bin_emit_pair:  appends one pair's entries, keys offset by its camera's bin_base, values tagged with its slot;
//   launch_bin_list_sort:  the stable sort of the list by bin id, over `bins` bins, with the histograms in `ghist`.
void launch_bin_list_begin(const BinScratch &bs, uint32_t *ghist, cudaStream_t s);
void launch_bin_emit_pair(const uint32_t *order, const uint32_t *rect, const uint32_t *block_bits, uint32_t n, uint32_t binsX,
                          uint32_t bin_base, uint32_t slot, bool clear_overflow, uint32_t bins, const BinScratch &bs, uint32_t *ghist,
                          cudaStream_t s);
cudaError_t launch_bin_list_sort(uint32_t bins, const BinScratch &bs, SortScratch sc, uint32_t *ghist, cudaStream_t s, BinScratch *sorted,
                                 int *launches);
// k_bin_ranges over the run's bins, k_tile_order over its raster tiles (history indexed by tile_base + tile), and the raster.
// Every render target of the run has rt_format.
void launch_raster_cameras(const DrawObjects &objs, const DrawCameras &cams, const DepthSurfaces &depth_surfs, uint32_t bins,
                           uint32_t tiles, uint32_t blend_mode, uint32_t rt_format, const BinScratch &bs, cudaStream_t s);
// One object's raster: records `draw`, quad depths `zndc` (when depth-tested), `extras`: a selection or a scene depth buffer
// (the SEL instantiation).  scene_depth: the W x H depth buffer it is tested against (none: no test).  opt: tile partition,
// band_packed, blend mode and GS_FLAG_LOAD_RT.  Images here are linear device memory (pointer, pitch) or, when the pointer is
// null, a CUDA array behind a surface object.
void launch_raster(const FrameConsts &fc, const GsRenderOptions &opt, const float4 *draw, const float *zndc, bool extras,
                   const BinScratch &bs, void *rt, uint32_t rt_pitch_bytes, uint32_t rt_format, Surface rt_surf, cudaStream_t s,
                   const SceneDepth &scene_depth);
extern unsigned long long *g_raster_stats;   // diagnostics, see GS_RASTER_STATS
uint32_t partition_own_bin_rows(const GsRenderOptions &opt, uint32_t binsY);
uint32_t partition_own_tile_rows(const GsRenderOptions &opt, uint32_t binsY);
void launch_unshuffle(const void *gathered, uint32_t parts, uint32_t band, uint32_t rows_pp, uint32_t fmt, void *out, uint32_t pitch,
                      uint32_t W, uint32_t H, cudaStream_t s);
void launch_composite(const void *rt, uint32_t rt_pitch, Surface rt_surf, uint32_t rt_format, void *target, uint32_t tgt_pitch,
                      Surface tgt_surf, uint32_t tgt_format, uint32_t W, uint32_t H, cudaStream_t s);

}  // namespace gs
