// gs_raster.cu -- tile binning, front-to-back compositing and the final composite pass.
//
// The reference draws one instanced quad per splat through the hardware rasteriser with
// fixed-function blending `Blend OneMinusDstAlpha One` into an RGBA16F target
// (S/RenderGaussianSplats.shader:10-12,35-108; draw call R/GaussianSplatRenderer.cs:156-165).
// A CUDA device has neither rasteriser nor ROP, so the same pixels are produced by:
//   1. bin   -- walk the splats in sorted order; each emits one (bin id, splat id) entry per
//               64x64-pixel bin its visible footprint can touch (rect written by k_calc_view).
//               Bins are coarser than the 16x16 raster tiles on purpose: 2.5x fewer entries to
//               emit and sort, and the per-warp ballot cull below makes a foreign entry cost 1/32
//               of an evaluation.  Emission order == depth order, so one STABLE radix sort by
//               bin id (one onesweep pass up to 512 bins, e.g. 1920x1080 = 510 bins, else 2
//               passes) yields per-bin lists that are already in draw order.  No 64-bit
//               (tile|depth) re-sort of duplicated keys.
//   2. raster-- one CTA per tile, one pixel per thread.  The tile's list is consumed in
//               batches of 256 raster-ready records (written by k_calc_view) that land in shared
//               memory by cp.async, double buffered; every warp owns an 8x4 pixel block and
//               first culls a batch against that block with one ballot per 32 splats, so
//               small splats cost 1/32 of a pixel evaluation where they do not land.
//               Blending reproduces the ROP: dst = src*(1-dst.a) + dst, rounded to half after
//               every splat (GS_BLEND_FP16_ROP) -- or kept in float32 (GS_BLEND_FP32).
//   3. composite (S/GaussianComposite.shader:35-39).
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "gs_kernels.cuh"
#include "gs_packed_float.cuh"
#include "gs_srgb8.cuh"

namespace gs {

constexpr int kBinItems = 8;                  // ranks per thread
constexpr int kBinBlock = 256 * kBinItems;    // ranks per block

// ---- 1. count + scan + emit in ONE pass ---------------------------------------------------------
// Blocks take their index by atomic ticket, publish their entry total with a LOCAL flag, resolve
// their exclusive offset by a warp-parallel decoupled look-back (32 predecessors per probe, gs_common.cuh), then
// emit (tile id, splat id) entries in depth order.
enum : uint32_t { kBinFlagLocal = kLbLocal, kBinFlagIncl = kLbIncl, kBinValMask = kLbMask };

__device__ __forceinline__ uint32_t entry_tile(uint32_t e, uint32_t r, const Partition &p, uint32_t tilesX) {
  const uint32_t x0 = r & 255u, y0 = (r >> 8) & 255u, x1 = (r >> 16) & 255u;
  const uint32_t w = x1 - x0 + 1;
  uint32_t krow = 0, col = e;
  if (e >= w) { krow = e / w; col = e - krow * w; }
  const uint32_t ty = p.count <= 1 ? y0 + krow : p.kth_own_row(p.own_rows_below(y0) + krow);
  return ty * tilesX + x0 + col;
}

// APPEND (one pair of a run, see DrawCameras): the entries go behind the entry_count[2] already listed, each key is the bin
// id plus key_base (the camera's first bin in the run) and each value is tagged `tag | splat id` (tag = the pair's slot <<
// kSlotShift).  clear_overflow: the overflow flag entry_count[1] is set from this list's total; otherwise it is only ever set.
template <bool APPEND>
__global__ void __launch_bounds__(256) k_bin_emit(const uint32_t *__restrict__ order, const uint32_t *__restrict__ rect,
                                                  const uint32_t *__restrict__ block_bits, uint32_t bits_words, uint32_t n, Partition part,
                                                  uint32_t tilesX, volatile uint32_t *status,
                                                  uint32_t *ticket, uint32_t capacity, uint32_t *__restrict__ keys,
                                                  uint32_t *__restrict__ vals, uint32_t *__restrict__ entry_count,
                                                  uint32_t *__restrict__ ghist, uint32_t digit_bits, bool two_pass, bool clear_overflow,
                                                  uint32_t tag, uint32_t key_base) {
  extern __shared__ uint32_t s_bits[];   // the view kernel's block bitmap (bits_words words), or nothing when it is too large to hold
  __shared__ uint32_t s_w[8];
  __shared__ uint32_t s_block, s_excl, s_base;
  chain_wait();   // nothing before the wait: the ticket, the list's length and block_bits / rect all come from predecessors
  chain_release();
  if (APPEND && threadIdx.x == 0) {
    // read before this block publishes its status: the last block writes the new total only after every block has published
    s_base = *(volatile uint32_t *)(entry_count + 2);
    __threadfence();
  }
  __shared__ uint32_t s_dh[512];   // digit histograms of the sort by the bin ids we emit: [0,256) pass 0 and [256,512) pass 1
                                   // of two passes, or all 512 for one pass of up to 9 bits (ghist's layout)
  __shared__ uint2 s_items[kBinBlock];     // per warp: its drawable ranks, squeezed together in order
  __shared__ uint32_t s_pre[kBinBlock];
  const uint32_t nblocks = (n + kBinBlock - 1) / kBinBlock;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_block = atomicAdd(ticket, 1u);
  for (uint32_t i = threadIdx.x; i < bits_words; i += 256) s_bits[i] = __ldg(block_bits + i);
  s_dh[threadIdx.x] = 0; s_dh[threadIdx.x + 256] = 0;
  const uint32_t dmask = (1u << digit_bits) - 1u;
  __syncthreads();
  const uint32_t b = s_block;
  // warp-striped ranks: item i of lane l is rank wbase + i*32 + l (coalesced loads; the warp's 256 ranks are consecutive)
  const uint32_t wbase = b * kBinBlock + warp * (32 * kBinItems) + lane;
  uint32_t id[kBinItems], rc[kBinItems];
#pragma unroll
  for (int i = 0; i < kBinItems; ++i) {
    const uint32_t r = wbase + i * 32;
    id[i] = (r < n) ? __ldg(order + r) : 0xFFFFFFFFu;
  }
  // the rectangle of a splat is a random 4-byte gather; the view kernel's per-block bits (in shared memory) say where there
  // is nothing to fetch
#pragma unroll
  for (int i = 0; i < kBinItems; ++i) {
    rc[i] = kRectEmpty;
    if (id[i] != 0xFFFFFFFFu) {
      const uint32_t bw = bits_words ? s_bits[id[i] >> 13] : __ldg(block_bits + (id[i] >> 13));
      if ((bw >> ((id[i] >> 8) & 31u)) & 1u) rc[i] = __ldg(rect + id[i]);
    }
  }
  // Most ranks have nothing to emit (70 % of cfg2's splats draw nothing; in a group of G only 1/G of the rest is ours).
  // The warp first squeezes its drawable ranks, in order, into shared memory, and everything below -- entry counts, prefix
  // scans, the emission loop -- runs over those K <= 256 items in chunks of 32 instead of over 8 sparse slots.
  uint2 *w_items = s_items + warp * (32 * kBinItems);     // (splat id, rect)
  uint32_t *w_pre = s_pre + warp * (32 * kBinItems);      // exclusive prefix of the item's entries inside its chunk
  const uint32_t lt = (1u << lane) - 1u;
  uint32_t K = 0;
#pragma unroll
  for (int i = 0; i < kBinItems; ++i) {
    const bool has = rect_entries(rc[i], part) != 0;
    const uint32_t bal = __ballot_sync(0xffffffffu, has);
    if (has) w_items[K + __popc(bal & lt)] = make_uint2(id[i], rc[i]);
    K += __popc(bal);
  }
  __syncwarp();
  const uint32_t nchunks = (K + 31) >> 5;
  uint32_t ctot[kBinItems];   // entries of chunk j (warp-uniform)
  uint32_t wsum = 0;
#pragma unroll
  for (int j = 0; j < kBinItems; ++j) {
    ctot[j] = 0;
    if ((uint32_t)j < nchunks) {
      const uint32_t k = j * 32 + lane;
      const uint32_t c = k < K ? rect_entries(w_items[k].y, part) : 0u;
      uint32_t inc = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= (uint32_t)o) inc += t;
      }
      w_pre[k] = inc - c;
      ctot[j] = __shfl_sync(0xffffffffu, inc, 31);
      wsum += ctot[j];
    }
  }
  if (lane == 0) s_w[warp] = wsum;
  __syncthreads();
  uint32_t woff = 0, total = 0;
#pragma unroll
  for (uint32_t w = 0; w < 8; ++w) {
    const uint32_t c = s_w[w];
    if (w < warp) woff += c;
    total += c;
  }
  if (warp == 0) {
    if (lane == 0) status[b] = (b == 0 ? kBinFlagIncl : kBinFlagLocal) | total;
    uint32_t excl = 0;
    if (b > 0) {
      excl = lookback_exclusive(status, b);
      // prefixes saturate instead of wrapping at 2^30: a saturated total is > any capacity, so it is reported as overflow
      if (lane == 0) status[b] = kBinFlagIncl | min(excl + total, (uint32_t)kBinValMask);
    }
    if (lane == 0) {
      if (APPEND) excl = min(s_base + excl, (uint32_t)kBinValMask);
      s_excl = excl;
      if (b == nblocks - 1) {
        const uint32_t all = min(excl + total, (uint32_t)kBinValMask);
        if (clear_overflow) entry_count[1] = all > capacity ? 1u : 0u;   // overflow: lists are truncated, the API reports it
        else if (all > capacity) entry_count[1] = 1u;
        entry_count[0] = all > capacity ? capacity : all;
        entry_count[2] = all;
      }
    }
  }
  __syncthreads();
  // Emission is warp-cooperative: the 32 items of a chunk own one contiguous output range; lane x of the warp writes entry x
  // of that range (owner found by a 5-step shuffle search over the lanes' prefix sums), so every store is a full coalesced
  // line regardless of how many bins each splat touches.
  uint32_t off = s_excl + woff;
#pragma unroll
  for (int j = 0; j < kBinItems; ++j) {
    if ((uint32_t)j >= nchunks) break;
    const uint32_t k = j * 32 + lane;
    const uint2 it = k < K ? w_items[k] : make_uint2(0xFFFFFFFFu, kRectEmpty);
    const uint32_t pre = k < K ? w_pre[k] : 0xFFFFFFFFu;   // lanes past the end never own an entry
    const uint32_t T = ctot[j];
    for (uint32_t e0 = 0; e0 < T; e0 += 32) {
      const uint32_t x = e0 + lane;
      // owner = last lane whose exclusive prefix is <= x
      uint32_t lo = 0, hi = 31;
#pragma unroll
      for (int step = 0; step < 5; ++step) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        const uint32_t pm = __shfl_sync(0xffffffffu, pre, mid);
        if (pm <= x) lo = mid; else hi = mid - 1;
      }
      const uint32_t opre = __shfl_sync(0xffffffffu, pre, lo);
      const uint32_t orc = __shfl_sync(0xffffffffu, it.y, lo);
      const uint32_t oid = __shfl_sync(0xffffffffu, it.x, lo);
      const uint32_t o = off + x;
      if (x < T && o < capacity) {
        const uint32_t tile = entry_tile(x - opre, orc, part, tilesX) + (APPEND ? key_base : 0u);
        keys[o] = tile;
        vals[o] = APPEND ? (tag | oid) : oid;
        atomicAdd(&s_dh[tile & dmask], 1u);
        if (two_pass) atomicAdd(&s_dh[256 + ((tile >> digit_bits) & dmask)], 1u);
      }
    }
    off += T;
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < 512; i += 256) {
    const uint32_t c = s_dh[i];
    if (c) atomicAdd(&ghist[i], c);
  }
}

// digit width and pass count of the stable sort by bin id: one pass while the bin count fits a digit (<= 512 bins, e.g.
// 1200x797 = 19x13 in 8 bits, 1920x1080 = 30x17 in 9), else two passes of the narrowest digit that covers it, up to two
// 8-bit passes for 65536 bins (16384x16384).  The 8-bit plan's digit histograms are ghist's first two rows of 256 and its
// look-back 2 x 256 words per tile, within the depth sort's allocation (4 x 256).
static void bin_sort_plan(uint32_t bins, int *bits, int *passes) {
  if (bins <= 512u) { *passes = 1; *bits = bins <= 32u ? 5 : bins <= 64u ? 6 : bins <= 128u ? 7 : bins <= 256u ? 8 : 9; return; }
  *passes = 2;
  *bits = bins <= 1024u ? 5 : bins <= 4096u ? 6 : bins <= 16384u ? 7 : 8;
}

// the sort by bin id of a list whose digit histograms are in sc.ghist; an odd number of passes leaves it in the sorter's
// ping-pong buffers
static cudaError_t sort_bin_list(int bits, int passes, const BinScratch &bs, const SortScratch &sc, cudaStream_t s, BinScratch *sorted) {
  // the entry count lives on the device: a persistent grid sorts whatever it is (no capacity-sized grid or memset)
  const cudaError_t e = launch_sort_pairs(bs.tile_keys, bs.tile_vals, bs.entry_count, bs.capacity, passes, bits, true, sc, s, nullptr,
                                          nullptr, /*count_is_capacity=*/false);
  if (e != cudaSuccess) return e;
  if (passes & 1) { sorted->tile_keys = sc.alt_keys; sorted->tile_vals = sc.alt_vals; }
  return cudaSuccess;
}

// the shared-memory copy of the view kernel's block bitmap (0 words: read through L1)
static uint32_t bin_bits_words(uint32_t n) {
  static int bits_global = -1;   // GS_WALK_BITS_GLOBAL=1 forces the large-asset path (bitmap read through L1) for tests
  if (bits_global < 0) { const char *e = getenv("GS_WALK_BITS_GLOBAL"); bits_global = (e && e[0] == '1') ? 1 : 0; }
  uint32_t words = (uint32_t)block_bits_words(n);
  if (bits_global) words = 0;
  if (words * 4u > 16u * 1024u) words = 0;   // beside the kernel's 28 KB of static shared memory only 20 KB of the default 48
                                              // remain: a larger bitmap (> 33 M splats) is read through L1 instead
  return words;
}

void launch_bin_list_begin(const BinScratch &bs, uint32_t *ghist, cudaStream_t s) {
  ClearSpans cl = {};
  cl.ptr[0] = bs.entry_count + 2; cl.words[0] = 1;   // the pairs append behind an empty list
  cl.ptr[1] = ghist; cl.words[1] = 4 * 256;
  launch_clear(cl, s);
}

// the look-back clear and k_bin_emit of one object's entries, counted into ghist by the digit plan of `bins` bins
template <bool APPEND>
static void bin_emit(const uint32_t *order, const uint32_t *rect, const uint32_t *block_bits, uint32_t n, const Partition &part,
                     uint32_t binsX, uint32_t bins, bool clear_overflow, uint32_t tag, uint32_t key_base, const BinScratch &bs,
                     uint32_t *ghist, cudaStream_t s, uint32_t *clear_ghist = nullptr) {
  int bits, passes;
  bin_sort_plan(bins, &bits, &passes);
  const uint32_t nblocks = (n + kBinBlock - 1) / kBinBlock, words = bin_bits_words(n);
  ClearSpans cl = {};
  cl.ptr[0] = bs.block_sums; cl.words[0] = (size_t)nblocks + 1;   // [0] ticket, [1..] look-back status
  cl.ptr[1] = clear_ghist; cl.words[1] = 4 * 256;
  launch_clear(cl, s);
  chain_launch(k_bin_emit<APPEND>, nblocks, 256, words * 4u, s, order, rect, block_bits, words, n, part, binsX, bs.block_sums + 1,
               bs.block_sums, bs.capacity, bs.tile_keys, bs.tile_vals, bs.entry_count, ghist, (uint32_t)bits, passes == 2, clear_overflow,
               tag, key_base);
}

void launch_bin_emit_pair(const uint32_t *order, const uint32_t *rect, const uint32_t *block_bits, uint32_t n, uint32_t binsX,
                          uint32_t bin_base, uint32_t slot, bool clear_overflow, uint32_t bins, const BinScratch &bs, uint32_t *ghist,
                          cudaStream_t s) {
  bin_emit<true>(order, rect, block_bits, n, Partition{0, 0, 1, 0, 0, 0}, binsX, bins, clear_overflow, slot << kSlotShift, bin_base, bs,
                 ghist, s);
}

cudaError_t launch_bin_list_sort(uint32_t bins, const BinScratch &bs, SortScratch sc, uint32_t *ghist, cudaStream_t s, BinScratch *sorted,
                                 int *launches) {
  int bits, passes;
  bin_sort_plan(bins, &bits, &passes);
  *sorted = bs;
  *launches = passes;
  sc.ghist = ghist;
  return sort_bin_list(bits, passes, bs, sc, s, sorted);
}

cudaError_t launch_binning(const FrameConsts &fc, const GsRenderOptions &opt, const uint32_t *order, const uint32_t *rect,
                           const uint32_t *block_bits, uint32_t n, bool clear_overflow, const BinScratch &bs, const SortScratch &sc,
                           cudaStream_t s, BinScratch *sorted, int *launches) {
  const uint32_t bins = fc.binsX * fc.binsY;
  // the digit histograms are the depth sort's: cleared with the emit's look-back, after the view-calc (and so the sort) completed
  bin_emit<false>(order, rect, block_bits, n, make_partition(opt), fc.binsX, bins, clear_overflow, 0u, 0u, bs, sc.ghist, s, sc.ghist);
  const cudaError_t e = launch_bin_list_sort(bins, bs, sc, sc.ghist, s, sorted, launches);
  *launches += 2;   // look-back clear, bin_emit
  return e;
}

// ---- 2. raster ---------------------------------------------------------------------------------
__device__ __forceinline__ float round_half(float v) { return __half2float(__float2half_rn(v)); }

// first index in sorted keys[0,m) whose key is >= target; all 32 lanes of a warp cooperate
__device__ __forceinline__ uint32_t lower_bound32(const uint32_t *__restrict__ keys, uint32_t m, uint32_t target, uint32_t lane) {
  uint32_t lo = 0, hi = m;
  while (hi - lo > 32) {
    const uint32_t len = hi - lo;
    const uint32_t p = lo + (uint32_t)(((uint64_t)len * (lane + 1)) / 33);   // lo < p < hi, increasing with lane
    const uint32_t below = __ballot_sync(0xffffffffu, __ldg(keys + p) < target);
    const int c = __popc(below);                                             // predicate is monotone over lanes
    const uint32_t p_lo = __shfl_sync(0xffffffffu, p, c > 0 ? c - 1 : 0), p_hi = __shfl_sync(0xffffffffu, p, c < 32 ? c : 31);
    if (c > 0) lo = p_lo + 1;
    if (c < 32) hi = p_hi;
  }
  const uint32_t p = lo + lane;
  const uint32_t below = __ballot_sync(0xffffffffu, p < hi && __ldg(keys + p) < target);
  return lo + __popc(below);
}

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async4(void *smem_dst, const void *gmem_src) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// one warp per bin: [start,end) of the bin's entries in the sorted list, by two 32-ary searches (5 probes for 10M entries)
__global__ void __launch_bounds__(256) k_bin_ranges(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ entry_count,
                                                    uint32_t bins, uint2 *__restrict__ ranges) {
  const uint32_t bin = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  chain_wait();   // the sorted list and its length come from the bin sort
  chain_release();
  if (bin >= bins) return;
  const uint32_t m = __ldg(entry_count);
  const uint32_t a = lower_bound32(keys, m, bin, lane), b = lower_bound32(keys, m, bin + 1, lane);
  if (lane == 0) ranges[bin] = make_uint2(a, b);
}

// Launch order of the raster tiles: longest-processing-time first, from the cost each tile measured last frame
// (counting sort over 64 log-scale buckets, one CTA).  Pixels do not depend on the order; only the tail does.
__global__ void __launch_bounds__(1024) k_tile_order(const uint32_t *__restrict__ cost, uint32_t ntiles, uint32_t ntx, Partition part,
                                                     uint32_t *__restrict__ order) {
  // `cost` is indexed by the tile's id in the whole image (ty * ntx + tx) so that a moving partition keeps its history;
  // `order` receives the ids of OUR ntiles tiles (own tile row k = kth_own_tile_row(k)), most expensive first
  __shared__ uint32_t s_hist[64], s_base[64];
  __shared__ uint32_t s_any;
  // The whole body runs before the wait, beside the bin sort: it reads only tile_cost, last written by an earlier frame's
  // raster, and writes only tile_order, last read by that raster -- both completed before this frame's first kernel began.
  // Releasing at once is safe because the successor (k_bin_ranges) waits before it does anything.
  chain_release();
  if (threadIdx.x < 64) s_hist[threadIdx.x] = 0;
  if (threadIdx.x == 0) s_any = 0;
  __syncthreads();
  auto bucket = [](uint32_t c) -> uint32_t {   // 0 for cost 0, else 2*log2 resolution, descending order wanted
    if (c == 0) return 0u;
    const uint32_t l = 31u - (uint32_t)__clz(c);
    const uint32_t half = l ? ((c >> (l - 1)) & 1u) : 0u;
    return min(63u, 1u + 2u * l + half);
  };
  auto global_id = [&](uint32_t t) -> uint32_t { const uint32_t k = t / ntx; return part.kth_own_tile_row(k) * ntx + (t - k * ntx); };
  for (uint32_t t = threadIdx.x; t < ntiles; t += 1024) {
    const uint32_t c = cost[global_id(t)];
    if (c) s_any = 1;
    atomicAdd(&s_hist[63u - bucket(c)], 1u);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    for (int b = 0; b < 64; ++b) { s_base[b] = run; run += s_hist[b]; }
  }
  __syncthreads();
  if (!s_any) {   // no history (first frame / new resolution): a stride permutation spreads spatial clusters
    for (uint32_t t = threadIdx.x; t < ntiles; t += 1024) order[t] = global_id((ntiles % 1031u) ? (uint32_t)(((uint64_t)t * 1031u) % ntiles) : t);
  } else {
    for (uint32_t t = threadIdx.x; t < ntiles; t += 1024) {
      const uint32_t gid = global_id(t);
      order[atomicAdd(&s_base[63u - bucket(cost[gid])], 1u)] = gid;
    }
  }
  chain_wait();
}

// per raster-tile row: the sum of its tiles' costs (what the group path balances its row ranges with).  accumulate != 0 adds
// the sums to what row_cost holds: several splat objects drawn into one target are balanced on their summed cost.
__global__ void __launch_bounds__(256) k_row_costs(const uint32_t *__restrict__ cost, uint32_t ntx, uint32_t t0, uint32_t t1,
                                                   uint32_t *__restrict__ row_cost, uint32_t accumulate) {
  const uint32_t row = t0 + blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= t1) return;
  uint32_t acc = 0;
  for (uint32_t x = lane; x < ntx; x += 32) acc += cost[row * ntx + x];
#pragma unroll
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) row_cost[row] = accumulate ? row_cost[row] + acc : acc;
}
void launch_row_costs(const uint32_t *cost, uint32_t ntx, uint32_t t0, uint32_t t1, uint32_t *row_cost, cudaStream_t s, bool accumulate) {
  if (t1 > t0) k_row_costs<<<(t1 - t0 + 7) / 8, 256, 0, s>>>(cost, ntx, t0, t1, row_cost, accumulate ? 1u : 0u);
}

// Can any pixel centre of the 8x4 block centred on (bcx, bcy) lie inside the splat's quad, |qa| <= 2 and |qb| <= 2 with
// q = (dot(d, i1), dot(d, i2))?  (A = cx, cy, i1x, i1y; i2 = (i2x, i2y).)  The pixel centres lie within 3.5 / 1.5 pixels of
// the block's centre, so each q of a pixel differs from its value at the centre by at most r = 3.5 |ix| + 1.5 |iy|.  Both
// evaluations round, by far less than 1e-5 of the magnitudes involved, and that much is added to the bound.  A candidate
// this test drops is one for which the per-pixel test finds no pixel inside, so the candidates that are evaluated, and
// their order, are unchanged; it only saves the candidate loop's quad test for splats whose box touches the block but
// whose quad does not.  A NaN keeps the candidate.
__device__ __forceinline__ bool block_may_touch_quad(const float4 &A, float i2x, float i2y, float bcx, float bcy) {
  const float dxc = bcx - A.x, dyc = A.y - bcy;   // as the per-pixel test: pixel y grows down, NDC y up
  auto axis_ok = [&](float ix, float iy) {
    const float tx = dxc * ix, ty = dyc * iy;
    const float r = 3.5f * fabsf(ix) + 1.5f * fabsf(iy);
    const float bound = 2.0f + r;
    const float slack = 1e-5f * (fabsf(tx) + fabsf(ty) + bound);
    return !(fabsf(tx + ty) > bound + slack);
  };
  return axis_ok(A.z, A.w) && axis_ok(i2x, i2y);
}

// The texel of a CUDA-array image that holds the pixel at byte column x_bytes (a multiple of sizeof(T), the texel size), row y:
// offset by the surface's origin, through surf2D* on a 2-D array, surf2DLayered* on a layer of a layered one.  LAYERED false:
// the image is known to be a 2-D array, and only the 2-D call is compiled.
template <bool LAYERED, class T>
__device__ __forceinline__ void surf_load(T *v, const Surface &s, uint32_t x_bytes, uint32_t y) {
  x_bytes += s.x * (uint32_t)sizeof(T);
  y += s.y;
  if (LAYERED && s.layer >= 0) surf2DLayeredread(v, s.obj, (int)x_bytes, (int)y, s.layer);
  else surf2Dread(v, s.obj, (int)x_bytes, (int)y);
}
template <bool LAYERED, class T>
__device__ __forceinline__ void surf_store(const T &v, const Surface &s, uint32_t x_bytes, uint32_t y) {
  x_bytes += s.x * (uint32_t)sizeof(T);
  y += s.y;
  if (LAYERED && s.layer >= 0) surf2DLayeredwrite(v, s.obj, (int)x_bytes, (int)y, s.layer);
  else surf2Dwrite(v, s.obj, (int)x_bytes, (int)y);
}

// SEL ("extras"): a separate instantiation for frames with an edit selection and / or a scene depth buffer bound, so that
// ordinary frames pay nothing.  Selected splats (records with opacity -1) take the pixel shader's other branch
// (S/RenderGaussianSplats.shader:87-101); with `scene_depth` every fragment is depth-tested like the pass's ZTest LEqual
// (reversed Z: quad depth >= stored depth), the per-splat quad depths being staged beside the records.  The scene depth is read
// once per pixel, from linear memory or a CUDA array (layer), by a branch that is uniform over the grid.  The other
// instantiations take an unused null pointer in its place.
// SURF: the target is a CUDA array, read and written through `surf` instead of `rt`/`pitch`: 1, a 2-D array (GS_MEM_ARRAY);
// 2, some target is one layer of a layered array (GS_MEM_ARRAY_LAYER; surf.layer picks the surface call at the load and the
// store).  Separate instantiations, so that the linear and the 2-D array ones keep their code.
// MULTI: a run (DrawCameras) of several (camera, object) pairs.  The list holds every pair's entries, each tagged with its slot
// in `objs`; the records are gathered from that pair's buffers, and each camera's result is what drawing its objects one after
// the other leaves.  The grid covers every camera's tiles; a tile finds its camera c in `cams`, which gives it the screen size, bins, image (pointer and pitch, or a surface when the pointer is null), scene depth buffer and load
// flag that the other instantiations take from fc and the image arguments.  The camera's bin ids start at its bin_base in
// bin_ranges; tile_cost is indexed by tile_base + the tile.  SURF: some camera's image is a CUDA array.  MULTI with SEL is held
// to 32 registers, 8 CTAs per SM, which its shared memory also fits (selected runs measured 20 % slower at 7); so is SEL into a
// layer (SURF 2), which the rectangle origin of its surface accesses would otherwise take to 38 registers, 6 CTAs per SM.
template <bool FP16_ROP, int OUT_FMT, bool STATS, bool SEL = false, int SURF = 0, bool MULTI = false>
__global__ void __launch_bounds__(256, SEL && (MULTI || SURF == 2) ? 8 : 0)
k_raster(FrameConsts fc, Partition part, const float4 *__restrict__ draw, const uint2 *__restrict__ bin_ranges,
         const uint32_t *__restrict__ tile_vals, const uint32_t *__restrict__ tile_order, uint32_t *__restrict__ tile_cost, uint32_t ntx,
         uint8_t *__restrict__ rt, uint32_t pitch, Surface surf, uint32_t band_packed, uint32_t load_rt,
         unsigned long long *stats, const float *__restrict__ zndc, std::conditional_t<SEL, SceneDepth, const float *> scene_depth,
         std::conditional_t<MULTI, DrawObjects, NoRasterObjects> objs, std::conditional_t<MULTI, DrawCameras, NoRasterObjects> cams,
         std::conditional_t<MULTI && SEL, DepthSurfaces, NoRasterObjects> depth_surfs) {
  uint32_t st_batches = 0, st_culls = 0, st_cand = 0, st_eval = 0, st_blend = 0;   // GS_RASTER_STATS diagnostics (per warp)
  unsigned long long st_t0 = 0;
  chain_wait();   // nothing before the wait: the bin ranges come from the predecessor
  chain_release();
  if (STATS) asm volatile("mov.u64 %0, %globaltimer;" : "=l"(st_t0));
  // two staging buffers of 256 raster records (3 x float4 each, planar [buf][plane][entry]): batch k+1 lands
  // asynchronously while batch k is composited
  __shared__ __align__(128) float4 s_rec[2][3][256];  // plane 0: cx, cy, i1x, i1y   1: i2x, i2y, opacity, hx   2: r, g, b, hy
  __shared__ float s_z[SEL ? 2 : 1][SEL ? 256 : 1];   // quad depths of the staged batch (depth test only)
  // MULTI: the object table, staged where a slot can index it without local memory, and each staged entry's slot
  __shared__ const float4 *s_draw[MULTI ? kRunObjects : 1];
  __shared__ const float *s_zndc[MULTI ? kRunObjects : 1];
  __shared__ uint8_t s_slot[MULTI ? 2 : 1][MULTI ? 256 : 1];
  // MULTI: the tile's first tile / bin in the run, and its camera (found again where it is used, so that nothing of it is held
  // in registers across the blend loop)
  uint32_t lin = 0, tile_base = 0, bin_base = 0;
  auto camera_index = [&](const auto &cs) -> uint32_t {   // (generic: instantiated only where MULTI calls it)
    uint32_t c = 0;
    for (uint32_t k = 1; k < cs.count; ++k) if (lin >= cs.cam[k].tile_base) c = k;
    return c;
  };
  auto camera = [&](const auto &cs) -> const RasterCamera & { return cs.cam[camera_index(cs)]; };
  bool depth_test = false;   // MULTI: the tile's camera's
  if constexpr (SEL) depth_test = scene_depth.bound();
  if constexpr (MULTI) {
    if (threadIdx.x < objs.count) { s_draw[threadIdx.x] = objs.draw[threadIdx.x]; s_zndc[threadIdx.x] = objs.zndc[threadIdx.x]; }
    __syncthreads();
    lin = __ldg(tile_order + blockIdx.x);
    const RasterCamera &cam = camera(cams);
    fc.screenW = (float)cam.W; fc.screenH = (float)cam.H; fc.binsX = cam.binsX;
    ntx = cam.ntx; load_rt = cam.load;
    if constexpr (SEL) depth_test = cam.depth != nullptr || ((depth_surfs.on_surface >> camera_index(cams)) & 1u);   // the buffer itself is found again at its one load
    tile_base = cam.tile_base; bin_base = cam.bin_base;
  }
  bool surf_io = SURF != 0;
  auto camera_image = [&]() {
    if constexpr (MULTI) { const RasterCamera &cam = camera(cams); rt = cam.rt; pitch = cam.pitch; surf = cam.surf; surf_io = SURF != 0 && rt == nullptr; }
  };
  // FP32 blending into an RGBA16F target: drawing the objects one after the other stores (rounds to half) each object's result
  // and the next object starts from it.  Rounding is idempotent, so rounding at the next object's first candidate is exact.
  constexpr bool kRoundAtObject = MULTI && !FP16_ROP && OUT_FMT == GS_PIX_RGBA16F;
  uint32_t depth_mask = 0, cur_slot = 0;

  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // 1-D grid over raster tiles: tile = (16-pixel column, R * own 64-pixel bin row + tile row inside that bin row)
  constexpr uint32_t R = kBin / kTile;   // raster tiles per bin edge
  // launch order != raster order: CTA i takes tile order[i] (k_tile_order: most expensive first, by last frame's cost),
  // so the expensive tiles start early instead of forming the tail
  if (!MULTI) lin = __ldg(tile_order + blockIdx.x);   // tile id in the whole image: ty * ntx + tx (MULTI: in the run)
  const uint32_t ty = (lin - tile_base) / ntx;
  const uint32_t tx = (lin - tile_base) - ty * ntx, brow = ty / R;
  if (ty * kTile >= (uint32_t)fc.screenH) { if (threadIdx.x == 0) tile_cost[lin] = 0; return; }
  __shared__ uint32_t s_cost;
  if (threadIdx.x == 0) s_cost = 0;
  if constexpr (MULTI) depth_mask = objs.depth_mask;
  // [start,end) of this tile's bin in the bin-sorted entry list (k_bin_ranges); R*R tiles share one list
  const uint2 range = __ldg(bin_ranges + bin_base + brow * fc.binsX + (tx / R));
  const uint32_t bx = tx * kTile + (warp & 1) * 8, by = ty * kTile + (warp >> 1) * 4;
  const uint32_t px = bx + (lane & 7), py = by + (lane >> 3);
  const float pxc = (float)px + 0.5f, pyc = (float)py + 0.5f;
  const float bcx = (float)bx + 4.0f, bcy = (float)by + 2.0f;
  const bool in_image = px < (uint32_t)fc.screenW && py < (uint32_t)fc.screenH;

  float d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;  // ClearRenderTarget(0,0,0,0), R/GaussianSplatRenderer.cs:196
  // whether any splat blended into this pixel: under GS_FLAG_LOAD_RT a pixel nothing blends into is not written, so it keeps
  // the words it was loaded with (the ROP writes only where a fragment blends; the half -> float -> half round trip would
  // replace a NaN's payload with the canonical NaN)
  bool blended = false;
  // the scene's depth at this pixel (depth target bound at R/GaussianSplatRenderer.cs:195; ZTest LEqual, ZWrite Off)
  float zscene = 0.0f;
  if constexpr (SEL) {
    if (depth_test && in_image) {
      const size_t at = (size_t)py * (uint32_t)fc.screenW + px;
      if constexpr (MULTI) {
        const uint32_t c = camera_index(cams);
        if ((depth_surfs.on_surface >> c) & 1u) surf_load<true>(&zscene, depth_surfs.surf[c], px * 4u, py);
        else zscene = __ldg(cams.cam[c].depth + at);
      } else if (scene_depth.on_surface) {
        surf_load<true>(&zscene, scene_depth.surf, px * 4u, py);
      } else {
        zscene = __ldg(scene_depth.ptr + at);
      }
    }
  }
  // where this pixel lives in the target (band-packed: own bin row k of an interleaved partition -> rows [64k, 64k+64))
  const uint32_t out_row = band_packed ? part.own_rows_below(brow) * kBin + (py - brow * kBin) : py;
  if (load_rt && in_image) {
    // GS_FLAG_LOAD_RT: the target was cleared once and earlier renderers of this camera already drew into it
    // (R/GaussianSplatRenderer.cs:111-168 loops the active splat objects over ONE _GaussianSplatRT); blend under what is there
    camera_image();
    const uint8_t *row = rt + (size_t)out_row * pitch;
    if (OUT_FMT == GS_PIX_RGBA16F) {
      uint2 v;
      if (surf_io) surf_load<SURF == 2>(&v, surf, px * 8u, out_row);
      else v = reinterpret_cast<const uint2 *>(row)[px];
      d0 = f16lo(v.x); d1 = f16hi(v.x); d2 = f16lo(v.y); d3 = f16hi(v.y);
    } else {
      float4 v;
      if (surf_io) surf_load<SURF == 2>(&v, surf, px * 16u, out_row);
      else v = reinterpret_cast<const float4 *>(row)[px];
      d0 = v.x; d1 = v.y; d2 = v.z; d3 = v.w;
    }
  }

  // three-deep pipeline: splat ids of batch k+2 (register) -> records of batch k+1 (cp.async in flight) -> batch k (composited)
  auto load_id = [&](uint32_t e) -> uint32_t { return e < range.y ? __ldg(tile_vals + e) : 0xFFFFFFFFu; };
  auto stage = [&](int buf, uint32_t id) {
    if constexpr (MULTI) {
      if (id != 0xFFFFFFFFu) {
        const uint32_t slot = id >> kSlotShift, lid = id & kLocalIdMask;
        s_slot[buf][tid] = (uint8_t)slot;
        const float4 *src = s_draw[slot] + (size_t)lid * 3;
        cp_async16(&s_rec[buf][0][tid], src);
        cp_async16(&s_rec[buf][1][tid], src + 1);
        cp_async16(&s_rec[buf][2][tid], src + 2);
        if (SEL && depth_test && s_zndc[slot]) cp_async4(&s_z[SEL ? buf : 0][SEL ? tid : 0], s_zndc[slot] + lid);
      }
    } else if (id != 0xFFFFFFFFu) {
      const float4 *src = draw + (size_t)id * 3;
      cp_async16(&s_rec[buf][0][tid], src);
      cp_async16(&s_rec[buf][1][tid], src + 1);
      cp_async16(&s_rec[buf][2][tid], src + 2);
      if (SEL && depth_test) cp_async4(&s_z[SEL ? buf : 0][SEL ? tid : 0], zndc + id);
    }
    cp_async_commit();
  };
  uint32_t id_next = load_id(range.x + tid);
  stage(0, id_next);
  id_next = load_id(range.x + 256 + tid);

  int buf = 0;
  for (uint32_t base = range.x; base < range.y; base += 256, buf ^= 1) {
    stage(buf ^ 1, id_next);                       // batch k+1 -> other buffer (free since the barrier that ended batch k-1)
    id_next = load_id(base + 512 + tid);           // ids of batch k+2
    cp_async_wait<1>();                            // batch k has landed (this thread's copies) ...
    __syncthreads();                               // ... and everyone else's
    const float4 *s_a = s_rec[buf][0], *s_b = s_rec[buf][1], *s_c = s_rec[buf][2];

    const uint32_t cnt = min(256u, range.y - base);
    ++st_batches;
    for (uint32_t c0 = 0; c0 < cnt; c0 += 32) {
      // a warp whose 32 pixels all reached dst.a == 1 ignores everything behind exactly: skip the batch remainder
      if (__all_sync(0xffffffffu, d3 == 1.0f || !in_image)) break;
      if (STATS) ++st_culls;
      // one ballot culls 32 splats against this warp's 8x4 pixel block
      const uint32_t e = c0 + lane;
      bool hit = false;
      if (e < cnt) {
        const float4 A = s_a[e];
        const float hx = s_b[e].w, hy = s_c[e].w;
        hit = (fabsf(A.x - bcx) <= hx + 3.5f) && (fabsf(A.y - bcy) <= hy + 1.5f);
        if (hit) {
          const float4 B = s_b[e];
          hit = block_may_touch_quad(A, B.x, B.y, bcx, bcy);
        }
      }
      uint32_t mask = __ballot_sync(0xffffffffu, hit);
      while (mask) {
        const uint32_t j = c0 + __ffs(mask) - 1;
        mask &= mask - 1;
        if (STATS) ++st_cand;
        const float4 A = s_a[j], B = s_b[j];
        const float dx = pxc - A.x, dy = A.y - pyc;  // pixel y grows down, NDC y up
        const float qa = fmaf(dy, A.w, dx * A.z), qb = fmaf(dy, B.y, dx * B.x);
        const bool inside = (fabsf(qa) <= 2.0f) && (fabsf(qb) <= 2.0f);  // quad corners at +-2 (:54-55)
        if (!__any_sync(0xffffffffu, inside)) continue;
        uint32_t slot = 0;
        if constexpr (MULTI) {
          slot = s_slot[buf][j];
          if (kRoundAtObject && slot != cur_slot) {
            cur_slot = slot;
            d0 = round_half(d0); d1 = round_half(d1); d2 = round_half(d2); d3 = round_half(d3);
          }
        }
        ++st_eval;
        const float power = -fmaf(qb, qb, qa * qa);                       // -dot(i.pos, i.pos) (:81)
        float alpha = exp_neg(power);                                     // half alpha = exp(power) (:82)
        bool tint = false, outline = false;
        if (SEL && B.z < 0.0f) {                                          // "selected": outline, more opacity, magenta tint (:87-101)
          tint = true;
          if (alpha > 7.0f / 255.0f) {
            if (alpha < 10.0f / 255.0f) { alpha = 1.0f; outline = true; }
            alpha = __saturatef(alpha + 0.3f);
          }
        } else {
          alpha = __saturatef(alpha * B.z);                               // :83-86 (saturate: NaN -> 0, one instruction)
        }
        // discard below 1/255 (:103-104); a pixel with dst.a == 1 ignores every later splat, as the early-outs assume: a zero
        // blend factor contributes nothing, even to an inf colour (DESIGN §4)
        bool pass = inside && alpha >= 0.003921569f && d3 != 1.0f;
        if (SEL && depth_test && (!MULTI || ((depth_mask >> slot) & 1u)))
          pass = pass && (s_z[SEL ? buf : 0][SEL ? j : 0] >= zscene);   // ZTest LEqual, reversed Z (MULTI: objects that bind it)
        if (pass) {
          if (STATS) ++st_blend;
          float4 C = s_c[j];
          if (SEL && tint) {
            if (outline) { C.x = 1.0f; C.y = 0.0f; C.z = 1.0f; }
            C.x = lerpf(C.x, 1.0f, 0.5f); C.y = lerpf(C.y, 0.0f, 0.5f); C.z = lerpf(C.z, 1.0f, 0.5f);
          }
          const float om = 1.0f - d3;                                     // Blend OneMinusDstAlpha One (:11)
          float n0 = fmaf(C.x * alpha, om, d0), n1 = fmaf(C.y * alpha, om, d1), n2 = fmaf(C.z * alpha, om, d2),
                n3 = fmaf(alpha, om, d3);
          if (FP16_ROP) {  // the ROP stores half: round every channel (two packed f32x2 -> f16x2 conversions)
            const float2 lo = __half22float2(__floats2half2_rn(n0, n1)), hi = __half22float2(__floats2half2_rn(n2, n3));
            n0 = lo.x; n1 = lo.y; n2 = hi.x; n3 = hi.y;
          }
          d0 = n0; d1 = n1; d2 = n2; d3 = n3;
          blended = true;
        }
      }
    }
    // a pixel whose dst.a == 1 ignores every later splat exactly (src*0 + dst): safe early out.  The barrier also
    // frees this batch's buffer for the copies issued at the top of the next-but-one iteration.
    if (__syncthreads_and(d3 == 1.0f || !in_image)) break;
  }
  cp_async_wait<0>();
  // this tile's cost for next frame's launch order: the slowest warp's work (evaluations dominate, culls and batches add)
  if (lane == 0) atomicMax(&s_cost, st_eval * 4 + st_batches * 16 + 1);
  __syncthreads();
  if (threadIdx.x == 0) tile_cost[lin] = s_cost;
  if (STATS) {
    const uint32_t bl = __reduce_add_sync(0xffffffffu, st_blend);
    if (lane == 0) {
      atomicAdd(stats + 0, (unsigned long long)st_batches); atomicAdd(stats + 1, (unsigned long long)st_culls);
      atomicAdd(stats + 2, (unsigned long long)st_cand); atomicAdd(stats + 3, (unsigned long long)st_eval);
      atomicAdd(stats + 4, (unsigned long long)bl); atomicAdd(stats + 5, (unsigned long long)(range.y - range.x));
      unsigned long long t1;
      asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
      atomicAdd(stats + 6, t1 - st_t0);
      atomicMax(stats + 7, t1 - st_t0);
    }
  }

  if (in_image && (blended || !load_rt)) {
    camera_image();
    uint8_t *row = rt + (size_t)out_row * pitch;
    if (OUT_FMT == GS_PIX_RGBA16F) {
      uint2 o;
      o.x = f32tof16(d0) | (f32tof16(d1) << 16);
      o.y = f32tof16(d2) | (f32tof16(d3) << 16);
      if (surf_io) surf_store<SURF == 2>(o, surf, px * 8u, out_row);
      else reinterpret_cast<uint2 *>(row)[px] = o;
    } else {
      if (surf_io) surf_store<SURF == 2>(make_float4(d0, d1, d2, d3), surf, px * 16u, out_row);
      else reinterpret_cast<float4 *>(row)[px] = make_float4(d0, d1, d2, d3);
    }
  }
}

unsigned long long *g_raster_stats = nullptr;

void launch_raster(const FrameConsts &fc, const GsRenderOptions &opt, const float4 *draw, const float *zndc, bool extras,
                   const BinScratch &bs, void *rt, uint32_t rt_pitch_bytes, uint32_t rt_format, Surface rt_surf, cudaStream_t s,
                   const SceneDepth &scene_depth) {
  const Partition part = make_partition(opt);
  const uint32_t rows = part.own_tile_rows(fc.binsY);
  if (!rows || !fc.binsX) return;
  const uint32_t ntx = ((uint32_t)fc.screenW + kTile - 1) / kTile, ntiles = ntx * rows;
  const uint32_t grid = ntiles;
  chain_launch(k_tile_order, 1, 1024, 0, s, bs.tile_cost, ntiles, ntx, part, bs.tile_order);
  const bool rop = opt.blend_mode == GS_BLEND_FP16_ROP;
  uint8_t *out = reinterpret_cast<uint8_t *>(rt);
  // GS_RASTER_STATS=1: per-frame work counters of a one-object draw (diagnostics; printed by tools/raster_stats.py through
  // gs_debug_raster_stats)
  static unsigned long long *stats = nullptr;
  static int want = -1;
  if (want < 0) { const char *e = getenv("GS_RASTER_STATS"); want = (e && e[0] == '1') ? 1 : 0; }
  if (want && !stats) { cudaMalloc(&stats, 64); g_raster_stats = stats; }
  if (stats) cudaMemsetAsync(stats, 0, 64, s);
  const uint32_t bins = fc.binsX * fc.binsY;
  uint2 *ranges = reinterpret_cast<uint2 *>(bs.bin_ranges);
  const uint32_t packed = part.range ? 0u : opt.band_packed, load = (opt.flags & GS_FLAG_LOAD_RT) ? 1u : 0u;
  chain_launch(k_bin_ranges, (bins + 7) / 8, 256, 0, s, bs.tile_keys, bs.entry_count, bins, ranges);
#define GS_RASTER_ARGS(DEPTH)                                                                                                    \
  grid, 256, 0, s, fc, part, draw, ranges, bs.tile_vals, bs.tile_order, bs.tile_cost, ntx, out, rt_pitch_bytes, rt_surf, packed,  \
      load, stats, zndc, DEPTH, NoRasterObjects{}, NoRasterObjects{}, NoRasterObjects{}
#define GS_LAUNCH_RASTER(ROP, FMT, SURF)                                                                                        \
  do {                                                                                                                         \
    if (extras) chain_launch(k_raster<ROP, FMT, false, true, SURF>, GS_RASTER_ARGS(scene_depth));                              \
    else if (stats) chain_launch(k_raster<ROP, FMT, true, false, SURF>, GS_RASTER_ARGS(nullptr));                              \
    else chain_launch(k_raster<ROP, FMT, false, false, SURF>, GS_RASTER_ARGS(nullptr));                                        \
  } while (0)
  // a null `rt` means the target is a CUDA array behind rt_surf
#define GS_LAUNCH_RASTER_TARGET(ROP, FMT)                                                                                       \
  do {                                                                                                                         \
    if (out) GS_LAUNCH_RASTER(ROP, FMT, 0);                                                                                    \
    else if (rt_surf.layer < 0) GS_LAUNCH_RASTER(ROP, FMT, 1);                                                                 \
    else GS_LAUNCH_RASTER(ROP, FMT, 2);                                                                                        \
  } while (0)
  if (rt_format == GS_PIX_RGBA16F) {
    if (rop) GS_LAUNCH_RASTER_TARGET(true, GS_PIX_RGBA16F); else GS_LAUNCH_RASTER_TARGET(false, GS_PIX_RGBA16F);
  } else {
    if (rop) GS_LAUNCH_RASTER_TARGET(true, GS_PIX_RGBA32F); else GS_LAUNCH_RASTER_TARGET(false, GS_PIX_RGBA32F);
  }
#undef GS_LAUNCH_RASTER_TARGET
#undef GS_LAUNCH_RASTER
#undef GS_RASTER_ARGS
}

void launch_raster_cameras(const DrawObjects &objs, const DrawCameras &cams, const DepthSurfaces &depth_surfs, uint32_t bins,
                           uint32_t tiles, uint32_t blend_mode, uint32_t rt_format, const BinScratch &bs, cudaStream_t s) {
  const Partition whole{0, 0, 1, 0, 0, 0};
  // without a partition a tile's id is its launch-order id: ntx = tiles puts all of them in row 0
  chain_launch(k_tile_order, 1, 1024, 0, s, bs.tile_cost, tiles, tiles, whole, bs.tile_order);
  uint2 *ranges = reinterpret_cast<uint2 *>(bs.bin_ranges);
  chain_launch(k_bin_ranges, (bins + 7) / 8, 256, 0, s, bs.tile_keys, bs.entry_count, bins, ranges);
  FrameConsts fc;   // screen size and bins come from each tile's camera
  memset(&fc, 0, sizeof(fc));
  const bool rop = blend_mode == GS_BLEND_FP16_ROP;
  int surf = 0;   // the SURF instantiation: 2 if some image is a layer of a layered array, else 1 if some is a 2-D array
  for (uint32_t i = 0; i < cams.count; ++i)
    if (!cams.cam[i].rt) surf = std::max(surf, cams.cam[i].surf.layer < 0 ? 1 : 2);
#define GS_RASTER_CAMS(ROP, FMT, SURF)                                                                                          \
  do {                                                                                                                         \
    if (objs.extras)                                                                                                           \
      chain_launch(k_raster<ROP, FMT, false, true, SURF, true>, tiles, 256, 0, s, fc, whole, nullptr, ranges, bs.tile_vals,        \
          bs.tile_order, bs.tile_cost, 1u, nullptr, 0u, Surface{}, 0u, 0u, nullptr, nullptr, SceneDepth{}, objs, cams, depth_surfs);  \
    else                                                                                                                       \
      chain_launch(k_raster<ROP, FMT, false, false, SURF, true>, tiles, 256, 0, s, fc, whole, nullptr, ranges, bs.tile_vals,       \
          bs.tile_order, bs.tile_cost, 1u, nullptr, 0u, Surface{}, 0u, 0u, nullptr, nullptr, nullptr, objs, cams,                 \
          NoRasterObjects{});                                                                                                  \
  } while (0)
#define GS_RASTER_CAMS_TARGET(ROP, FMT)                                                                                         \
  do {                                                                                                                         \
    if (surf == 2) GS_RASTER_CAMS(ROP, FMT, 2); else if (surf) GS_RASTER_CAMS(ROP, FMT, 1); else GS_RASTER_CAMS(ROP, FMT, 0);   \
  } while (0)
  if (rt_format == GS_PIX_RGBA16F) {
    if (rop) GS_RASTER_CAMS_TARGET(true, GS_PIX_RGBA16F); else GS_RASTER_CAMS_TARGET(false, GS_PIX_RGBA16F);
  } else {
    if (rop) GS_RASTER_CAMS_TARGET(true, GS_PIX_RGBA32F); else GS_RASTER_CAMS_TARGET(false, GS_PIX_RGBA32F);
  }
#undef GS_RASTER_CAMS_TARGET
#undef GS_RASTER_CAMS
}

uint32_t partition_own_bin_rows(const GsRenderOptions &opt, uint32_t binsY) { return make_partition(opt).own_rows_below(binsY); }
uint32_t partition_own_tile_rows(const GsRenderOptions &opt, uint32_t binsY) { return make_partition(opt).own_tile_rows(binsY); }

// ---- 2b. multi-GPU epilogue: gathered band-packed targets -> one image ---------------------------
__global__ void __launch_bounds__(256) k_unshuffle(const uint8_t *__restrict__ gathered, Partition part, uint32_t rows_pp, uint32_t px_bytes,
                                                   uint8_t *__restrict__ out, uint32_t pitch, uint32_t W, uint32_t H) {
  const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= W || y >= H) return;
  const uint32_t ty = y / kBin;
  Partition owner = part;
  owner.index = part.count > 1 ? (ty / part.band) % part.count : 0;
  const uint32_t k = owner.own_rows_below(ty);
  const uint8_t *src = gathered + ((size_t)owner.index * rows_pp + (size_t)k * kBin + (y - ty * kBin)) * W * px_bytes;
  if (px_bytes == 8) reinterpret_cast<uint2 *>(out + (size_t)y * pitch)[x] = reinterpret_cast<const uint2 *>(src)[x];
  else reinterpret_cast<uint4 *>(out + (size_t)y * pitch)[x] = reinterpret_cast<const uint4 *>(src)[x];
}

void launch_unshuffle(const void *gathered, uint32_t parts, uint32_t band, uint32_t rows_pp, uint32_t fmt, void *out, uint32_t pitch,
                      uint32_t W, uint32_t H, cudaStream_t s) {
  Partition p{};
  p.count = parts; p.index = 0; p.band = band ? band : 1;
  dim3 grid((W + 31) / 32, (H + 7) / 8);
  k_unshuffle<<<grid, 256, 0, s>>>(reinterpret_cast<const uint8_t *>(gathered), p, rows_pp, fmt == GS_PIX_RGBA16F ? 8u : 16u,
                                   reinterpret_cast<uint8_t *>(out), pitch, W, H);
}

// ---- 3. composite (S/GaussianComposite.shader:35-39, Blend SrcAlpha OneMinusSrcAlpha :11) ------
// The camera target is RGBA16F, RGBA32F, B10G11R11_UFLOAT or R8G8B8A8_SRGB; the render target is never one of the last two.
__device__ __forceinline__ float gamma_to_linear(float x) {  // UnityCG.cginc GammaToLinearSpace (not vendored)
  return x * fmaf(x, fmaf(x, 0.305306011f, 0.682171111f), 0.012522878f);
}

// one pixel of an RGBA16F / RGBA32F image: linear memory at (base, pitch), or, when base is null, a CUDA array behind `surf`
__device__ __forceinline__ float4 load_px(const uint8_t *base, uint32_t pitch, const Surface &surf, uint32_t fmt, uint32_t x, uint32_t y) {
  if (fmt == GS_PIX_RGBA16F) {
    uint2 v;
    if (base) v = reinterpret_cast<const uint2 *>(base + (size_t)y * pitch)[x];
    else surf_load<true>(&v, surf, x * 8u, y);
    return make_float4(f16lo(v.x), f16hi(v.x), f16lo(v.y), f16hi(v.y));
  }
  float4 c;
  if (base) c = reinterpret_cast<const float4 *>(base + (size_t)y * pitch)[x];
  else surf_load<true>(&c, surf, x * 16u, y);
  return c;
}

// TGT_FMT: the camera target's pixel format, a template parameter so that the RGBA16F and RGBA32F instantiations carry no code
// of the packed and sRGB ones (a uniform run-time branch cost the RGBA16F composite 3 % at 1920 x 1080 on an H100).
template <uint32_t TGT_FMT>
__global__ void __launch_bounds__(256) k_composite(const uint8_t *__restrict__ rt, uint32_t rt_pitch, Surface rt_surf,
                                                   uint32_t rt_fmt, uint8_t *__restrict__ tgt, uint32_t tgt_pitch,
                                                   Surface tgt_surf, uint32_t W, uint32_t H) {
  const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= W || y >= H) return;
  const float4 c = load_px(rt, rt_pitch, rt_surf, rt_fmt, x, y);
  if (!(c.w > 0.0f)) return;  // SrcAlpha == 0 leaves the target untouched
  float4 d = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  if constexpr (TGT_FMT == GS_PIX_B10G11R11_UFLOAT) {   // a camera target only: no alpha, one 32-bit texel
    uint32_t v;
    if (tgt) v = reinterpret_cast<const uint32_t *>(tgt + (size_t)y * tgt_pitch)[x];
    else surf_load<true>(&v, tgt_surf, x * 4u, y);
    unpack_b10g11r11(v, &d.x, &d.y, &d.z);
  } else if constexpr (TGT_FMT == GS_PIX_R8G8B8A8_SRGB) {   // a camera target only: four bytes, RGB sRGB-encoded
    uint32_t v;
    if (tgt) v = reinterpret_cast<const uint32_t *>(tgt + (size_t)y * tgt_pitch)[x];
    else surf_load<true>(&v, tgt_surf, x * 4u, y);
    unpack_srgb8(v, &d.x, &d.y, &d.z, &d.w);
  } else {
    d = load_px(tgt, tgt_pitch, tgt_surf, TGT_FMT, x, y);
  }
  const float a = c.w, om = 1.0f - a;
  float4 o;
  o.x = fmaf(gamma_to_linear(__fdiv_rn(c.x, a)), a, d.x * om);
  o.y = fmaf(gamma_to_linear(__fdiv_rn(c.y, a)), a, d.y * om);
  o.z = fmaf(gamma_to_linear(__fdiv_rn(c.z, a)), a, d.z * om);
  o.w = fmaf(a, a, d.w * om);
  if constexpr (TGT_FMT == GS_PIX_B10G11R11_UFLOAT) {
    const uint32_t v = pack_b10g11r11(o.x, o.y, o.z);
    if (tgt) reinterpret_cast<uint32_t *>(tgt + (size_t)y * tgt_pitch)[x] = v;
    else surf_store<true>(v, tgt_surf, x * 4u, y);
  } else if constexpr (TGT_FMT == GS_PIX_R8G8B8A8_SRGB) {
    const uint32_t v = pack_srgb8(o.x, o.y, o.z, o.w);
    if (tgt) reinterpret_cast<uint32_t *>(tgt + (size_t)y * tgt_pitch)[x] = v;
    else surf_store<true>(v, tgt_surf, x * 4u, y);
  } else if constexpr (TGT_FMT == GS_PIX_RGBA16F) {
    uint2 v;
    v.x = f32tof16(o.x) | (f32tof16(o.y) << 16);
    v.y = f32tof16(o.z) | (f32tof16(o.w) << 16);
    if (tgt) reinterpret_cast<uint2 *>(tgt + (size_t)y * tgt_pitch)[x] = v;
    else surf_store<true>(v, tgt_surf, x * 8u, y);
  } else {
    if (tgt) reinterpret_cast<float4 *>(tgt + (size_t)y * tgt_pitch)[x] = o;
    else surf_store<true>(o, tgt_surf, x * 16u, y);
  }
}

void launch_composite(const void *rt, uint32_t rt_pitch, Surface rt_surf, uint32_t rt_format, void *target, uint32_t tgt_pitch,
                      Surface tgt_surf, uint32_t tgt_format, uint32_t W, uint32_t H, cudaStream_t s) {
  if (!W || !H) return;
  dim3 grid((W + 31) / 32, (H + 7) / 8);
  const uint8_t *r = reinterpret_cast<const uint8_t *>(rt);
  uint8_t *t = reinterpret_cast<uint8_t *>(target);
  if (tgt_format == GS_PIX_B10G11R11_UFLOAT)
    k_composite<GS_PIX_B10G11R11_UFLOAT><<<grid, 256, 0, s>>>(r, rt_pitch, rt_surf, rt_format, t, tgt_pitch, tgt_surf, W, H);
  else if (tgt_format == GS_PIX_R8G8B8A8_SRGB)
    k_composite<GS_PIX_R8G8B8A8_SRGB><<<grid, 256, 0, s>>>(r, rt_pitch, rt_surf, rt_format, t, tgt_pitch, tgt_surf, W, H);
  else if (tgt_format == GS_PIX_RGBA16F)
    k_composite<GS_PIX_RGBA16F><<<grid, 256, 0, s>>>(r, rt_pitch, rt_surf, rt_format, t, tgt_pitch, tgt_surf, W, H);
  else
    k_composite<GS_PIX_RGBA32F><<<grid, 256, 0, s>>>(r, rt_pitch, rt_surf, rt_format, t, tgt_pitch, tgt_surf, W, H);
}

}  // namespace gs
