// gs_pack.cu -- the asset packer on the GPU: gs_pack_asset / gs_kmeans / gs_pack_sizes (include/gsplat_b200.h).
//
// Writes the same bytes as the host packer (csrc/asset_creator.cpp gsa_create_asset, csrc/asset_cluster_bc7.cpp gsa_kmeans)
// for finite input.  The format itself -- sizes, the chunk record, the pcg stream, the scalar encoders, one splat's records,
// the chunk header, the k-means squared distance, the BC7 block encoder -- is gs_asset_format.h, shared with the host
// packer.  What this file does its own way, and what keeps it equal to the host's sequential code:
//   * sequential math.min / math.max folds become (value, index) reductions where the earliest index wins among equal values
//     (so -0 vs +0 comes out as the fold leaves it) and NaN never wins;
//   * every float sum the host evaluates sequentially is evaluated sequentially here too (per-1024 k-means++ block sums, the
//     prefix over blocks, the in-block pick scan); the host sums that are cheap stay on the host (validation distance sum);
//   * the tiled nearest-mean kernel keeps distance_squared's grouping: pairs of squares, ((h0+h1)+h2)+h3 per 8 dimensions,
//     tail left to right;
//   * a chunk whose range is 0 / 0 normalises to x86's default NaN (host_div);
//   * scale^(1/8) is a double pow narrowed to float; CUDA's pow may differ from glibc's in the last double ulp, which changes
//     the float only next to a float rounding midpoint.  Such values are flagged and recomputed on the host with std::pow.
//   * every random draw of the k-means is independent of the data, so the host replays gsa_kmeans' pcg stream and uploads
//     the batch index lists; the device never runs a sequential RNG.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <new>
#include <utility>
#include <vector>

#include "gs_internal.cuh"

namespace gs {
namespace {

constexpr uint32_t kMaxKmeansDim = 128;
static_assert(sizeof(GsInputSplat) == kRecFloats * 4, "InputSplatData must be 248 bytes");

// ---- ordered reductions: the result of a sequential Unity.Mathematics math.min / math.max fold ------------------------
// `acc = math.min(acc, x)` keeps acc only when acc < x strictly (or x is NaN): of equal values (+0 / -0) the LATER one wins.
// So b replaces a when it is strictly smaller (larger), or equal and later.  NaN never enters a reduction (see take()).
template <bool MAX>
__device__ __forceinline__ bool fold_better(float bv, uint32_t bi, float av, uint32_t ai) {
  return (MAX ? (av < bv) : (bv < av)) || (bv == av && bi > ai);
}
// k-means' nearest mean: strictly smaller, or equal and earlier (the first of equal distances wins)
template <bool MAX>
__device__ __forceinline__ bool better(float bv, uint32_t bi, float av, uint32_t ai) {
  return (MAX ? (av < bv) : (bv < av)) || (bv == av && bi < ai);
}
template <bool MAX>
__device__ __forceinline__ void take(float &v, uint32_t &i, float x, uint32_t xi) {   // one step of the fold
  if (!isnan(x) && (MAX ? !(v > x) : !(v < x))) { v = x; i = xi; }
}
template <bool MAX>
__device__ __forceinline__ void warp_reduce(float &v, uint32_t &i) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const uint32_t oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (fold_better<MAX>(ov, oi, v, i)) { v = ov; i = oi; }
  }
}
// block of 256 threads; every thread gets the result.  `sv` / `si`: 8 entries of shared scratch
template <bool MAX>
__device__ void block_reduce(float &v, uint32_t &i, float *sv, uint32_t *si) {
  warp_reduce<MAX>(v, i);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) { sv[w] = v; si[w] = i; }
  __syncthreads();
  v = sv[0]; i = si[0];
  for (int k = 1; k < (int)(blockDim.x >> 5); ++k)
    if (fold_better<MAX>(sv[k], si[k], v, i)) { v = sv[k]; i = si[k]; }
}

// ---- 1. bounds (E/...:361-385) ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_bounds(const float *__restrict__ rec, uint32_t n, float *part_v, uint32_t *part_i) {
  __shared__ float sv[8];
  __shared__ uint32_t si[8];
  float mn[3], mx[3];
  uint32_t imn[3], imx[3];
  for (int k = 0; k < 3; ++k) { mn[k] = INFINITY; mx[k] = -INFINITY; imn[k] = imx[k] = 0xFFFFFFFFu; }
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    for (int k = 0; k < 3; ++k) {
      const float p = rec[(size_t)i * kRecFloats + k];
      take<false>(mn[k], imn[k], p, i);
      take<true>(mx[k], imx[k], p, i);
    }
  for (int k = 0; k < 3; ++k) {
    block_reduce<false>(mn[k], imn[k], sv, si);
    block_reduce<true>(mx[k], imx[k], sv, si);
    if (threadIdx.x == 0) {
      part_v[blockIdx.x * 6 + k] = mn[k]; part_i[blockIdx.x * 6 + k] = imn[k];
      part_v[blockIdx.x * 6 + 3 + k] = mx[k]; part_i[blockIdx.x * 6 + 3 + k] = imx[k];
    }
  }
}
__global__ void __launch_bounds__(256) k_bounds_final(const float *part_v, const uint32_t *part_i, uint32_t parts, float *bounds) {
  __shared__ float sv[8];
  __shared__ uint32_t si[8];
  for (int q = 0; q < 6; ++q) {
    float v = q < 3 ? INFINITY : -INFINITY;
    uint32_t i = 0xFFFFFFFFu;
    for (uint32_t p = threadIdx.x; p < parts; p += blockDim.x) {
      const float pv = part_v[p * 6 + q];
      const uint32_t pi = part_i[p * 6 + q];
      if (q < 3 ? fold_better<false>(pv, pi, v, i) : fold_better<true>(pv, pi, v, i)) { v = pv; i = pi; }
    }
    if (q < 3) block_reduce<false>(v, i, sv, si); else block_reduce<true>(v, i, sv, si);
    if (threadIdx.x == 0) bounds[q] = v;
  }
}

// ---- 2. Morton reorder (E/...:387-429) ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_morton(const float *__restrict__ rec, uint32_t n, const float *__restrict__ bounds,
                                                uint32_t *lo, uint32_t *hi, uint32_t *idx) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float kScaler = (float)((1 << 21) - 1);
  uint32_t ip[3];
  for (int k = 0; k < 3; ++k) {
    const float inv = 1.0f / (bounds[3 + k] - bounds[k]);
    const float p = (rec[(size_t)i * kRecFloats + k] - bounds[k]) * inv * kScaler;
    ip[k] = (p >= 0.0f && p < 4294967296.0f) ? (uint32_t)p : 0u;
  }
  const uint64_t code = morton_encode3(ip[0], ip[1], ip[2]);
  lo[i] = (uint32_t)code;
  hi[i] = (uint32_t)(code >> 32);
  idx[i] = i;
}
__global__ void k_gather_u32(const uint32_t *__restrict__ src, const uint32_t *__restrict__ idx, uint32_t n, uint32_t *dst) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}
// dst row r = src row idx[r] (row = `w` floats read at `src_stride`, written densely)
__global__ void k_gather_rows(const float *__restrict__ src, uint32_t src_stride, uint32_t w, const uint32_t *__restrict__ idx,
                              uint32_t rows, float *__restrict__ dst) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)rows * w) return;
  const uint32_t r = (uint32_t)(t / w), c = (uint32_t)(t % w);
  dst[t] = src[(size_t)(idx ? idx[r] : r) * src_stride + c];
}

// ---- 3. k-means (K:29-136 of the reference, gsa_kmeans) --------------------------------------------------------------------
// Nearest mean of every point (AssignClustersJob, K:423-441: strict <, the first of equal distances wins, start FLT_MAX / 0).
// A CTA takes 64 points (all their dimensions in shared memory) against 64-centre tiles; a thread owns 4 points x 4 centres.
// gridDim.y splits the centre tiles (tile t goes to split t % gridDim.y); each split writes its (best, index) per point and
// k_nearest_combine folds the splits with the same tie rule.
constexpr int kNP = 64, kNC = 64;
__global__ void __launch_bounds__(256) k_nearest(const float *__restrict__ data, uint32_t stride, uint32_t dim, uint32_t npts,
                                                 const float *__restrict__ means, uint32_t k, float *part_best, uint32_t *part_idx) {
  extern __shared__ float4 smem4[];
  float *sP = (float *)smem4;            // [dim][64]
  float *sC = sP + (size_t)dim * kNP;    // [8][64]
  const uint32_t p0 = blockIdx.x * kNP;
  for (uint32_t e = threadIdx.x; e < dim * kNP; e += blockDim.x) {
    const uint32_t p = e / dim, j = e % dim;
    sP[j * kNP + p] = (p0 + p < npts) ? data[(size_t)(p0 + p) * stride + j] : 0.0f;
  }
  const uint32_t tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float best[4];
  uint32_t bi[4];
  for (int r = 0; r < 4; ++r) { best[r] = FLT_MAX; bi[r] = 0; }
  const uint32_t tiles = (k + kNC - 1) / kNC, dim8 = dim & ~7u;
  for (uint32_t tile = blockIdx.y; tile < tiles; tile += gridDim.y) {
    const uint32_t c0 = tile * kNC;
    float d[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int l = 0; l < 4; ++l) d[r][l] = 0.0f;
    for (uint32_t j0 = 0; j0 < dim; j0 += 8) {
      const uint32_t w = j0 < dim8 ? 8u : dim - dim8;
      __syncthreads();
      for (uint32_t e = threadIdx.x; e < kNC * 8; e += blockDim.x) {
        const uint32_t c = e >> 3, jj = e & 7;
        sC[jj * kNC + c] = (c0 + c < k && jj < w) ? means[(size_t)(c0 + c) * dim + j0 + jj] : 0.0f;
      }
      __syncthreads();
      if (w == 8) {
        float4 a[8], m[8];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          a[jj] = *(const float4 *)&sP[(j0 + jj) * kNP + ty * 4];
          m[jj] = *(const float4 *)&sC[jj * kNC + tx * 4];
        }
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int l = 0; l < 4; ++l) {
            float h[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float av0 = ((const float *)&a[2 * q])[r], av1 = ((const float *)&a[2 * q + 1])[r];
              const float mv0 = ((const float *)&m[2 * q])[l], mv1 = ((const float *)&m[2 * q + 1])[l];
              const float t0 = av0 - mv0, t1 = av1 - mv1;
              h[q] = t0 * t0 + t1 * t1;
            }
            d[r][l] += ((h[0] + h[1]) + h[2]) + h[3];
          }
      } else {
        for (uint32_t jj = 0; jj < w; ++jj) {
          const float4 a = *(const float4 *)&sP[(j0 + jj) * kNP + ty * 4];
          const float4 m = *(const float4 *)&sC[jj * kNC + tx * 4];
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int l = 0; l < 4; ++l) {
              const float t = ((const float *)&a)[r] - ((const float *)&m)[l];
              d[r][l] += t * t;
            }
        }
      }
    }
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      const uint32_t c = c0 + tx * 4 + l;
      if (c < k)
#pragma unroll
        for (int r = 0; r < 4; ++r)
          if (d[r][l] < best[r]) { best[r] = d[r][l]; bi[r] = c; }
    }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
#pragma unroll
    for (int o = 8; o; o >>= 1) {   // the 16 threads of one point row are 16 consecutive lanes
      const float ov = __shfl_xor_sync(0xffffffffu, best[r], o);
      const uint32_t oi = __shfl_xor_sync(0xffffffffu, bi[r], o);
      if (better<false>(ov, oi, best[r], bi[r])) { best[r] = ov; bi[r] = oi; }
    }
    const uint32_t p = p0 + ty * 4 + r;
    if (tx == 0 && p < npts) { part_best[(size_t)blockIdx.y * npts + p] = best[r]; part_idx[(size_t)blockIdx.y * npts + p] = bi[r]; }
  }
}
__global__ void k_nearest_combine(const float *part_best, const uint32_t *part_idx, uint32_t npts, uint32_t splits, int32_t *labels,
                                  float *best_out) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npts) return;
  float b = part_best[p];
  uint32_t i = part_idx[p];
  for (uint32_t s = 1; s < splits; ++s) {
    const float ob = part_best[(size_t)s * npts + p];
    const uint32_t oi = part_idx[(size_t)s * npts + p];
    if (better<false>(ob, oi, b, i)) { b = ob; i = oi; }
  }
  if (labels) labels[p] = (int32_t)i;
  if (best_out) best_out[p] = b;
}

// One round of KMeansPlusPlus (K:325-411): distances to the newest centre (all of them for the first round), the
// per-1024-point sums in index order, then -- in the last CTA to finish -- the prefix over the sums, PickPointIndex
// (binary search + in-block scan, K:273-323) and the new centre.  One CTA per 1024 points.
constexpr uint32_t kSumBatch = 1024;
__global__ void __launch_bounds__(1024) k_kpp_round(const float *__restrict__ pts, uint32_t dim, uint32_t m, float *min_dist,
                                                    uint8_t *taken, float *means, uint32_t rc, int first, float *partial,
                                                    uint32_t *ticket, uint32_t rng) {
  __shared__ float sv[kSumBatch];
  __shared__ uint8_t st[kSumBatch];
  __shared__ bool last;
  __shared__ uint32_t s_lo, s_point;
  __shared__ float s_acc, s_rval;
  const uint32_t t = threadIdx.x, b = blockIdx.x, i = b * kSumBatch + t, nb = gridDim.x;
  const float *newest = means + (size_t)(rc - 1) * dim;
  float v = 0.0f;
  uint8_t tk = 1;
  if (i < m) {
    tk = taken[i];
    if (!tk) {
      const float d = distance_squared(pts + (size_t)i * dim, newest, dim);
      const float old = min_dist[i];
      v = first ? d : ((d < old) ? d : old);   // std::min(min_dist, d)
      min_dist[i] = v;
      __threadfence();
    }
  }
  sv[t] = v;
  st[t] = tk;
  __syncthreads();
  if (t == 0) {
    float sum = 0.0f;
    for (uint32_t j = 0; j < kSumBatch; ++j)
      if (!st[j]) sum += sv[j];
    partial[b] = sum;
    __threadfence();
    last = atomicAdd(ticket, 1u) == nb - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (t == 0) {
    float total = 0.0f;
    for (uint32_t bb = 0; bb < nb; ++bb) { total += __ldcg(&partial[bb]); partial[bb] = total; }
    const float rval = pcg_hash_float(rng + rc, total);
    uint32_t lo = 0, hi = nb;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) / 2;
      if (partial[mid] < rval) lo = mid + 1; else hi = mid;
    }
    s_lo = lo;
    s_acc = lo > 0 ? partial[lo - 1] : 0.0f;
    s_rval = rval;
  }
  __syncthreads();
  const uint32_t lo = s_lo;
  {
    const uint32_t j = lo * kSumBatch + t;
    const bool in = lo < nb && j < m;
    sv[t] = in ? __ldcg(&min_dist[j]) : 0.0f;
    st[t] = in ? __ldcg(&taken[j]) : (uint8_t)1;
  }
  __syncthreads();
  if (t == 0) {
    const float rval = s_rval;
    float acc = s_acc;
    int64_t point = -1;
    if (lo < nb)
      for (uint32_t j = 0; j < kSumBatch; ++j) {
        if (st[j]) continue;
        acc += sv[j];
        if (acc >= rval) { point = (int64_t)lo * kSumBatch + j; break; }
      }
    if (point < 0)
      for (uint64_t j = (uint64_t)(lo + 1) * kSumBatch; j < m; ++j) {
        if (__ldcg(&taken[j])) continue;
        acc += __ldcg(&min_dist[j]);
        if (acc >= rval) { point = (int64_t)j; break; }
      }
    if (point < 0)
      for (int64_t j = (int64_t)m - 1; j >= 0; --j)
        if (!__ldcg(&taken[j])) { point = j; break; }
    if (point < 0) point = 0;
    taken[point] = 1;
    s_point = (uint32_t)point;
    *ticket = 0;
  }
  __syncthreads();
  for (uint32_t c = t; c < dim; c += blockDim.x) means[(size_t)rc * dim + c] = pts[(size_t)s_point * dim + c];
}

// UpdateCentroidsJob (K:479-505): sequential over the batch, but only per centre.  The first batch point of each centre
// applies all of that centre's points in batch order, alpha = 1 / count.
__global__ void k_mb_update(const float *__restrict__ bp, const int32_t *__restrict__ lab, uint32_t bs, uint32_t dim, float *means,
                            float *counts) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= bs) return;
  const int32_t c = lab[i];
  for (uint32_t j = 0; j < i; ++j)
    if (lab[j] == c) return;
  float cnt = counts[c];
  float *mu = means + (size_t)c * dim;
  for (uint32_t j = i; j < bs; ++j) {
    if (lab[j] != c) continue;
    cnt += 1.0f;
    const float alpha = 1.0f / cnt;
    const float *p = bp + (size_t)j * dim;
    for (uint32_t q = 0; q < dim; ++q) mu[q] = mu[q] + alpha * (p[q] - mu[q]);
  }
  counts[c] = cnt;
}

// ---- 4. chunks (E/...:520-639) ------------------------------------------------------------------------------------------
// scale^(1/8) as (float)pow((double)s, 0.125).  A result within 2^-45 (relative) of a float rounding midpoint is listed for
// the host: CUDA's double pow is within 2 ulp, glibc's within 1, so elsewhere both round to the same float.
__global__ void k_pow_scales(float *rec, uint32_t n, uint32_t *fix_idx, float *fix_val, uint32_t *fix_count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int k = 0; k < 3; ++k) {
    float *sp = &rec[(size_t)i * kRecFloats + kOffScale + k];
    const float s = *sp;
    const double r = pow((double)s, (double)(1.0f / 8.0f));
    const float f = (float)r;
    if (isfinite(r) && f != 0.0f) {
      const double below = 0.5 * ((double)f + (double)nextafterf(f, -INFINITY));
      const double above = 0.5 * ((double)f + (double)nextafterf(f, INFINITY));
      const double tol = fabs(r) * 0x1p-45;
      if (fabs(r - below) <= tol || fabs(r - above) <= tol) {
        const uint32_t slot = atomicAdd(fix_count, 1u);
        fix_idx[slot] = i * 3u + (uint32_t)k;
        fix_val[slot] = s;
      }
    }
    *sp = f;
  }
}
__global__ void k_scatter_scales(float *rec, const uint32_t *idx, const float *val, uint32_t count) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < count) rec[(size_t)(idx[t] / 3u) * kRecFloats + kOffScale + idx[t] % 3u] = val[t];
}

// a / b as an x86 host computes it: a chunk whose range is 0 (|min| >= 256, where min + 1e-5 rounds back to min) divides
// 0 by 0, and the NaN that writes into Float32 / Float16 blobs is x86's default NaN 0xFFC00000, not the GPU's 0x7FFFFFFF
__device__ __forceinline__ float host_div(float a, float b) { const float q = a / b; return isnan(q) ? __uint_as_float(0xFFC00000u) : q; }

// One CTA per 256 splats: min/max of position, scale^(1/8), colour (dc0, square_centered01(opacity)) and the 15 SH
// coefficients per channel, ChunkInfo, then every value normalised to its chunk range.
__global__ void __launch_bounds__(256) k_chunks(float *rec, uint32_t n, Chunk *chunks) {
  __shared__ float sv[8];
  __shared__ uint32_t si[8];
  __shared__ float s_mn[13], s_mx[13];
  const uint32_t t = threadIdx.x, i = blockIdx.x * kChunkSize + t;
  const bool live = i < n;
  float *s = rec + (size_t)(live ? i : 0) * kRecFloats;
  if (live) s[kOffOpacity] = square_centered01(s[kOffOpacity]);
  __syncthreads();
  // q: 0..2 pos, 3..5 scale, 6..9 colour (dc0 rgb, opacity), 10..12 SH channel
  for (int q = 0; q < 13; ++q) {
    float mn = INFINITY, mx = -INFINITY;
    uint32_t imn = 0xFFFFFFFFu, imx = 0xFFFFFFFFu;
    if (live) {
      if (q < 10) {
        const float x = q < 3 ? s[q] : q < 6 ? s[kOffScale + q - 3] : q < 9 ? s[kOffDc0 + q - 6] : s[kOffOpacity];
        take<false>(mn, imn, x, t);
        take<true>(mx, imx, x, t);
      } else {
        for (uint32_t j = 0; j < 15; ++j) {
          const float x = s[kOffSh + j * 3 + (q - 10)];
          take<false>(mn, imn, x, t * 15 + j);
          take<true>(mx, imx, x, t * 15 + j);
        }
      }
    }
    block_reduce<false>(mn, imn, sv, si);
    block_reduce<true>(mx, imx, sv, si);
    if (t == 0) { s_mn[q] = mn; s_mx[q] = unity_max(mx, mn + 1.0e-5f); }
  }
  __syncthreads();
  if (t == 0) {   // stored through the 16-byte aligned device view: four 16-byte stores
    const ChunkInfo info = encode_chunk(s_mn, s_mx);
    Chunk c;
    memcpy(&c, &info, sizeof(c));
    chunks[blockIdx.x] = c;
  }
  if (!live) return;
  for (int k = 0; k < 3; ++k) {
    s[k] = host_div(s[k] - s_mn[k], s_mx[k] - s_mn[k]);
    s[kOffScale + k] = host_div(s[kOffScale + k] - s_mn[3 + k], s_mx[3 + k] - s_mn[3 + k]);
    s[kOffDc0 + k] = host_div(s[kOffDc0 + k] - s_mn[6 + k], s_mx[6 + k] - s_mn[6 + k]);
  }
  s[kOffOpacity] = host_div(s[kOffOpacity] - s_mn[9], s_mx[9] - s_mn[9]);
  for (int j = 0; j < 15; ++j)
    for (int k = 0; k < 3; ++k) s[kOffSh + j * 3 + k] = host_div(s[kOffSh + j * 3 + k] - s_mn[10 + k], s_mx[10 + k] - s_mn[10 + k]);
}

// ---- 5. emit (E/...:705-1066) ---------------------------------------------------------------------------------------------
struct EmitArgs {
  const float *rec;
  uint32_t n;
  EmitTarget to;           // image: BC7's float image, of float4 texels
  const int32_t *labels;   // clustered SH: palette index per splat
};
__global__ void __launch_bounds__(256) k_emit(EmitArgs a) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  emit_splat(a.to, i, a.rec + (size_t)i * kRecFloats, a.to.shf > 3 ? (uint32_t)a.labels[i] : 0u);
}
// ConvertSHClustersJob (E/...:443-468): 15 x half3 + one zero half3 per palette entry
__global__ void k_palette(const float *means, uint32_t k, uint8_t *sh) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= k * 45) return;
  put16(sh + (size_t)(t / 45) * 96 + (t % 45) * 2, unity_f32tof16(means[t]));
}

// ---- 6. BC7 mode 6: one thread per 4x4 block ----------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_bc7(const float4 *__restrict__ image, uint32_t bw, uint32_t nblocks, uint8_t *out) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblocks) return;
  const uint32_t bx = b % bw, by = b / bw;
  float rgba[64];
  for (int i = 0; i < 16; ++i) {
    const float4 p = image[(size_t)(by * 4 + i / 4) * kTexWidth + bx * 4 + i % 4];
    rgba[i * 4] = p.x; rgba[i * 4 + 1] = p.y; rgba[i * 4 + 2] = p.z; rgba[i * 4 + 3] = p.w;
  }
  const Bc7Block e = bc7_encode_block(rgba);
  uint64_t *o = (uint64_t *)(out + (size_t)b * 16);
  o[0] = e.lo;
  o[1] = e.hi;
}

// ---- host side ----------------------------------------------------------------------------------------------------------
#define PK_TRY(expr) GS_CUDA_TRY(ctx, expr)
#define PK_LAUNCHED() GS_CUDA_TRY(ctx, cudaGetLastError())

inline uint32_t blocks_for(uint64_t items, uint32_t per) { return (uint32_t)((items + per - 1) / per); }

// labels[p] (may be NULL) / best[p] (may be NULL) = nearest of the k means for each of the npts points
// scratch_v / scratch_i: the per-split partial results, grown to the largest call (final labelling)
int nearest(GsContext *ctx, const float *data, uint32_t stride, uint32_t dim, uint32_t npts, const float *means, uint32_t k,
            int32_t *labels, float *best, Buffer<float> &scratch_v, Buffer<uint32_t> &scratch_i) {
  const uint32_t ptiles = blocks_for(npts, kNP), ctiles = blocks_for(k, kNC);
  const uint32_t want = std::max(1u, (sm_count() * 4u) / std::max(1u, ptiles));
  const uint32_t splits = std::min(ctiles, std::min(want, 64u));
  const size_t need = (size_t)splits * npts;
  PK_TRY(scratch_v.reserve(need, {ctx->stream}));
  PK_TRY(scratch_i.reserve(need, {ctx->stream}));
  const size_t smem = ((size_t)dim * kNP + 8 * kNC) * sizeof(float);
  k_nearest<<<dim3(ptiles, splits), 256, smem, ctx->stream>>>(data, stride, dim, npts, means, k, scratch_v.get(), scratch_i.get());
  k_nearest_combine<<<blocks_for(npts, 256), 256, 0, ctx->stream>>>(scratch_v.get(), scratch_i.get(), npts, splits, labels, best);
  ctx->launches += 2;
  PK_LAUNCHED();
  return GS_OK;
}

// gsa_kmeans on the device.  data: n rows of `dim` floats at `stride`; d_means k x dim, d_labels n (device).
int kmeans_device(GsContext *ctx, const float *data, uint32_t stride, uint32_t dim, uint32_t n, uint32_t batch, float passes,
                  float *d_means, uint32_t k, int32_t *d_labels) {
  cudaStream_t st = ctx->stream;
  batch = std::min(n, batch);
  const uint32_t m = std::min(10u * k, n);   // initialize_centroids' batch
  // the host replays every random draw of gsa_kmeans
  uint32_t rng = 1;
  std::vector<uint8_t> picked(n, 0);
  std::vector<uint32_t> cb(m), vb(m);
  random_batch(n, rng, m, picked.data(), cb.data());
  random_batch(n, rng, m, picked.data(), vb.data());
  uint32_t point0[3], rng_at[3];
  for (int a = 0; a < 3; ++a) { point0[a] = pcg_random(rng) % m; rng_at[a] = rng; }
  uint32_t iters = 0;
  const float calc_limit = (float)n * passes;
  for (float done = 0.0f; done < calc_limit; done += (float)batch) ++iters;
  std::vector<uint32_t> mb((size_t)iters * batch);
  for (uint32_t it = 0; it < iters; ++it) random_batch(n, rng, batch, picked.data(), mb.data() + (size_t)it * batch);
  ctx->pack_stats[1] = iters;
  ctx->pack_stats[2] = 3ull * (k - 1);

  Buffer<uint32_t> d_idx, d_mb, ticket;
  Buffer<float> d_cb, d_vb, min_dist, partial, cur, best, counts, bpts, sv;
  Buffer<uint8_t> taken;
  Buffer<int32_t> blab;
  Buffer<uint32_t> si;
  const uint32_t nb = blocks_for(m, kSumBatch);
  PK_TRY(d_idx.reserve(m, {st}));
  PK_TRY(d_cb.reserve((size_t)m * dim, {st}));
  PK_TRY(d_vb.reserve((size_t)m * dim, {st}));
  PK_TRY(min_dist.reserve(m, {st}));
  PK_TRY(best.reserve(m, {st}));
  PK_TRY(taken.reserve(m, {st}));
  PK_TRY(partial.reserve(nb, {st}));
  PK_TRY(ticket.reserve(1, {st}));
  PK_TRY(cur.reserve((size_t)k * dim, {st}));
  PK_TRY(counts.reserve(k, {st}));
  PK_TRY(d_mb.reserve(std::max<size_t>(mb.size(), 1), {st}));
  PK_TRY(bpts.reserve((size_t)batch * dim, {st}));
  PK_TRY(blab.reserve(batch, {st}));
  PK_TRY(cudaMemcpyAsync(d_idx.get(), cb.data(), (size_t)m * 4, cudaMemcpyHostToDevice, st));
  k_gather_rows<<<blocks_for((uint64_t)m * dim, 256), 256, 0, st>>>(data, stride, dim, d_idx.get(), m, d_cb.get());
  PK_TRY(cudaStreamSynchronize(st));   // d_idx is reused for the validation batch
  PK_TRY(cudaMemcpyAsync(d_idx.get(), vb.data(), (size_t)m * 4, cudaMemcpyHostToDevice, st));
  k_gather_rows<<<blocks_for((uint64_t)m * dim, 256), 256, 0, st>>>(data, stride, dim, d_idx.get(), m, d_vb.get());
  PK_TRY(cudaMemsetAsync(ticket.get(), 0, 4, st));
  PK_TRY(cudaMemsetAsync(d_means, 0, (size_t)k * dim * 4, st));
  PK_LAUNCHED();

  // InitializeCentroids (K:507-569): three k-means++ attempts on the centroid batch, the one with the smallest validation
  // distance sum wins (sum on the host, sequential like gsa_kmeans)
  std::vector<float> hbest(m);
  float min_dist_sum = FLT_MAX;
  for (int a = 0; a < 3; ++a) {
    PK_TRY(cudaMemsetAsync(taken.get(), 0, m, st));
    PK_TRY(cudaMemsetAsync(taken.get() + point0[a], 1, 1, st));
    PK_TRY(cudaMemcpyAsync(cur.get(), d_cb.get() + (size_t)point0[a] * dim, (size_t)dim * 4, cudaMemcpyDeviceToDevice, st));
    for (uint32_t rc = 1; rc < k; ++rc)
      k_kpp_round<<<nb, kSumBatch, 0, st>>>(d_cb.get(), dim, m, min_dist.get(), taken.get(), cur.get(), rc, rc == 1, partial.get(), ticket.get(),
                                            rng_at[a]);
    ctx->launches += k - 1;
    PK_LAUNCHED();
    int rc = nearest(ctx, d_vb.get(), dim, dim, m, cur.get(), k, nullptr, best.get(), sv, si);
    if (rc) return rc;
    PK_TRY(cudaMemcpyAsync(hbest.data(), best.get(), (size_t)m * 4, cudaMemcpyDeviceToHost, st));
    PK_TRY(cudaStreamSynchronize(st));
    float dist_sum = 0.0f;
    for (uint32_t i = 0; i < m; ++i) dist_sum += hbest[i];
    if (dist_sum < min_dist_sum) {
      min_dist_sum = dist_sum;
      PK_TRY(cudaMemcpyAsync(d_means, cur.get(), (size_t)k * dim * 4, cudaMemcpyDeviceToDevice, st));
    }
  }
  // mini-batch passes (K:29-136)
  PK_TRY(cudaMemsetAsync(counts.get(), 0, (size_t)k * 4, st));
  if (iters) PK_TRY(cudaMemcpyAsync(d_mb.get(), mb.data(), mb.size() * 4, cudaMemcpyHostToDevice, st));
  for (uint32_t it = 0; it < iters; ++it) {
    k_gather_rows<<<blocks_for((uint64_t)batch * dim, 256), 256, 0, st>>>(data, stride, dim, d_mb.get() + (size_t)it * batch, batch, bpts.get());
    int rc = nearest(ctx, bpts.get(), dim, dim, batch, d_means, k, blab.get(), nullptr, sv, si);
    if (rc) return rc;
    k_mb_update<<<blocks_for(batch, 128), 128, 0, st>>>(bpts.get(), blab.get(), batch, dim, d_means, counts.get());
    ctx->launches += 2;
  }
  PK_LAUNCHED();
  // final labelling of every point
  int rc = nearest(ctx, data, stride, dim, n, d_means, k, d_labels, nullptr, sv, si);
  if (rc) return rc;
  PK_TRY(cudaStreamSynchronize(st));   // the host vectors above are freed on return
  return GS_OK;
}

}  // namespace
}  // namespace gs

using namespace gs;

extern "C" {

int gs_pack_sizes(uint32_t n, uint32_t pf, uint32_t sf, uint32_t cf, uint32_t shf, GsPackSizes *out) {
  if (!out) return fail(nullptr, GS_ERR_INVALID_ARGUMENT, "out is null");
  if (!calc_sizes(n, pf, sf, cf, shf, out))
    return fail(nullptr, GS_ERR_UNSUPPORTED_FORMAT, "unknown format, or clustered SH with no more splats than palette entries");
  return GS_OK;
}

int gs_debug_pack_stats(GsContext *ctx, uint64_t out[4]) {
  if (!ctx || !out) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null argument");
  memcpy(out, ctx->pack_stats, sizeof(ctx->pack_stats));
  return GS_OK;
}

int gs_kmeans(GsContext *ctx, uint32_t dim, const float *data, uint32_t n, uint32_t batch, float passes, float *means_out, uint32_t k,
              int32_t *labels_out) {
  if (!ctx || !data || !means_out || !labels_out) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null argument");
  // gsa_kmeans' argument rules, plus the dimension bound of the device kernels
  if (dim < 1 || dim > kMaxKmeansDim || batch < 1 || !(passes >= 0.0001f) || k < 1 || n < k)
    return fail(ctx, GS_ERR_INVALID_ARGUMENT, "gs_kmeans needs 1 <= dim <= 128, batch >= 1, passes >= 0.0001 and 1 <= k <= n");
  GS_CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  Buffer<float> d_data, d_means;
  Buffer<int32_t> d_labels;
  GS_CUDA_TRY(ctx, d_data.reserve((size_t)n * dim, {ctx->stream}));
  GS_CUDA_TRY(ctx, d_means.reserve((size_t)k * dim, {ctx->stream}));
  GS_CUDA_TRY(ctx, d_labels.reserve(n, {ctx->stream}));
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(d_data.get(), data, (size_t)n * dim * 4, cudaMemcpyHostToDevice, ctx->stream));
  int rc = kmeans_device(ctx, d_data.get(), dim, dim, n, batch, passes, d_means.get(), k, d_labels.get());
  if (rc) return rc;
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(means_out, d_means.get(), (size_t)k * dim * 4, cudaMemcpyDeviceToHost, ctx->stream));
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(labels_out, d_labels.get(), (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  GS_CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return GS_OK;
}

int gs_pack_asset(GsContext *ctx, const GsPackDesc *desc, GsPackedAsset *blobs_out, GsAsset **asset_out) {
  if (asset_out) *asset_out = nullptr;
  if (!ctx || !desc) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "null context or descriptor");
  if (!blobs_out && !asset_out) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "gs_pack_asset needs blobs_out and/or asset_out");
  if (!desc->splats || desc->splat_count == 0) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "no splats");
  if (desc->memory > GS_MEM_DEVICE) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "bad input memory kind");
  if (desc->splat_count >= (1u << 30)) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "splat_count must be < 2^30");
  const uint32_t n = desc->splat_count, pf = desc->pos_format, sf = desc->scale_format, cf = desc->color_format, shf = desc->sh_format;
  GsPackSizes sz;
  if (!calc_sizes(n, pf, sf, cf, shf, &sz))
    return fail(ctx, GS_ERR_UNSUPPORTED_FORMAT, "unknown format, or clustered SH with no more splats than palette entries");
  if (blobs_out) {
    if (blobs_out->memory > GS_MEM_DEVICE) return fail(ctx, GS_ERR_INVALID_ARGUMENT, "bad output memory kind");
    if (!blobs_out->pos || !blobs_out->other || !blobs_out->color || !blobs_out->sh || (sz.chunk_bytes && !blobs_out->chunks))
      return fail(ctx, GS_ERR_INVALID_ARGUMENT, "a blob buffer of blobs_out is null");
  }
  GS_CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  ctx->pack_stats[0] = ctx->pack_stats[1] = ctx->pack_stats[2] = 0;
  cudaStream_t st = ctx->stream;
  const bool chunked = sz.chunk_bytes != 0, clustered = shf > 3;

  // input
  const float *in = (const float *)desc->splats;
  Buffer<float> d_in;
  if (desc->memory == GS_MEM_HOST) {
    GS_CUDA_TRY(ctx, d_in.reserve((size_t)n * kRecFloats, {st}));
    GS_CUDA_TRY(ctx, cudaMemcpyAsync(d_in.get(), desc->splats, (size_t)n * sizeof(GsInputSplat), cudaMemcpyHostToDevice, st));
    in = d_in.get();
  }
  // 1. bounds
  const uint32_t bgrid = std::min(blocks_for(n, 256), sm_count() * 4u);
  Buffer<float> part_v, d_bounds;
  Buffer<uint32_t> part_i;
  GS_CUDA_TRY(ctx, part_v.reserve((size_t)bgrid * 6, {st}));
  GS_CUDA_TRY(ctx, part_i.reserve((size_t)bgrid * 6, {st}));
  GS_CUDA_TRY(ctx, d_bounds.reserve(6, {st}));
  k_bounds<<<bgrid, 256, 0, st>>>(in, n, part_v.get(), part_i.get());
  k_bounds_final<<<1, 256, 0, st>>>(part_v.get(), part_i.get(), bgrid, d_bounds.get());
  // 2. Morton order: (code, index) by two stable LSD sorts -- low word with the identity as payload, then the high word
  Buffer<uint32_t> lo, hi, idx;
  GS_CUDA_TRY(ctx, lo.reserve(n, {st}));
  GS_CUDA_TRY(ctx, hi.reserve(n, {st}));
  GS_CUDA_TRY(ctx, idx.reserve(n, {st}));
  k_morton<<<blocks_for(n, 256), 256, 0, st>>>(in, n, d_bounds.get(), lo.get(), hi.get(), idx.get());
  int rc = ensure_sort_scratch(ctx, n);
  if (rc) return rc;
  GS_CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_scalar.get(), &n, 4, cudaMemcpyHostToDevice, st));
  GS_CUDA_TRY(ctx, launch_sort_pairs(lo.get(), idx.get(), ctx->d_scalar.get(), n, 4, 8, false, sort_scratch(ctx), st));
  k_gather_u32<<<blocks_for(n, 256), 256, 0, st>>>(hi.get(), idx.get(), n, lo.get());
  GS_CUDA_TRY(ctx, launch_sort_pairs(lo.get(), idx.get(), ctx->d_scalar.get(), n, 4, 8, false, sort_scratch(ctx), st));
  ctx->launches += 5 + 2 * 5;
  GS_CUDA_TRY(ctx, cudaGetLastError());
  Buffer<float> recs;
  GS_CUDA_TRY(ctx, recs.reserve((size_t)n * kRecFloats, {st}));
  k_gather_rows<<<blocks_for((uint64_t)n * kRecFloats, 256), 256, 0, st>>>(in, kRecFloats, kRecFloats, idx.get(), n, recs.get());
  GS_CUDA_TRY(ctx, cudaGetLastError());

  // the blobs, in HBM; allocated like gs_asset_upload's (16 bytes of slack; a clustered palette backs all 65536 entries)
  Buffer<uint8_t> b_pos, b_other, b_color, b_sh, b_chunks;
  const uint64_t sh_alloc = std::max<uint64_t>(sz.sh_bytes, clustered ? 65536ull * 96ull : 0ull) + 16;
  GS_CUDA_TRY(ctx, b_pos.reserve(sz.pos_bytes + 16, {st}));
  GS_CUDA_TRY(ctx, b_other.reserve(sz.other_bytes + 16, {st}));
  GS_CUDA_TRY(ctx, b_color.reserve(sz.color_bytes + 16, {st}));
  GS_CUDA_TRY(ctx, b_sh.reserve(sh_alloc, {st}));
  if (chunked) GS_CUDA_TRY(ctx, b_chunks.reserve(sz.chunk_bytes + 16, {st}));
  GS_CUDA_TRY(ctx, cudaMemsetAsync(b_pos.get(), 0, sz.pos_bytes + 16, st));
  GS_CUDA_TRY(ctx, cudaMemsetAsync(b_other.get(), 0, sz.other_bytes + 16, st));
  GS_CUDA_TRY(ctx, cudaMemsetAsync(b_color.get(), 0, sz.color_bytes + 16, st));
  GS_CUDA_TRY(ctx, cudaMemsetAsync(b_sh.get(), 0, sh_alloc, st));
  if (chunked) GS_CUDA_TRY(ctx, cudaMemsetAsync(b_chunks.get(), 0, sz.chunk_bytes + 16, st));

  // 3. SH palette: k-means over the reordered, not yet normalised SH
  Buffer<float> means;
  Buffer<int32_t> labels;
  if (clustered) {
    static const float kPasses[5] = {0.3f, 0.4f, 0.5f, 0.8f, 1.2f};   // Cluster64k..4k, as gsa_create_asset
    const uint32_t k = sh_count(shf, n);
    GS_CUDA_TRY(ctx, means.reserve((size_t)k * 45, {st}));
    GS_CUDA_TRY(ctx, labels.reserve(n, {st}));
    if ((rc = kmeans_device(ctx, recs.get() + kOffSh, kRecFloats, 45, n, 2048, kPasses[shf - 4], means.get(), k, labels.get()))) return rc;
    k_palette<<<blocks_for((uint64_t)k * 45, 256), 256, 0, st>>>(means.get(), k, b_sh.get());
    GS_CUDA_TRY(ctx, cudaGetLastError());
  }
  // 4. chunks
  Buffer<uint32_t> fix_idx, fix_count;
  Buffer<float> fix_val;
  if (chunked) {
    GS_CUDA_TRY(ctx, fix_idx.reserve((size_t)n * 3, {st}));
    GS_CUDA_TRY(ctx, fix_val.reserve((size_t)n * 3, {st}));
    GS_CUDA_TRY(ctx, fix_count.reserve(1, {st}));
    GS_CUDA_TRY(ctx, cudaMemsetAsync(fix_count.get(), 0, 4, st));
    k_pow_scales<<<blocks_for(n, 256), 256, 0, st>>>(recs.get(), n, fix_idx.get(), fix_val.get(), fix_count.get());
    uint32_t count = 0;
    GS_CUDA_TRY(ctx, cudaMemcpyAsync(&count, fix_count.get(), 4, cudaMemcpyDeviceToHost, st));
    GS_CUDA_TRY(ctx, cudaStreamSynchronize(st));
    ctx->pack_stats[0] = count;
    if (count) {   // the host's own pow for the values next to a rounding midpoint
      std::vector<float> v(count);
      GS_CUDA_TRY(ctx, cudaMemcpyAsync(v.data(), fix_val.get(), (size_t)count * 4, cudaMemcpyDeviceToHost, st));
      GS_CUDA_TRY(ctx, cudaStreamSynchronize(st));
      for (float &x : v) x = (float)std::pow((double)x, (double)(1.0f / 8.0f));
      GS_CUDA_TRY(ctx, cudaMemcpyAsync(fix_val.get(), v.data(), (size_t)count * 4, cudaMemcpyHostToDevice, st));
      k_scatter_scales<<<blocks_for(count, 256), 256, 0, st>>>(recs.get(), fix_idx.get(), fix_val.get(), count);
      GS_CUDA_TRY(ctx, cudaStreamSynchronize(st));   // `v` is freed at the end of this scope
    }
    k_chunks<<<blocks_for(n, kChunkSize), kChunkSize, 0, st>>>(recs.get(), n, (Chunk *)b_chunks.get());
    GS_CUDA_TRY(ctx, cudaGetLastError());
  }
  // 5. emit, 6. BC7
  Buffer<float4> image;
  if (cf == GS_COL_BC7) {
    const size_t texels = (size_t)sz.tex_width * sz.tex_height;
    GS_CUDA_TRY(ctx, image.reserve(texels, {st}));
    GS_CUDA_TRY(ctx, cudaMemsetAsync(image.get(), 0, texels * 16, st));
  }
  EmitArgs ea{recs.get(), n, {b_pos.get(), b_other.get(), b_color.get(), b_sh.get(), (float *)image.get(), pf, sf, cf, shf}, labels.get()};
  k_emit<<<blocks_for(n, 256), 256, 0, st>>>(ea);
  if (cf == GS_COL_BC7) {
    const uint32_t bw = sz.tex_width / 4, nblocks = bw * (sz.tex_height / 4);
    k_bc7<<<blocks_for(nblocks, 128), 128, 0, st>>>(image.get(), bw, nblocks, b_color.get());
  }
  GS_CUDA_TRY(ctx, cudaGetLastError());

  if (blobs_out) {
    const cudaMemcpyKind kind = blobs_out->memory == GS_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    GS_CUDA_TRY(ctx, cudaMemcpyAsync(blobs_out->pos, b_pos.get(), sz.pos_bytes, kind, st));
    GS_CUDA_TRY(ctx, cudaMemcpyAsync(blobs_out->other, b_other.get(), sz.other_bytes, kind, st));
    GS_CUDA_TRY(ctx, cudaMemcpyAsync(blobs_out->color, b_color.get(), sz.color_bytes, kind, st));
    GS_CUDA_TRY(ctx, cudaMemcpyAsync(blobs_out->sh, b_sh.get(), sz.sh_bytes, kind, st));
    if (chunked) GS_CUDA_TRY(ctx, cudaMemcpyAsync(blobs_out->chunks, b_chunks.get(), sz.chunk_bytes, kind, st));
    float hb[6];
    GS_CUDA_TRY(ctx, cudaMemcpyAsync(hb, d_bounds.get(), sizeof(hb), cudaMemcpyDeviceToHost, st));
    GS_CUDA_TRY(ctx, cudaStreamSynchronize(st));
    memcpy(blobs_out->bounds_min, hb, 12);
    memcpy(blobs_out->bounds_max, hb + 3, 12);
  }
  if (asset_out) {
    GsAsset *as = new (std::nothrow) GsAsset();
    if (as) as->blobs = new (std::nothrow) GsBlobs();
    if (!as || !as->blobs) {
      delete as;
      return fail(ctx, GS_ERR_OUT_OF_MEMORY, "host allocation failed");
    }
    as->ctx = ctx;
    GsBlobs &b = *as->blobs;
    b.pos = std::move(b_pos); b.other = std::move(b_other); b.color = std::move(b_color); b.sh = std::move(b_sh);
    b.chunks = std::move(b_chunks);
    const cudaError_t e = asset_init_work(ctx, as, n, pf, sf, shf, cf, chunked ? (uint32_t)(sz.chunk_bytes / 64) : 0u);
    if (e != cudaSuccess) {
      gs_asset_destroy(as);
      return fail_cuda(ctx, e, "gs_pack_asset", __FILE__, __LINE__);
    }
    *asset_out = as;
  }
  GS_CUDA_TRY(ctx, cudaStreamSynchronize(st));   // the scratch buffers are freed on return
  return GS_OK;
}

}  // extern "C"
