// gs_view.cu -- CSSetIndices, CSCalcDistances, CSCalcViewData as sm_90a kernels.
//
// Reference behaviour: S/SplatUtilities.compute:59-82,107-252 and the decode library
// S/GaussianSplatting.hlsl:5-11,29-90,130-229,261-300,346-608.  Design (not a port):
//   * one CTA == one 256-splat chunk, so the 64-byte chunk header is fetched once per CTA
//     into shared memory and broadcast; every packed stream is read with the widest
//     aligned vector load its stride allows;
//   * the 40-byte SplatViewData records of a CTA are staged in shared memory and leave as
//     fully coalesced 16-byte stores (a 40-byte stride cannot be stored with float4);
//   * the same kernel emits the splat's screen-tile rectangle (4 bytes) for the binner,
//     so the raster stage never has to touch the 40-byte record to count tiles;
//   * CSCalcDistances writes the depth keys in natural order (coalesced) and accumulates the four
//     8-bit digit histograms on the way; the gather through last frame's order is folded into
//     pass 0 of the radix sort, so neither a histogram read nor a gathered key array exists.
#include "gs_kernels.cuh"
#include "gs_bc7.cuh"

namespace gs {

__global__ void __launch_bounds__(256) k_set_indices(uint32_t *__restrict__ order, uint32_t n) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) order[i] = i;
}

// ------------------------------------------------------------------------------------------
// CSCalcDistances (+ fused digit histograms for the sort)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float3 load_pos(const AssetView &a, uint32_t idx) {
  float3 p = load_vector(a.pos, (uint64_t)idx * vec_stride(a.posFmt), a.posFmt);
  uint32_t ci = idx >> 8;
  if (ci < a.chunkCount) {  // LoadSplatPos, S/GaussianSplatting.hlsl:409-421
    const float4 *c = reinterpret_cast<const float4 *>(a.chunks + ci);
    float4 px_py = __ldg(c + 1);  // posX.xy posY.xy
    float2 pz = __ldg(reinterpret_cast<const float2 *>(c + 2));
    p.x = lerpf(px_py.x, px_py.y, p.x);
    p.y = lerpf(px_py.z, px_py.w, p.y);
    p.z = lerpf(pz.x, pz.y, p.z);
  }
  return p;
}

constexpr int kDistItems = 4;  // keys per thread: 4 CONSECUTIVE splats, so Norm11 / Float32 positions come in as 16-byte vectors

// Per-splat depth keys in NATURAL order + the four digit histograms of the sort.  The reference's
// CSCalcDistances writes key(pos[order[i]]) (S/SplatUtilities.compute:76-81); the multiset of keys -- all the
// histograms need -- does not depend on the order, and the gather through `order` happens inside pass 0
// of the radix sort (gs_sort.cu, GATHER), so this kernel is fully coalesced and nothing is gathered twice.
//
// SLABS (the group path, SURVEY 8e.2): the sort is sharded by KEY RANGE.  The G-1 splitters are the current keys of the
// splats that stood at the quantile positions of last frame's order (replicated data, so every GPU derives the same
// values); splat i belongs to slab c = #{splitters <= key(i)}.  Besides the key table this kernel then writes a bit mask
// of the splats of THIS GPU's slab, restricts the digit histograms to them, and counts #{key >= splitter j} for every j,
// which gives every GPU the size and offset of every slab without any exchange.
template <int MAXT>   // 0: no slabs; else the largest splitter count compiled for
__global__ void __launch_bounds__(256) k_calc_distances(AssetView a, float4 row, uint32_t *__restrict__ key_table,
                                                        uint32_t *__restrict__ ghist, SlabArgs sl) {
  __shared__ uint32_t sh[4 * 256];
  __shared__ uint32_t s_thr[MAXT + 1];
  __shared__ uint32_t s_ge[MAXT + 1];
  for (int i = threadIdx.x; i < 1024; i += 256) sh[i] = 0;
  // Without slabs, everything but the flush into ghist runs before the wait: its predecessor is the k_clear that starts the
  // depth sort, which releases at once, so this kernel can run beside the end of the previous frame's raster.  Pre-wait
  // reads: the asset's position blobs and chunks, which no kernel writes.  Pre-wait writes: key_table, which only pass 0 of
  // this asset's depth sort reads; the kernels still running are at most that k_clear and the node before it, never a
  // depth sort's pass 0 (a sort ends with its last pass).  ghist is cleared by the k_clear, so it is counted into after the
  // wait.  The slab variant (group path) reads last frame's order and writes the slab masks: it waits first.
  if (MAXT) {
    chain_wait();
    chain_release();
  }
  const uint32_t nthr = MAXT ? sl.count - 1 : 0;   // number of splitters
  if (MAXT) {
    if (threadIdx.x < nthr) {
      const uint32_t id = __ldg(sl.order_prev + sl.qpos[threadIdx.x]);
      const float3 p = load_pos(a, id);
      s_thr[threadIdx.x] = float_to_sortable_uint(fmaf(row.z, p.z, fmaf(row.y, p.y, fmaf(row.x, p.x, row.w))));
      s_ge[threadIdx.x] = 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {   // ascending splitters (camera motion can reorder last frame's quantile splats)
      for (uint32_t i = 1; i < nthr; ++i) {
        const uint32_t v = s_thr[i];
        uint32_t j = i;
        while (j > 0 && s_thr[j - 1] > v) { s_thr[j] = s_thr[j - 1]; --j; }
        s_thr[j] = v;
      }
      if (blockIdx.x == 0) for (uint32_t i = 0; i < nthr; ++i) sl.info[i] = s_thr[i];
    }
  }
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  uint32_t lo = 0, hi = 0;
  bool has_hi = false;
  if (MAXT) {
    if (sl.index > 0) lo = s_thr[sl.index - 1];
    if (sl.index < nthr) { hi = s_thr[sl.index]; has_hi = true; }
  }
  uint32_t ge[MAXT + 1];
#pragma unroll
  for (int j = 0; j < MAXT; ++j) ge[j] = 0;
  // persistent CTAs: the shared histograms are flushed to the 1024 global counters once per CTA, not once per
  // 1024 splats (6M same-address L2 atomics were the whole cost of this kernel)
  for (uint32_t tile = blockIdx.x; tile * (256u * kDistItems) < a.n; tile += gridDim.x) {
  const uint32_t first = (tile * 256 + threadIdx.x) * kDistItems;   // multiple of 4: the 4 splats share a chunk
  float3 p[kDistItems];
  const bool full = first + kDistItems <= a.n;
  if (full && a.posFmt == 2) {          // Norm11: 4 x 4 bytes
    const uint4 e = __ldg(reinterpret_cast<const uint4 *>(a.pos) + (first >> 2));
    p[0] = dec_11_10_11(e.x); p[1] = dec_11_10_11(e.y); p[2] = dec_11_10_11(e.z); p[3] = dec_11_10_11(e.w);
  } else if (full && a.posFmt == 0) {   // Float32: 4 x 12 bytes = 3 vectors
    const uint4 *q = reinterpret_cast<const uint4 *>(a.pos) + (size_t)(first >> 2) * 3;
    const uint4 e0 = __ldg(q), e1 = __ldg(q + 1), e2 = __ldg(q + 2);
    p[0] = make_float3(__uint_as_float(e0.x), __uint_as_float(e0.y), __uint_as_float(e0.z));
    p[1] = make_float3(__uint_as_float(e0.w), __uint_as_float(e1.x), __uint_as_float(e1.y));
    p[2] = make_float3(__uint_as_float(e1.z), __uint_as_float(e1.w), __uint_as_float(e2.x));
    p[3] = make_float3(__uint_as_float(e2.y), __uint_as_float(e2.z), __uint_as_float(e2.w));
  } else {
#pragma unroll
    for (int it = 0; it < kDistItems; ++it)
      p[it] = (first + it < a.n) ? load_vector(a.pos, (uint64_t)(first + it) * vec_stride(a.posFmt), a.posFmt) : make_float3(0.f, 0.f, 0.f);
  }
  const uint32_t ci = first >> 8;
  if (ci < a.chunkCount) {  // LoadSplatPos, S/GaussianSplatting.hlsl:409-421
    const float4 *c = reinterpret_cast<const float4 *>(a.chunks + ci);
    const float4 px_py = __ldg(c + 1);
    const float2 pz = __ldg(reinterpret_cast<const float2 *>(c + 2));
#pragma unroll
    for (int it = 0; it < kDistItems; ++it) {
      p[it].x = lerpf(px_py.x, px_py.y, p[it].x);
      p[it].y = lerpf(px_py.z, px_py.w, p[it].y);
      p[it].z = lerpf(pz.x, pz.y, p[it].z);
    }
  }
  uint32_t k[kDistItems];
#pragma unroll
  for (int it = 0; it < kDistItems; ++it) k[it] = float_to_sortable_uint(fmaf(row.z, p[it].z, fmaf(row.y, p[it].y, fmaf(row.x, p[it].x, row.w))));
  if (full) {
    reinterpret_cast<uint4 *>(key_table)[first >> 2] = make_uint4(k[0], k[1], k[2], k[3]);
  } else {
    for (int it = 0; it < kDistItems; ++it)
      if (first + it < a.n) key_table[first + it] = k[it];
  }
  uint32_t nib = 0;   // slab membership of this thread's 4 splats
#pragma unroll
  for (int it = 0; it < kDistItems; ++it) {
    const bool live = first + it < a.n;
    bool mine = live;
    if (MAXT) {
      mine = live && k[it] >= lo && (!has_hi || k[it] < hi);
      if (mine) nib |= 1u << it;
      if (live) {
#pragma unroll
        for (int j = 0; j < MAXT; ++j) if ((uint32_t)j < nthr) ge[j] += (k[it] >= s_thr[j]) ? 1u : 0u;
      }
    }
    if (mine) {
      atomicAdd(&sh[k[it] & 255u], 1u);
      atomicAdd(&sh[256 + ((k[it] >> 8) & 255u)], 1u);
    }
    // The two high digits are nearly constant inside a warp (Morton-ordered neighbours have similar depth);
    // plain atomics would serialise 32-way on one bank, so a uniform warp is counted with one add.
    const uint32_t hi16 = k[it] >> 16;
    const uint32_t hi0 = __shfl_sync(0xffffffffu, hi16, 0);
    const uint32_t minemask = __ballot_sync(0xffffffffu, mine);
    if (minemask == 0xffffffffu && __all_sync(0xffffffffu, hi16 == hi0)) {
      if (lane == 0) { atomicAdd(&sh[512 + (hi0 & 255u)], 32u); atomicAdd(&sh[768 + (hi0 >> 8)], 32u); }
    } else if (mine) {
      atomicAdd(&sh[512 + (hi16 & 255u)], 1u);
      atomicAdd(&sh[768 + (hi16 >> 8)], 1u);
    }
  }
  if (MAXT) {   // 8 lanes x 4 bits = one mask word (first is a multiple of 4, 8 consecutive threads cover 32 splats)
    uint32_t w = nib << ((lane & 7u) * 4u);
    w |= __shfl_xor_sync(0xffffffffu, w, 1);
    w |= __shfl_xor_sync(0xffffffffu, w, 2);
    w |= __shfl_xor_sync(0xffffffffu, w, 4);
    if ((lane & 7u) == 0 && first < a.n) sl.mask[first >> 5] = w;
    // one BIT per 128 consecutive splats (= this warp's share of the tile): "somebody here belongs to my slab" (zeroed before
    // the launch).  Morton-local splats lie in a narrow depth range, so most groups belong to one or two slabs; the
    // compaction keeps this bitmap in shared memory and touches a group's mask words only where the bit is set.
    const uint32_t anyw = __ballot_sync(0xffffffffu, nib != 0);
    if (lane == 0 && anyw && first < a.n) atomicOr(sl.group_bits + (first >> 12), 1u << ((first >> 7) & 31u));
  }
  }  // tile loop
  if (MAXT) {
#pragma unroll
    for (int j = 0; j < MAXT; ++j) {
      if ((uint32_t)j < nthr) {
        uint32_t v = ge[j];
#pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0 && v) atomicAdd(&s_ge[j], v);
      }
    }
  }
  __syncthreads();
  if (!MAXT) {
    chain_wait();
    chain_release();
  }
  for (int i = threadIdx.x; i < 1024; i += 256) {
    uint32_t c = sh[i];
    if (c) atomicAdd(&ghist[i], c);
  }
  if (MAXT && threadIdx.x < nthr) {
    const uint32_t c = s_ge[threadIdx.x];
    if (c) atomicAdd(&sl.info[kMaxSlabs + threadIdx.x], c);
  }
}

// ------------------------------------------------------------------------------------------
// CSCalcViewData
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ bool is_splat_cut(const FrameConsts &fc, const GsCutout *__restrict__ cut, float3 p) {
  // S/SplatUtilities.compute:164-187
  bool finalCut = false;
  for (uint32_t i = 0; i < fc.cutoutCount; ++i) {
    const GsCutout &c = cut[i];
    uint32_t type = c.type_and_flags & 0xFFu;
    if (type == 0xFFu) continue;
    bool invert = (c.type_and_flags & 0xFF00u) != 0;
    const float *m = c.mat;  // column-major
    float cx = fmaf(m[8], p.z, fmaf(m[4], p.y, fmaf(m[0], p.x, m[12])));
    float cy = fmaf(m[9], p.z, fmaf(m[5], p.y, fmaf(m[1], p.x, m[13])));
    float cz = fmaf(m[10], p.z, fmaf(m[6], p.y, fmaf(m[2], p.x, m[14])));
    if (type == 0) { if (cx * cx + cy * cy + cz * cz <= 1.0f) return invert; }
    if (type == 1) { if (fabsf(cx) <= 1.0f && fabsf(cy) <= 1.0f && fabsf(cz) <= 1.0f) return invert; }
    finalCut |= !invert;
  }
  return finalCut;
}

// Raw SH words of one splat, loaded with 16-byte vector loads (strides 32/60/96/192 keep
// at least 4-byte alignment; 60 is only 4-aligned so Norm11 uses word loads).
template <int FMT>
struct ShRaw;
template <>
struct ShRaw<3> {  // Norm6: 15 x u16 + pad = 32 B
  uint32_t w[8];
  __device__ __forceinline__ void load(const uint8_t *p) {
    uint4 a = __ldg(reinterpret_cast<const uint4 *>(p)), b = __ldg(reinterpret_cast<const uint4 *>(p + 16));
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
  }
  __device__ __forceinline__ float3 get(int j) const { return dec_5_6_5((w[j >> 1] >> ((j & 1) * 16)) & 0xffffu); }
};
template <>
struct ShRaw<2> {  // Norm11: 15 x u32 = 60 B
  uint32_t w[15];
  __device__ __forceinline__ void load(const uint8_t *p) {
#pragma unroll
    for (int j = 0; j < 15; ++j) w[j] = __ldg(reinterpret_cast<const uint32_t *>(p) + j);
  }
  __device__ __forceinline__ float3 get(int j) const { return dec_11_10_11(w[j]); }
};
template <>
struct ShRaw<1> {  // Float16: 45 halfs + pad = 96 B
  uint32_t w[24];
  __device__ __forceinline__ void load(const uint8_t *p) {
#pragma unroll
    for (int q = 0; q < 6; ++q) {
      uint4 a = __ldg(reinterpret_cast<const uint4 *>(p) + q);
      w[q * 4] = a.x; w[q * 4 + 1] = a.y; w[q * 4 + 2] = a.z; w[q * 4 + 3] = a.w;
    }
  }
  __device__ __forceinline__ float h(int k) const { return (k & 1) ? f16hi(w[k >> 1]) : f16lo(w[k >> 1]); }
  __device__ __forceinline__ float3 get(int j) const { return make_float3(h(j * 3), h(j * 3 + 1), h(j * 3 + 2)); }
};
template <>
struct ShRaw<4> : ShRaw<1> {};  // Cluster4k..64k: a Float16 palette entry (SHTableItemFloat16), picked by a per-splat u16 index
template <>
struct ShRaw<0> {  // Float32: 45 floats + pad = 192 B
  uint32_t w[48];
  __device__ __forceinline__ void load(const uint8_t *p) {
#pragma unroll
    for (int q = 0; q < 12; ++q) {
      uint4 a = __ldg(reinterpret_cast<const uint4 *>(p) + q);
      w[q * 4] = a.x; w[q * 4 + 1] = a.y; w[q * 4 + 2] = a.z; w[q * 4 + 3] = a.w;
    }
  }
  __device__ __forceinline__ float3 get(int j) const {
    return make_float3(__uint_as_float(w[j * 3]), __uint_as_float(w[j * 3 + 1]), __uint_as_float(w[j * 3 + 2]));
  }
};

__device__ __forceinline__ float3 operator*(float s, float3 v) { return make_float3(s * v.x, s * v.y, s * v.z); }
__device__ __forceinline__ float3 operator*(float3 v, float s) { return make_float3(v.x * s, v.y * s, v.z * s); }
__device__ __forceinline__ float3 operator+(float3 a, float3 b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 operator-(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float3 neg(float3 a) { return make_float3(-a.x, -a.y, -a.z); }

// CULL (used by the fused gs_frame): in the reference _SplatViewData only carries CSCalcViewData's results to the draw.
// The fused frame hands them over as 48-byte draw records instead, so (a) the 40-byte view record is a dead store and is
// not written at all (245 MB/frame at 6.1 M splats), and (b) for a splat that can never produce a fragment -- quad off
// screen, which a cheap extent bound often shows before any covariance maths, or opacity below the 1/255 discard -- the
// colour half (SH fetch + ShadeSH, 2/3 of the bytes, ~half of the arithmetic) is dead code too.  gs_calc_view (the
// stand-alone entry point) always runs the full kernel, so _SplatViewData parity is checked on that one.
__device__ __forceinline__ void prefetch_l1(const void *p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
// where texel `ti` of the 2048-wide colour image lives (BC7: its 16-byte 4x4 block, blocks row-major)
template <bool BC7>
__device__ __forceinline__ const uint8_t *color_texel_ptr(const AssetView &a, uint32_t ti) {
  if (BC7) return a.color + ((uint64_t)((ti / kTexWidth) >> 2) * (kTexWidth / 4) + ((ti & (kTexWidth - 1)) >> 2)) * 16u;
  return a.color + (uint64_t)ti * (a.colFmt == 0 ? 16u : a.colFmt == 1 ? 8u : 4u);
}

// The fused Norm6 kernel (the Medium preset's frame) sits at a register-allocation cliff: left alone ptxas picks 60 registers
// (4 CTAs/SM); asked for 5 CTAs/SM it fits 48 without a spill, which was measured faster.
template <int SHFMT, bool CULL, bool BC7>
__global__ void __launch_bounds__(256, (CULL && SHFMT == 3 && !BC7) ? 5 : 1)
k_calc_view(AssetView a, FrameConsts fc, const GsCutout *__restrict__ cutouts, const uint32_t *__restrict__ deleted,
            const uint32_t *__restrict__ selected, uint32_t *__restrict__ view_out, uint32_t *__restrict__ rect_out, float4 *__restrict__ draw_out,
            uint32_t *__restrict__ block_bits, float *__restrict__ zndc, Partition part, uint32_t early) {
  __shared__ __align__(16) uint32_t s_view[256 * 10];
  __shared__ __align__(16) Chunk s_chunk;
  const uint32_t idx = blockIdx.x * 256 + threadIdx.x;
  const bool chunked = blockIdx.x < a.chunkCount;
  // early != 0: the host knows the predecessor is the depth sort of this asset (which reads and writes keys, order and the
  // sort scratch only), so the whole body runs before the wait and overlaps the sort's last pass.  Pre-wait reads: the
  // asset's blobs, fc, cutouts / deleted / selected (their uploads are copies, which complete before it starts); pre-wait writes: view_out,
  // rect_out, draw_out, zndc and this CTA's bit of block_bits, which only the previous frame's binner and raster read, and
  // those completed before the sort began.  Otherwise the kernel waits first: in a run, a view-calc may follow an emit that
  // reads this asset's rect / block_bits.  The early kernel releases nothing itself (its successor is placed as it exits).
  if (!early) {
    chain_wait();
    chain_release();
  }
  if (chunked && threadIdx.x < 4)
    reinterpret_cast<uint4 *>(&s_chunk)[threadIdx.x] = __ldg(reinterpret_cast<const uint4 *>(a.chunks + blockIdx.x) + threadIdx.x);
  // the per-splat streams do not depend on the chunk header: start them before the barrier so the CTA pays one
  // memory latency, not two (a CTA with nothing to draw was 2 dependent round trips long)
  if (idx < a.n) {
    prefetch_l1(a.pos + (uint64_t)idx * vec_stride(a.posFmt));
    prefetch_l1(a.other + (uint64_t)idx * (4 + vec_stride(a.scaleFmt) + (SHFMT == 4 ? 2u : 0u)));
    if (!CULL) {
      prefetch_l1(color_texel_ptr<BC7>(a, splat_index_to_texel(idx)));
      if (fc.shOrder >= 1 && SHFMT != 4) prefetch_l1(a.sh + (uint64_t)idx * (SHFMT == 0 ? 192u : SHFMT == 1 ? 96u : SHFMT == 2 ? 60u : 32u));
    }
  }
  __syncthreads();

  if (CULL && chunked) {
    // Hierarchical cull on the asset's own chunk bounds (free metadata: SplatChunkInfo pos min/max, scale max): if the
    // chunk's box, grown by the largest screen reach any of its 256 splats can have, misses the screen -- or lies entirely
    // behind the camera -- every splat of this CTA is undrawable and only its (empty) bin rect is written.
    __shared__ int s_cull;
    if (threadIdx.x < 32) {
      const uint32_t l = threadIdx.x & 7;
      const float bx = (l & 1) ? s_chunk.posX.y : s_chunk.posX.x, by = (l & 2) ? s_chunk.posY.y : s_chunk.posY.x,
                  bz = (l & 4) ? s_chunk.posZ.y : s_chunk.posZ.x;
      const float wx = fmaf(fc.o2w[2], bz, fmaf(fc.o2w[1], by, fmaf(fc.o2w[0], bx, fc.o2w[3])));
      const float wy = fmaf(fc.o2w[6], bz, fmaf(fc.o2w[5], by, fmaf(fc.o2w[4], bx, fc.o2w[7])));
      const float wz = fmaf(fc.o2w[10], bz, fmaf(fc.o2w[9], by, fmaf(fc.o2w[8], bx, fc.o2w[11])));
      const float cxp = fmaf(fc.vp[2], wz, fmaf(fc.vp[1], wy, fmaf(fc.vp[0], wx, fc.vp[3])));
      const float cyp = fmaf(fc.vp[6], wz, fmaf(fc.vp[5], wy, fmaf(fc.vp[4], wx, fc.vp[7])));
      const float cwp = fmaf(fc.vp[14], wz, fmaf(fc.vp[13], wy, fmaf(fc.vp[12], wx, fc.vp[15])));
      const bool behind = cwp <= 0.0f;   // clip.w is affine in position: its sign over the box is decided at the corners
      // view depth of the corner from the model-view matrix itself (not from clip.w: an orthographic projection has w == 1)
      const float tzc = fmaf(fc.mv[10], bz, fmaf(fc.mv[9], by, fmaf(fc.mv[8], bx, fc.mv[11])));
      const uint32_t nb = __ballot_sync(0xffffffffu, behind) & 0xffu;
      const uint32_t neg = __ballot_sync(0xffffffffu, tzc < 0.0f) & 0xffu;
      bool cull = nb == 0xffu;
      if (nb == 0u) {
        const float iw = 1.0f / cwp;
        float x0 = (cxp * iw * 0.5f + 0.5f) * fc.screenW, y0 = (0.5f - 0.5f * cyp * iw) * fc.screenH, x1 = x0, y1 = y0, zmin = fabsf(tzc);
#pragma unroll
        for (int o = 4; o; o >>= 1) {
          x0 = fminf(x0, __shfl_xor_sync(0xffffffffu, x0, o)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, o));
          y0 = fminf(y0, __shfl_xor_sync(0xffffffffu, y0, o)); y1 = fmaxf(y1, __shfl_xor_sync(0xffffffffu, y1, o));
          zmin = fminf(zmin, __shfl_xor_sync(0xffffffffu, zmin, o));
        }
        // |tz| over the box is at least the smallest corner value when the corners agree in sign (tz is affine); a box that
        // straddles tz = 0 gets no bound at all (reach = the 4096-pixel axis clamp)
        if (neg != 0u && neg != 0xffu) zmin = 0.0f;
        // largest decoded scale in the chunk: lerp(min,max,t)^8 <= max^8 for t in [0,1]
        float sm = fmaxf(f16hi(s_chunk.sclX), fmaxf(f16hi(s_chunk.sclY), f16hi(s_chunk.sclZ)));
        sm *= sm; sm *= sm; sm *= sm;
        const float reach = quad_reach(fc.extentK * sm * sm / (zmin * zmin) + 0.3f);
        // a range partition (group path) composites only its own pixel rows: everything else on the screen is some other GPU's
        const float ylo = part.range ? (float)(part.t0 * kTile) : 0.0f, yhi = part.range ? fminf((float)(part.t1 * kTile), fc.screenH) : fc.screenH;
        cull = (x1 + reach < 0.0f) || (x0 - reach > fc.screenW) || (y1 + reach < ylo) || (y0 - reach > yhi);
      }
      if (threadIdx.x == 0) s_cull = cull ? 1 : 0;
    }
    __syncthreads();
    if (s_cull) {
      if (idx < a.n) rect_out[idx] = kRectEmpty;
      if (threadIdx.x == 0) atomicAnd(block_bits + (blockIdx.x >> 5), ~(1u << (blockIdx.x & 31u)));
      if (early) chain_wait();
      return;
    }
  }

  uint32_t vw[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) vw[k] = 0;
  uint32_t rect = kRectEmpty;

  if (idx < a.n) {
    // ---- LoadSplatData, S/GaussianSplatting.hlsl:428-608 ----
    const uint32_t otherStride = 4 + vec_stride(a.scaleFmt) + (SHFMT == 4 ? 2u : 0u);  // + u16 SH index when clustered, :447-448
    const uint64_t otherAddr = (uint64_t)idx * otherStride;
    float3 pos = load_vector(a.pos, (uint64_t)idx * vec_stride(a.posFmt), a.posFmt);
    uint32_t rq;
    float3 scale;
    if (SHFMT != 4 && a.scaleFmt == 2) {  // 8-byte record: one aligned 64-bit load
      uint2 o = __ldg(reinterpret_cast<const uint2 *>(a.other + otherAddr));
      rq = o.x;
      scale = dec_11_10_11(o.y);
    } else if (SHFMT != 4 && a.scaleFmt == 0) {  // 16-byte record
      uint4 o = __ldg(reinterpret_cast<const uint4 *>(a.other + otherAddr));
      rq = o.x;
      scale = make_float3(__uint_as_float(o.y), __uint_as_float(o.z), __uint_as_float(o.w));
    } else {
      rq = (otherAddr & 3) == 0 ? ld_u32(a.other + otherAddr) : ld_u32_a2(a.other + otherAddr);
      scale = load_vector(a.other, otherAddr + 4, a.scaleFmt);
    }
    // DecodeRotation(DecodePacked_10_10_10_2), :219-229,:293-300
    float4 rot;
    {
      float px = (float)(rq & 1023) * GS_INV(1023.0f), py = (float)((rq >> 10) & 1023) * GS_INV(1023.0f),
            pz = (float)((rq >> 20) & 1023) * GS_INV(1023.0f);
      uint32_t qi = rq >> 30;  // round(w/3*3)
      const float kSqrt2 = 1.41421354f, kInvSqrt2 = 0.707106769f;
      float x = fmaf(px, kSqrt2, -kInvSqrt2), y = fmaf(py, kSqrt2, -kInvSqrt2), z = fmaf(pz, kSqrt2, -kInvSqrt2);
      float w = sqrtf(1.0f - satf(fmaf(z, z, fmaf(y, y, x * x))));
      rot = make_float4(x, y, z, w);
      if (qi == 0) rot = make_float4(w, x, y, z);
      if (qi == 1) rot = make_float4(x, w, y, z);
      if (qi == 2) rot = make_float4(x, y, w, z);
    }
    // colour texel (Morton-swizzled 2048-wide image), :423-426
    float4 col = make_float4(0.f, 0.f, 0.f, 0.f);
    auto load_color = [&]() {
      const uint32_t ti = splat_index_to_texel(idx);
      if (a.colFmt == 0) {
        col = __ldg(reinterpret_cast<const float4 *>(a.color) + ti);
      } else if (a.colFmt == 1) {
        uint2 e = __ldg(reinterpret_cast<const uint2 *>(a.color) + ti);
        col = make_float4(f16lo(e.x), f16hi(e.x), f16lo(e.y), f16hi(e.y));
      } else {
        uint32_t e;
        if (!BC7) {
          e = __ldg(reinterpret_cast<const uint32_t *>(a.color) + ti);
        } else {  // BC7: the texel's 4x4 block (16 B), then the one texel this splat owns (gs_bc7.cuh)
          const uint32_t x = ti & (kTexWidth - 1), y = ti / kTexWidth;
          const uint4 b = __ldg(reinterpret_cast<const uint4 *>(color_texel_ptr<true>(a, ti)));
          e = bc7::decode_texel(b.x, b.y, b.z, b.w, (y & 3u) * 4u + (x & 3u));
        }
        col = make_float4(__fdiv_rn((float)(e & 255u), 255.0f), __fdiv_rn((float)((e >> 8) & 255u), 255.0f),
                          __fdiv_rn((float)((e >> 16) & 255u), 255.0f), __fdiv_rn((float)(e >> 24), 255.0f));
      }
    };
    ShRaw<SHFMT> shr;
    constexpr uint32_t shStride = SHFMT == 0 ? 192u : (SHFMT == 1 || SHFMT == 4) ? 96u : SHFMT == 2 ? 60u : 32u;
    // shIndex, :467-470: the splat's own slot, or its palette entry
    const uint32_t shIdx = SHFMT == 4 ? ld_u16(a.other + otherAddr + otherStride - 2) : idx;
    if (!CULL) {
      load_color();
      if (fc.shOrder >= 1) shr.load(a.sh + (uint64_t)shIdx * shStride);
    }

    float3 shMin = make_float3(0.f, 0.f, 0.f), shMax = make_float3(1.f, 1.f, 1.f);
    if (chunked) {  // :565-603
      pos.x = lerpf(s_chunk.posX.x, s_chunk.posX.y, pos.x);
      pos.y = lerpf(s_chunk.posY.x, s_chunk.posY.y, pos.y);
      pos.z = lerpf(s_chunk.posZ.x, s_chunk.posZ.y, pos.z);
      scale.x = lerpf(f16lo(s_chunk.sclX), f16hi(s_chunk.sclX), scale.x);
      scale.y = lerpf(f16lo(s_chunk.sclY), f16hi(s_chunk.sclY), scale.y);
      scale.z = lerpf(f16lo(s_chunk.sclZ), f16hi(s_chunk.sclZ), scale.z);
      scale.x *= scale.x; scale.x *= scale.x; scale.x *= scale.x;
      scale.y *= scale.y; scale.y *= scale.y; scale.y *= scale.y;
      scale.z *= scale.z; scale.z *= scale.z; scale.z *= scale.z;
      shMin = make_float3(f16lo(s_chunk.shR), f16lo(s_chunk.shG), f16lo(s_chunk.shB));
      shMax = make_float3(f16hi(s_chunk.shR), f16hi(s_chunk.shG), f16hi(s_chunk.shB));
    }
    auto finish_color = [&]() {  // chunk un-lerp of colour + opacity, :573-583
      if (chunked) {
        col.x = lerpf(f16lo(s_chunk.colR), f16hi(s_chunk.colR), col.x);
        col.y = lerpf(f16lo(s_chunk.colG), f16hi(s_chunk.colG), col.y);
        col.z = lerpf(f16lo(s_chunk.colB), f16hi(s_chunk.colB), col.z);
        col.w = lerpf(f16lo(s_chunk.colA), f16hi(s_chunk.colA), col.w);
        // InvSquareCentered01, :5-11
        float x = col.w - 0.5f;
        x *= 0.5f;
        float sg = (x > 0.0f) ? 1.0f : ((x < 0.0f) ? -1.0f : 0.0f);
        col.w = sqrtf(fabsf(x)) * sg + 0.5f;
      }
    };
    if (!CULL) finish_color();
    const bool shLerp = chunked && SHFMT != 0 && SHFMT != 4;  // shFormat > FLOAT32 && <= NORM6, :585
    auto SH = [&](int j) -> float3 {
      float3 v = shr.get(j - 1);
      if (shLerp) { v.x = lerpf(shMin.x, shMax.x, v.x); v.y = lerpf(shMin.y, shMax.y, v.y); v.z = lerpf(shMin.z, shMax.z, v.z); }
      return v;
    };

    // ---- CSCalcViewData body, S/SplatUtilities.compute:199-251 ----
    float3 cw = make_float3(fmaf(fc.o2w[2], pos.z, fmaf(fc.o2w[1], pos.y, fmaf(fc.o2w[0], pos.x, fc.o2w[3]))),
                            fmaf(fc.o2w[6], pos.z, fmaf(fc.o2w[5], pos.y, fmaf(fc.o2w[4], pos.x, fc.o2w[7]))),
                            fmaf(fc.o2w[10], pos.z, fmaf(fc.o2w[9], pos.y, fmaf(fc.o2w[8], pos.x, fc.o2w[11]))));
    float4 clip;
    clip.x = fmaf(fc.vp[2], cw.z, fmaf(fc.vp[1], cw.y, fmaf(fc.vp[0], cw.x, fc.vp[3])));
    clip.y = fmaf(fc.vp[6], cw.z, fmaf(fc.vp[5], cw.y, fmaf(fc.vp[4], cw.x, fc.vp[7])));
    clip.z = fmaf(fc.vp[10], cw.z, fmaf(fc.vp[9], cw.y, fmaf(fc.vp[8], cw.x, fc.vp[11])));
    clip.w = fmaf(fc.vp[14], cw.z, fmaf(fc.vp[13], cw.y, fmaf(fc.vp[12], cw.x, fc.vp[15])));
    if (fc.bitsValid) {
      if (__ldg(deleted + (idx >> 5)) & (1u << (idx & 31))) clip.w = 0.0f;
    }
    if (fc.cutoutCount && is_splat_cut(fc, cutouts, pos)) clip.w = 0.0f;
    vw[0] = __float_as_uint(clip.x); vw[1] = __float_as_uint(clip.y); vw[2] = __float_as_uint(clip.z); vw[3] = __float_as_uint(clip.w);

    // the splat's edit-selection bit, fetched where it is needed (kept out of the long-lived registers)
    auto sel_bit = [&]() -> bool { return fc.selValid && ((__ldg(selected + (idx >> 5)) >> (idx & 31)) & 1u); };
    bool far_off = false;
    if (CULL && clip.w > 0.0f) {
      // Cheap conservative screen-extent bound BEFORE the covariance maths: lambda1 <= |J|_2^2 |W|_2^2 smax^2 + 0.3 with
      // |J|_2^2 = focal^2 (1 + |u|^2) / tz^2 (make_frame_consts, gs_api.cu), and the +-2 quad reaches at most quad_reach()
      // pixels from its centre.  A splat whose centre is further than that outside the screen can never produce a fragment:
      // the fused frame stores {pos, 0, 0} for it and skips rotation, covariance, eigen-decomposition and colour.
      const float tzq = fmaf(fc.mv[10], pos.z, fmaf(fc.mv[9], pos.y, fmaf(fc.mv[8], pos.x, fc.mv[11])));
      const float smax = fmaxf(scale.x, fmaxf(scale.y, scale.z));
      const float reach = quad_reach(fc.extentK * smax * smax / (tzq * tzq) + 0.3f);
      const float iw = 1.0f / clip.w;
      const float pcx = (clip.x * iw * 0.5f + 0.5f) * fc.screenW, pcy = (0.5f - 0.5f * clip.y * iw) * fc.screenH;
      const float ylo = part.range ? (float)(part.t0 * kTile) : 0.0f, yhi = part.range ? fminf((float)(part.t1 * kTile), fc.screenH) : fc.screenH;
      far_off = (pcx + reach < 0.0f) || (pcx - reach > fc.screenW) || (pcy + reach < ylo) || (pcy - reach > yhi);
    }

    if (!(clip.w <= 0.0f) && !far_off) {
      // CalcMatrixFromRotationScale, S/GaussianSplatting.hlsl:29-46
      const float x = rot.x, y = rot.y, z = rot.z, w = rot.w;
      float m[3][3];
      m[0][0] = (1.0f - 2.0f * (y * y + z * z)) * scale.x; m[0][1] = (2.0f * (x * y - w * z)) * scale.y; m[0][2] = (2.0f * (x * z + w * y)) * scale.z;
      m[1][0] = (2.0f * (x * y + w * z)) * scale.x; m[1][1] = (1.0f - 2.0f * (x * x + z * z)) * scale.y; m[1][2] = (2.0f * (y * z - w * x)) * scale.z;
      m[2][0] = (2.0f * (x * z - w * y)) * scale.x; m[2][1] = (2.0f * (y * z + w * x)) * scale.y; m[2][2] = (1.0f - 2.0f * (x * x + y * y)) * scale.z;
      // CalcCovariance3D :48-53 (* splatScale^2, S/SplatUtilities.compute:233-235)
      float sig[3][3];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = r; c < 3; ++c) sig[r][c] = sig[c][r] = (m[r][0] * m[c][0] + m[r][1] * m[c][1] + m[r][2] * m[c][2]) * fc.splatScale2;
      // CalcCovariance2D :56-90
      float vx = fmaf(fc.mv[2], pos.z, fmaf(fc.mv[1], pos.y, fmaf(fc.mv[0], pos.x, fc.mv[3])));
      float vy = fmaf(fc.mv[6], pos.z, fmaf(fc.mv[5], pos.y, fmaf(fc.mv[4], pos.x, fc.mv[7])));
      float tz = fmaf(fc.mv[10], pos.z, fmaf(fc.mv[9], pos.y, fmaf(fc.mv[8], pos.x, fc.mv[11])));
      float cxn = fminf(fmaxf(__fdiv_rn(vx, tz), -fc.limX), fc.limX), cyn = fminf(fmaxf(__fdiv_rn(vy, tz), -fc.limY), fc.limY);
      float tx = cxn * tz, ty = cyn * tz;
      float j00 = __fdiv_rn(fc.focal, tz), j02 = -__fdiv_rn(fc.focal * tx, tz * tz), j12 = -__fdiv_rn(fc.focal * ty, tz * tz);
      float T[2][3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        T[0][c] = j00 * fc.mv[c] + j02 * fc.mv[8 + c];
        T[1][c] = j00 * fc.mv[4 + c] + j12 * fc.mv[8 + c];
      }
      float vt[3][2];
#pragma unroll
      for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int i = 0; i < 2; ++i) vt[k][i] = sig[k][0] * T[i][0] + sig[k][1] * T[i][1] + sig[k][2] * T[i][2];
      float cov00 = T[0][0] * vt[0][0] + T[0][1] * vt[1][0] + T[0][2] * vt[2][0];
      float cov01 = T[0][0] * vt[0][1] + T[0][1] * vt[1][1] + T[0][2] * vt[2][1];
      float cov11 = T[1][0] * vt[0][1] + T[1][1] * vt[1][1] + T[1][2] * vt[2][1];
      cov00 += 0.3f; cov11 += 0.3f;
      // Second-stage cull (fused frame only), now that the 2-D covariance is known: the quad's half extents are
      // 2 (l1 |v_x| + l2 |v_y|) with l_i^2 = 2 lambda_i (lambda2 raised to 0.1 at most), and by Cauchy-Schwarz
      // l1 |v_x| + l2 |v_y| <= sqrt(2) sqrt(l1^2 v_x^2 + l2^2 v_y^2) <= sqrt(2) sqrt(2 cov00 + 0.2): at most 4 sqrt(cov + 0.1)
      // pixels per axis, a factor sqrt(2) from exact.  A quad that cannot reach the screen -- or, in a group, this GPU's rows --
      // skips eigen-decomposition, footprint and colour.
      bool reachable = true;
      if (CULL) {
        const float rx = 4.04f * sqrtf(cov00 + 0.1f) + 2.0f, ry = 4.04f * sqrtf(cov11 + 0.1f) + 2.0f;
        const float iw = 1.0f / clip.w;
        const float pcx = (clip.x * iw * 0.5f + 0.5f) * fc.screenW, pcy = (0.5f - 0.5f * clip.y * iw) * fc.screenH;
        const float ylo = part.range ? (float)(part.t0 * kTile) : 0.0f, yhi = part.range ? fminf((float)(part.t1 * kTile), fc.screenH) : fc.screenH;
        reachable = !((pcx + rx < 0.0f) || (pcx - rx > fc.screenW) || (pcy + ry < ylo) || (pcy - ry > yhi));
      }
      if (reachable) {
      // DecomposeCovariance, S/SplatUtilities.compute:149-159
      float mid = 0.5f * (cov00 + cov11);
      float hd = (cov00 - cov11) * 0.5f;
      float radius = sqrtf(hd * hd + cov01 * cov01);
      float lambda1 = mid + radius;
      float lambda2 = fmaxf(mid - radius, 0.1f);
      float dvx = cov01, dvy = lambda1 - cov00;
      float dl = sqrtf(dvx * dvx + dvy * dvy);
      dvx = __fdiv_rn(dvx, dl); dvy = __fdiv_rn(dvy, dl);
      dvy = -dvy;
      float l1 = fminf(sqrtf(2.0f * lambda1), 4096.0f), l2 = fminf(sqrtf(2.0f * lambda2), 4096.0f);
      float a1x = l1 * dvx, a1y = l1 * dvy, a2x = l2 * dvy, a2y = l2 * -dvx;
      vw[4] = __float_as_uint(a1x); vw[5] = __float_as_uint(a1y); vw[6] = __float_as_uint(a2x); vw[7] = __float_as_uint(a2y);
      bool drawable = true;
      if (CULL) {
        // can the +-2 quad touch a pixel centre at all?  (65000 = the largest opacity CSCalcViewData can emit: the
        // visible part is then the whole quad; a smaller opacity only shrinks it)
        SplatFootprint g0;
        // (multi-GPU: ... or only rows of other ranks' bands -- then its colour is somebody else's job)
        drawable = splat_footprint(clip, a1x, a1y, a2x, a2y, 65000.0f, fc.screenW, fc.screenH, g0) &&
                   rect_entries(footprint_tile_rect(g0, fc, part), part) != 0;
        if (drawable) {
          load_color();
          finish_color();
          // alpha = sat(exp_neg(..) * half(min(opacity*scale, 65000))) stays below 1/255 when the half is below 0.00392
          // (a selected splat's alpha does not depend on its opacity at all)
          drawable = __half2float(__float2half_rn(fminf(col.w * fc.opacityScale, 65000.0f))) >= 0.00392f || sel_bit();
          if (drawable && fc.shOrder >= 1) shr.load(a.sh + (uint64_t)shIdx * shStride);
        }
      }
      if (drawable) {
      // colour: ShadeSH(objViewDir), :240-248 + S/GaussianSplatting.hlsl:139-179
        float wx = fc.cam_pos[0] - cw.x, wy = fc.cam_pos[1] - cw.y, wz = fc.cam_pos[2] - cw.z;
        float ox = fmaf(fc.w2o[2], wz, fmaf(fc.w2o[1], wy, fc.w2o[0] * wx));
        float oy = fmaf(fc.w2o[5], wz, fmaf(fc.w2o[4], wy, fc.w2o[3] * wx));
        float oz = fmaf(fc.w2o[8], wz, fmaf(fc.w2o[7], wy, fc.w2o[6] * wx));
        float ol = sqrtf(ox * ox + oy * oy + oz * oz);
        ox = __fdiv_rn(ox, ol); oy = __fdiv_rn(oy, ol); oz = __fdiv_rn(oz, ol);
        const float dx = ox * -1.0f, dy = oy * -1.0f, dz = oz * -1.0f;  // dir *= -1
        float3 res = fc.shOnly ? make_float3(0.5f, 0.5f, 0.5f) : make_float3(col.x, col.y, col.z);
        if (fc.shOrder >= 1) {
          const float SH_C1 = 0.4886025f;
          res = res + SH_C1 * (neg(SH(1)) * dy + SH(2) * dz - SH(3) * dx);
          if (fc.shOrder >= 2) {
            const float xx = dx * dx, yy = dy * dy, zz = dz * dz, xy = dx * dy, yz = dy * dz, xz = dx * dz;
            res = res + ((1.0925484f * xy) * SH(4) + (-1.0925484f * yz) * SH(5) + (0.3153916f * (2.0f * zz - xx - yy)) * SH(6) +
                         (-1.0925484f * xz) * SH(7) + (0.5462742f * (xx - yy)) * SH(8));
            if (fc.shOrder >= 3) {
              res = res + ((-0.5900436f * dy * (3.0f * xx - yy)) * SH(9) + (2.8906114f * xy * dz) * SH(10) +
                           (-0.4570458f * dy * (4.0f * zz - xx - yy)) * SH(11) + (0.3731763f * dz * (2.0f * zz - 3.0f * xx - 3.0f * yy)) * SH(12) +
                           (-0.4570458f * dx * (4.0f * zz - xx - yy)) * SH(13) + (1.4453057f * dz * (xx - yy)) * SH(14) +
                           (-0.5900436f * dx * (xx - 3.0f * yy)) * SH(15));
            }
          }
        }
        res.x = (res.x > 0.0f) ? res.x : 0.0f; res.y = (res.y > 0.0f) ? res.y : 0.0f; res.z = (res.z > 0.0f) ? res.z : 0.0f;
        float alpha = fminf(col.w * fc.opacityScale, 65000.0f);
        vw[8] = (f32tof16(res.x) << 16) | f32tof16(res.y);
        vw[9] = (f32tof16(res.z) << 16) | f32tof16(alpha);
      }
      SplatFootprint fp;
      if (drawable && splat_footprint(clip, a1x, a1y, a2x, a2y, f16lo(vw[9]), fc.screenW, fc.screenH, fp, sel_bit())) {
        rect = footprint_tile_rect(fp, fc, part);
        if (rect != kRectEmpty) {
          // raster-ready record (48 B): everything the per-pixel loop needs, so the compositor stages it with three
          // 16-byte async copies and no arithmetic.  Colours are the half-rounded values of the SplatViewData record.
          float4 *d = draw_out + (size_t)idx * 3;
          d[0] = make_float4(fp.cx, fp.cy, fp.i1x, fp.i1y);
          d[1] = make_float4(fp.i2x, fp.i2y, fp.ca, fp.hx);
          d[2] = make_float4(f16hi(vw[8]), f16lo(vw[8]), f16hi(vw[9]), fp.hy);
          // depth of the (flat) quad's fragments, for the depth test against the scene's depth buffer when one is bound
          if (zndc) zndc[idx] = __fdiv_rn(clip.z, clip.w);
        }
      }
      }  // reachable
    }
    rect_out[idx] = rect;
  }
  {  // one BIT per 256-splat block: "some splat of this block has a bin rectangle" (set or cleared here, by its CTA).  The
     // binner walks the draw order and gathers a splat's rectangle only when its block's bit is set; the bitmap (n/2048 bytes:
     // 3 KB for cfg2) sits in the binner's shared memory, so the per-entry test is a shared-memory read and the random
     // 4-byte gathers are paid for blocks with something to draw only (every other GPU's blocks drop out in a group).
    const int any = __syncthreads_or(rect != kRectEmpty);
    if (threadIdx.x == 0) {
      if (any) atomicOr(block_bits + (blockIdx.x >> 5), 1u << (blockIdx.x & 31u));
      else atomicAnd(block_bits + (blockIdx.x >> 5), ~(1u << (blockIdx.x & 31u)));
    }
  }

  if (CULL) {
    if (early) chain_wait();
    return;
  }   // fused frame: the compositor reads the 48-byte draw records; _SplatViewData is not materialised
  // ---- coalesced store of the CTA's 256 x 40-byte records ----
#pragma unroll
  for (int k = 0; k < 10; ++k) s_view[threadIdx.x * 10 + k] = vw[k];
  __syncthreads();
  const uint32_t first = blockIdx.x * 256;
  const uint32_t cnt = min(256u, a.n - first);
  const uint32_t words = cnt * 10;
  uint4 *dst = reinterpret_cast<uint4 *>(view_out + (uint64_t)first * 10);
  const uint4 *src = reinterpret_cast<const uint4 *>(s_view);
  for (uint32_t q = threadIdx.x; q * 4 + 3 < words; q += 256) dst[q] = src[q];
  // tail words when cnt*10 is not a multiple of 4 (only the last CTA)
  for (uint32_t wi = (words & ~3u) + threadIdx.x; wi < words; wi += 256) view_out[(uint64_t)first * 10 + wi] = s_view[wi];
  if (early) chain_wait();
}

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
void launch_set_indices(uint32_t *order, uint32_t n, cudaStream_t s) {
  if (n) k_set_indices<<<(n + 255) / 256, 256, 0, s>>>(order, n);
}

void launch_calc_distances(const AssetView &a, const FrameConsts &fc, uint32_t *key_table, uint32_t *ghist, cudaStream_t s, const SlabArgs *slabs) {
  if (!a.n) return;
  const uint32_t per = 256 * kDistItems;
  const uint32_t tiles = (a.n + per - 1) / per;
  const uint32_t grid = min(tiles, sm_count() * 8u);
  const float4 row = make_float4(fc.sort_row[0], fc.sort_row[1], fc.sort_row[2], fc.sort_row[3]);
  SlabArgs none{};
  if (slabs && slabs->count > 1) cudaMemsetAsync(slabs->group_bits, 0, group_bits_words(a.n) * sizeof(uint32_t), s);
  if (!slabs || slabs->count <= 1) chain_launch(k_calc_distances<0>, grid, 256, 0, s, a, row, key_table, ghist, none);
  else if (slabs->count <= 2) chain_launch(k_calc_distances<1>, grid, 256, 0, s, a, row, key_table, ghist, *slabs);
  else if (slabs->count <= 4) chain_launch(k_calc_distances<3>, grid, 256, 0, s, a, row, key_table, ghist, *slabs);
  else if (slabs->count <= 8) chain_launch(k_calc_distances<7>, grid, 256, 0, s, a, row, key_table, ghist, *slabs);
  else chain_launch(k_calc_distances<kMaxSlabs - 1>, grid, 256, 0, s, a, row, key_table, ghist, *slabs);
}

template <bool CULL>
static void launch_calc_view_t(const AssetView &a, const FrameConsts &fc, const GsCutout *cutouts, const uint32_t *deleted, const uint32_t *selected, uint32_t *view,
                               uint32_t *rect, float4 *draw, uint32_t *block_bits, float *zndc, const Partition &part, bool after_sort,
                               cudaStream_t s) {
  const uint32_t grid = (a.n + 255) / 256, early = after_sort ? 1u : 0u;
  // BC7 colour (VeryLow preset) is a separate instantiation: the block decode must not cost the other formats registers
#define GS_VIEW(SH)                                                                                                        \
  do {                                                                                                                    \
    if (a.colFmt == 3)                                                                                                    \
      chain_launch(k_calc_view<SH, CULL, true>, grid, 256, 0, s, a, fc, cutouts, deleted, selected, view, rect, draw, block_bits, zndc, part, early); \
    else                                                                                                                  \
      chain_launch(k_calc_view<SH, CULL, false>, grid, 256, 0, s, a, fc, cutouts, deleted, selected, view, rect, draw, block_bits, zndc, part, early); \
  } while (0)
  switch (a.shFmt) {
    case 0: GS_VIEW(0); break;
    case 1: GS_VIEW(1); break;
    case 2: GS_VIEW(2); break;
    case 3: GS_VIEW(3); break;
    default: GS_VIEW(4); break;  // Cluster64k..4k
  }
#undef GS_VIEW
}

void launch_calc_view(const AssetView &a, const FrameConsts &fc, const GsCutout *cutouts, const uint32_t *deleted, const uint32_t *selected, uint32_t *view,
                      uint32_t *rect, float4 *draw, uint32_t *block_bits, float *zndc, bool cull_undrawable, const Partition &part, cudaStream_t s,
                      bool after_sort) {
  if (!a.n) return;
  // no clear of block_bits: every CTA sets or clears its own bit
  if (cull_undrawable) launch_calc_view_t<true>(a, fc, cutouts, deleted, selected, view, rect, draw, block_bits, zndc, part, after_sort, s);
  else launch_calc_view_t<false>(a, fc, cutouts, deleted, selected, view, rect, draw, block_bits, zndc, part, after_sort, s);
}

}  // namespace gs
