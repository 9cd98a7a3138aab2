// gs_common.cuh -- shared device/host definitions of libgsplat_b200 (sm_90a only).
//
// Arithmetic contract (DESIGN.md "Arithmetic"): IEEE float32, compiled with -fmad=false so
// nothing is contracted behind our back; FMAs are written explicitly with fmaf().  The
// CPU oracle (oracle/, test infrastructure) was designed against the same contract, which
// is what lets the parity tests ask for bit-equality instead of a tolerance.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gsplat_b200.h"
#include "gs_asset_format.h"   // kChunkSize, kTexWidth, vec_stride, splat_index_to_texel, ChunkInfo

namespace gs {

constexpr int kTile = 16;           // raster CTA tile edge in pixels
constexpr int kBin = 64;            // binning cell edge in pixels: one list per 64x64 cell, shared by its sixteen 16x16 raster tiles
constexpr int kViewStride = 40;     // sizeof(SplatViewData), S/GaussianSplatting.hlsl:610-615

// SplatChunkInfo as the frame kernels read it (S/GaussianSplatting.hlsl:196-202): ChunkInfo with float2 ranges, 16-byte aligned
struct __align__(16) Chunk {
  uint32_t colR, colG, colB, colA;
  float2 posX, posY, posZ;
  uint32_t sclX, sclY, sclZ;
  uint32_t shR, shG, shB;
};
static_assert(sizeof(Chunk) == sizeof(ChunkInfo) && offsetof(Chunk, posX) == offsetof(ChunkInfo, posX) &&
                  offsetof(Chunk, posZ) == offsetof(ChunkInfo, posZ) && offsetof(Chunk, sclX) == offsetof(ChunkInfo, sclX) &&
                  offsetof(Chunk, shB) == offsetof(ChunkInfo, shB),
              "Chunk is ChunkInfo's layout");
static_assert(kBin == (int)GS_BAND_PIXELS, "the public header documents the partition row height");

// SplatViewData as two 16-byte vectors + one 8-byte vector
struct ViewRec {
  float4 pos;     // clip-space centre
  float4 axes;    // axis1.xy, axis2.xy
  uint2 color;    // (f16 r << 16 | f16 g), (f16 b << 16 | f16 a)
};

// Per-frame constants, computed once on the host (gs_api.cu: make_frame_consts).
struct FrameConsts {
  float o2w[12];     // rows 0..2 of _MatrixObjectToWorld, row-major [r*4+c]
  float w2o[9];      // 3x3 of _MatrixWorldToObject, row-major
  float mv[12];      // rows 0..2 of _MatrixMV (view * o2w)
  float vp[16];      // UNITY_MATRIX_VP, row-major
  float sort_row[4]; // row 2 of (diag(1,1,-1)*view) * o2w  -- CSCalcDistances
  float cam_pos[3];
  float limX, limY, focal, splatScale2, opacityScale;
  float extentK;     // focal^2 * (1 + limX^2 + limY^2) * |MV3x3|_2^2 * splatScale^2: lambda1(cov2d) <= extentK * smax^2 / tz^2 + 0.3
  float screenW, screenH;
  uint32_t shOrder, shOnly;
  uint32_t cutoutCount, bitsValid;
  uint32_t selValid;       // an edit selection is bound (_SplatSelectedBits): selected splats take the pixel shader's other branch
  uint32_t binsX, binsY;   // kBin-pixel binning cells
};

struct AssetView {     // device pointers + formats of one uploaded asset
  uint32_t n;
  uint32_t posFmt, scaleFmt, shFmt, colFmt;
  uint32_t chunkCount;
  const uint8_t *pos, *other, *sh, *color;
  const Chunk *chunks;
};

// Pixels the +-2 quad of a splat can reach from its centre, given the bound `l1sq` on lambda1 of its 2-D covariance:
// 2 (|a1x| + |a2x|) <= 2 sqrt(2) |axis1|, |axis1| = min(sqrt(2 lambda1), 4096); 2.9 instead of 2.83 and the two extra pixels
// absorb float rounding and the slight non-orthonormality of an un-renormalised decoded rotation.
__device__ __forceinline__ float quad_reach(float l1sq) { return 2.9f * fminf(sqrtf(2.0f * l1sq), 4096.0f) + 2.0f; }

// ---- decoupled look-back over single-word block statuses, 32 predecessors per round ----------------------------------
// status[b] = (LOCAL | total) once block b knows its own total, (INCL | inclusive prefix) once it knows everything before
// it too; 0 = not published yet.  Called by ONE WARP of block b (b > 0), returns the exclusive prefix of b to every lane.
// (A 128-wide variant -- four predecessors per lane -- was measured and is SLOWER.  A round can only be summed once ALL the polled predecessors have published, so a wider round waits
// for the slowest of four times as many blocks; the wait for neighbours to publish, not the number of rounds, is what
// the barrier stalls in ncu are.)  Sums saturate at the value mask (callers treat a saturated total as overflow).
enum : uint32_t { kLbLocal = 1u << 30, kLbIncl = 2u << 30, kLbMask = (1u << 30) - 1u };

__device__ __forceinline__ uint32_t lookback_exclusive(volatile uint32_t *status, uint32_t b) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t excl = 0;
  int top = (int)b - 1;
  while (true) {
    const int idx = top - (int)lane;
    uint32_t v;
    do {
      v = idx >= 0 ? status[idx] : (uint32_t)kLbIncl;
    } while (__any_sync(0xffffffffu, v == 0));
    const uint32_t incl_mask = __ballot_sync(0xffffffffu, (v & kLbIncl) != 0);
    const int first = incl_mask ? __ffs(incl_mask) - 1 : 31;   // nearest predecessor that is already inclusive
    uint32_t contrib = ((int)lane <= first) ? (v & (uint32_t)kLbMask) : 0u;
#pragma unroll
    for (int o = 16; o; o >>= 1) contrib = min(contrib + __shfl_xor_sync(0xffffffffu, contrib, o), (uint32_t)kLbMask);
    excl = min(excl + contrib, (uint32_t)kLbMask);
    if (incl_mask) break;
    top -= 32;
  }
  return excl;
}

// ---- launch chain (programmatic dependent launch) ------------------------------------------------
// A kernel launched by chain_launch (gs_kernels.cuh) may be placed on the SMs while its predecessor on the stream still
// drains.  chain_wait() blocks until the predecessor grid has completed and its writes are visible; chain_release() lets
// the successor be placed once every CTA of this grid has released or exited.  Both are no-ops in an ordinary launch.
// Rules every chained kernel keeps (DESIGN §5 "Launch chain"):
//   * every CTA calls chain_wait() before it exits, on every path, so that a grid's completion implies its predecessor's;
//   * chain_release() comes after chain_wait(), so that when a kernel starts, every node before its immediate predecessor has
//     completed.  The exceptions release earlier only where the successor's pre-wait work is safe beside the releasing
//     kernel and the node before it (k_tile_order and the early k_calc_view, whose successors wait first, and the depth
//     sort's k_clear, whose successor k_calc_distances writes only key_table before its wait);
//   * work before chain_wait() touches nothing the immediate predecessor reads or writes (listed beside each call).
__device__ __forceinline__ void chain_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void chain_release() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- small device helpers -------------------------------------------------------------
__device__ __forceinline__ float f16lo(uint32_t v) { return __half2float(__ushort_as_half((unsigned short)(v & 0xffffu))); }
__device__ __forceinline__ float f16hi(uint32_t v) { return __half2float(__ushort_as_half((unsigned short)(v >> 16))); }
__device__ __forceinline__ uint32_t f32tof16(float f) { return (uint32_t)__half_as_ushort(__float2half_rn(f)); }
__device__ __forceinline__ float lerpf(float a, float b, float t) { return fmaf(t, b - a, a); }
__device__ __forceinline__ float satf(float v) { return (v > 0.0f) ? ((v < 1.0f) ? v : 1.0f) : 0.0f; }

// S/SplatUtilities.compute:52-57
__device__ __forceinline__ uint32_t float_to_sortable_uint(float f) {
  uint32_t fu = __float_as_uint(f);
  uint32_t mask = (uint32_t)(-(int32_t)(fu >> 31)) | 0x80000000u;
  return fu ^ mask;
}

// Deterministic exp for x <= 0 (see DESIGN.md): 2^(x*log2e), magic-number rint, degree-5 polynomial.
__device__ __forceinline__ float exp_neg(float x) {
  float t = x * 1.44269502f;
  t = (t > -125.0f) ? t : -125.0f;
  float m = t + 12582912.0f;
  float n = m - 12582912.0f;
  float f = t - n;
  float p = 0.0013276503887027502f;
  p = fmaf(p, f, 0.009675541892647743f);
  p = fmaf(p, f, 0.05550713092088699f);
  p = fmaf(p, f, 0.24022120237350464f);
  p = fmaf(p, f, 0.6931469440460205f);
  p = fmaf(p, f, 1.0000001192092896f);
  int ni = (int)(__float_as_uint(m) - 0x4B400000u);
  return __uint_as_float((uint32_t)((int)__float_as_uint(p) + (ni << 23)));
}

// ---- unorm decoders (S/GaussianSplatting.hlsl:261-300); "/K" == "* (1/K)" by contract ----
#define GS_INV(K) (1.0f / K)
__device__ __forceinline__ float3 dec_6_5_5(uint32_t e) {
  return make_float3((float)(e & 63) * GS_INV(63.0f), (float)((e >> 6) & 31) * GS_INV(31.0f), (float)((e >> 11) & 31) * GS_INV(31.0f));
}
__device__ __forceinline__ float3 dec_5_6_5(uint32_t e) {
  return make_float3((float)(e & 31) * GS_INV(31.0f), (float)((e >> 5) & 63) * GS_INV(63.0f), (float)((e >> 11) & 31) * GS_INV(31.0f));
}
__device__ __forceinline__ float3 dec_11_10_11(uint32_t e) {
  return make_float3((float)(e & 2047) * GS_INV(2047.0f), (float)((e >> 11) & 1023) * GS_INV(1023.0f), (float)((e >> 21) & 2047) * GS_INV(2047.0f));
}
__device__ __forceinline__ float3 dec_16_16_16(uint32_t lo, uint32_t hi) {
  return make_float3((float)(lo & 65535) * GS_INV(65535.0f), (float)((lo >> 16) & 65535) * GS_INV(65535.0f), (float)(hi & 65535) * GS_INV(65535.0f));
}

__device__ __forceinline__ uint32_t ld_u16(const uint8_t *p) { return (uint32_t)__ldg(reinterpret_cast<const unsigned short *>(p)); }
__device__ __forceinline__ uint32_t ld_u32(const uint8_t *p) { return __ldg(reinterpret_cast<const uint32_t *>(p)); }
// 4-byte value at a 2-byte-aligned address (strides 6 and 2 straddle words; the HLSL does the
// same with shifts, S/GaussianSplatting.hlsl:334-344)
__device__ __forceinline__ uint32_t ld_u32_a2(const uint8_t *p) { return ld_u16(p) | (ld_u16(p + 2) << 16); }

// LoadAndDecodeVector, S/GaussianSplatting.hlsl:346-392
__device__ __forceinline__ float3 load_vector(const uint8_t *base, uint64_t addr, uint32_t fmt) {
  const uint8_t *p = base + addr;
  if (fmt == 0) {
    if ((addr & 3) == 0) return make_float3(__uint_as_float(ld_u32(p)), __uint_as_float(ld_u32(p + 4)), __uint_as_float(ld_u32(p + 8)));
    return make_float3(__uint_as_float(ld_u32_a2(p)), __uint_as_float(ld_u32_a2(p + 4)), __uint_as_float(ld_u32_a2(p + 8)));
  } else if (fmt == 1) {
    return dec_16_16_16(ld_u32_a2(p), ld_u16(p + 4));
  } else if (fmt == 2) {
    return dec_11_10_11((addr & 3) == 0 ? ld_u32(p) : ld_u32_a2(p));
  }
  return dec_6_5_5(ld_u16(p));
}

}  // namespace gs

// ---- host-side error plumbing -------------------------------------------------------------
#define GS_CUDA_TRY(ctx, expr)                                                   \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) return gs::fail_cuda((ctx), _e, #expr, __FILE__, __LINE__); \
  } while (0)
