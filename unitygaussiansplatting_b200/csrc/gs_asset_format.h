// gs_asset_format.h -- the byte layout of a splat asset, shared by the host packer (asset_creator.cpp,
// asset_cluster_bc7.cpp: libgsplat_asset.so, g++), the GPU packer (gs_pack.cu) and gs_asset_upload's size checks
// (libgsplat_b200.so, nvcc): blob sizes, the chunk record, the k-means' pcg stream, the scalar encoders, one splat's
// records, the chunk header, the k-means squared distance and the BC7 mode-6 block encoder.  Each is written once here,
// so the two packers cannot drift apart; what they still do their own way (reductions, sorts, the k-means structure) is
// in DESIGN.md, "The packer on the GPU".
//
// Plain C++ without CUDA headers: under nvcc every function is __host__ __device__.  The arithmetic relies on what both
// builds guarantee: no contraction (-ffp-contract=off, -fmad=false), IEEE division and square root.
//
// Third-party arithmetic that is not in the reference: Unity.Mathematics 1.2.6 math.f32tof16 / math.min / math.max /
// math.saturate.  f32tof16 is restated from its published source (truncate the low 12 mantissa bits, add half, shift;
// i.e. round half up on bit 12); min / max return their second operand unless the first wins strictly or the second is
// NaN, so saturate(NaN) = max(0, min(1, NaN)) = 1.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define GS_FMT __host__ __device__ __forceinline__
#else
#define GS_FMT inline
#endif

namespace gs {

constexpr uint32_t kChunkSize = 256;   // R/GaussianSplatAsset.cs:14, S/GaussianSplatting.hlsl:207
constexpr uint32_t kTexWidth = 2048;   // R/GaussianSplatAsset.cs:15, S/GaussianSplatting.hlsl:181

// the input record, InputSplatData (GsaInputSplat / GsInputSplat): 62 floats
constexpr uint32_t kRecFloats = 62;
constexpr uint32_t kOffDc0 = 6, kOffSh = 9, kOffOpacity = 54, kOffScale = 55, kOffRot = 58;

GS_FMT uint32_t f32_bits(float f) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
#endif
}
GS_FMT float f32_from_bits(uint32_t u) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}

// ---- sizes (R/GaussianSplatAsset.cs) ----------------------------------------------------------------------------------
GS_FMT uint32_t vec_stride(uint32_t fmt) { return fmt == 0 ? 12u : fmt == 1 ? 6u : fmt == 2 ? 4u : 2u; }   // :39-49
GS_FMT uint32_t color_size(uint32_t fmt) { return fmt == 0 ? 16u : fmt == 1 ? 8u : fmt == 2 ? 4u : 1u; }   // :58-68, per texel
// :83-101; a clustered format's palette entries are SHTableItemFloat16
GS_FMT uint32_t sh_stride(uint32_t fmt) { return fmt == 0 ? 192u : fmt == 1 ? 96u : fmt == 2 ? 60u : fmt == 3 ? 32u : 96u; }
GS_FMT uint32_t sh_count(uint32_t fmt, uint32_t n) { return fmt <= 3 ? n : (65536u >> (fmt - 4)); }   // GetSHCount, :135-150
// rotation, scale, and the u16 palette index of clustered SH (E/GaussianSplatAssetCreator.cs:837-842)
GS_FMT uint32_t other_stride(uint32_t sf, uint32_t shf) { return 4 + vec_stride(sf) + (shf > 3 ? 2 : 0); }
GS_FMT uint32_t tex_height(uint64_t n) {   // :152-160: whole 16-row tiles of the 2048-wide image
  uint64_t h = (n + kTexWidth - 1) / kTexWidth;
  if (h == 0) h = 1;
  return (uint32_t)((h + 15) / 16 * 16);
}
GS_FMT bool uses_chunks(uint32_t pf, uint32_t sf, uint32_t cf, uint32_t shf) {   // E/...:54-58
  return pf != 0 || sf != 0 || cf != 0 || shf != 0;
}
GS_FMT uint64_t next_multiple(uint64_t v, uint64_t m) { return (v + m - 1) / m * m; }

// The five blob sizes (GsaSizes or GsPackSizes).  False for an unknown format, and for clustered SH whose palette would
// not be smaller than the data: the reference then skips clustering (E/...:480-482) and writes an asset its own shader
// mis-reads (no index in `other`, empty SH blob).
template <class Sizes>
inline bool calc_sizes(uint32_t n, uint32_t pf, uint32_t sf, uint32_t cf, uint32_t shf, Sizes *out) {
  if (pf > 3 || sf > 3 || cf > 3 || shf > 8) return false;
  if (shf > 3 && n <= sh_count(shf, n)) return false;
  out->tex_width = kTexWidth;
  out->tex_height = tex_height(n);
  out->pos_bytes = next_multiple((uint64_t)n * vec_stride(pf), 8);             // E/...:815
  out->other_bytes = next_multiple((uint64_t)n * other_stride(sf, shf), 8);    // E/...:837-842
  out->color_bytes = (uint64_t)kTexWidth * out->tex_height * color_size(cf);
  out->sh_bytes = (uint64_t)sh_count(shf, n) * sh_stride(shf);                 // clustered: the palette only (E/...:1048-1051)
  out->chunk_bytes = uses_chunks(pf, sf, cf, shf) ? (uint64_t)((n + kChunkSize - 1) / kChunkSize) * 64 : 0;
  return true;
}

// ---- the chunk record, SplatChunkInfo (R/GaussianSplatAsset.cs:231-237, 64 bytes) --------------------------------------
struct ChunkInfo {
  uint32_t colR, colG, colB, colA;
  float posX[2], posY[2], posZ[2];
  uint32_t sclX, sclY, sclZ;
  uint32_t shR, shG, shB;
};
static_assert(sizeof(ChunkInfo) == 64, "ChunkInfo must be 64 bytes");

// ---- the k-means' pcg stream (E/Utils/KMeansClustering.cs:571-593) ----------------------------------------------------
GS_FMT uint32_t pcg_step(uint32_t state) { return state * 747796405u + 2891336453u; }
GS_FMT uint32_t pcg_output(uint32_t state) {
  const uint32_t word = ((state >> ((state >> 28) + 4u)) ^ state) * 277803737u;
  return (word >> 22) ^ word;
}
GS_FMT uint32_t pcg_hash(uint32_t input) { return pcg_output(pcg_step(input)); }
GS_FMT uint32_t pcg_random(uint32_t &rng_state) {
  const uint32_t state = rng_state;
  rng_state = pcg_step(rng_state);
  return pcg_output(state);
}
GS_FMT float pcg_hash_float(uint32_t input, float up_to) {
  return (f32_from_bits(0x3f800000u | (pcg_hash(input) >> 9)) - 1.0f) * up_to;
}
// MakeBatchJob (K:456-477): `batch` distinct indices below n, in draw order.  `picked` (n flags) is all zero on entry and
// on return.
inline void random_batch(uint32_t n, uint32_t &rng, uint32_t batch, uint8_t *picked, uint32_t *out) {
  uint32_t seed = pcg_random(rng);
  uint32_t got = 0;
  while (got < batch) {
    const uint32_t index = pcg_hash(seed++) % n;
    if (!picked[index]) { picked[index] = 1; out[got++] = index; }
  }
  for (uint32_t i = 0; i < batch; ++i) picked[out[i]] = 0;
}

// DistanceSquared, K:138-206 (the x86 AVX path): per block of 8, pairs of squares added pairwise, then left to right
GS_FMT float distance_squared(const float *a, const float *b, uint32_t dim) {
  float d = 0.0f;
  uint32_t i = 0;
  for (; i + 7 < dim; i += 8) {
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { const float t = a[i + k] - b[i + k]; v[k] = t * t; }
    d += (v[0] + v[1]) + (v[2] + v[3]) + (v[4] + v[5]) + (v[6] + v[7]);
  }
  for (; i < dim; ++i) { const float t = a[i] - b[i]; d += t * t; }
  return d;
}

// ---- scalar encoders ----------------------------------------------------------------------------------------------------
// Unity.Mathematics math.f32tof16 (see the file header)
GS_FMT uint32_t unity_f32tof16(float x) {
  const int32_t infinity_32 = 255 << 23;
  const uint32_t msk = 0x7FFFF000u;
  const uint32_t ux = f32_bits(x), uux = ux & msk;
  const float a = f32_from_bits(uux) * 1.92592994e-34f;
  const float scaled = (260042752.0f < a) ? 260042752.0f : a;   // math.min(a, 260042752)
  uint32_t h = (f32_bits(scaled) + 0x1000u) >> 13;
  if ((int32_t)uux >= infinity_32) h = ((int32_t)uux > infinity_32) ? 0x7e00u : 0x7c00u;
  return h | ((ux & ~msk) >> 16);
}
// math.min / max / saturate: of two equal values (+0 / -0) the second is kept, a NaN second operand is ignored.  Every
// min / max fold of the importer (bounds, chunk ranges) goes through these.
GS_FMT float unity_min(float x, float y) { return (isnan(y) || x < y) ? x : y; }
GS_FMT float unity_max(float x, float y) { return (isnan(y) || x > y) ? x : y; }
GS_FMT float saturate(float v) { return unity_max(0.0f, unity_min(1.0f, v)); }   // clamp(v, 0, 1); NaN -> 1

// R/GaussianUtils.cs:25-30
GS_FMT float square_centered01(float x) {
  x -= 0.5f;
  const float sgn = (x > 0.0f) ? 1.0f : ((x < 0.0f) ? -1.0f : 0.0f);
  x *= x * sgn;
  return x * 2.0f + 0.5f;
}

// R/GaussianUtils.cs:81-95
GS_FMT uint64_t morton_part1by2(uint64_t x) {
  x &= 0x1fffff;
  x = (x ^ (x << 32)) & 0x1f00000000ffffULL;
  x = (x ^ (x << 16)) & 0x1f0000ff0000ffULL;
  x = (x ^ (x << 8)) & 0x100f00f00f00f00fULL;
  x = (x ^ (x << 4)) & 0x10c30c30c30c30c3ULL;
  x = (x ^ (x << 2)) & 0x1249249249249249ULL;
  return x;
}
GS_FMT uint64_t morton_encode3(uint32_t x, uint32_t y, uint32_t z) {
  return (morton_part1by2(z) << 2) | (morton_part1by2(y) << 1) | morton_part1by2(x);
}

// Linear texel index of splat `idx` in the 2048-wide colour image: Morton order inside 16x16 tiles
// (E/GaussianSplatAssetCreator.cs:863-871, S/GaussianSplatting.hlsl:120-127 + :183-194)
GS_FMT uint32_t splat_index_to_texel(uint32_t idx) {
  uint32_t t = (idx & 0xFF) | ((idx & 0xFE) << 7);
  t &= 0x5555;
  t = (t ^ (t >> 1)) & 0x3333;
  t = (t ^ (t >> 2)) & 0x0f0f;
  uint32_t mx = t & 0xF, my = t >> 8;
  uint32_t tile = idx >> 8;
  uint32_t x = (tile % (kTexWidth / 16)) * 16 + mx, y = (tile / (kTexWidth / 16)) * 16 + my;
  return y * kTexWidth + x;
}

// E/GaussianSplatAssetCreator.cs:705-725 -- all truncating casts
GS_FMT uint64_t enc_norm16(const float v[3]) {
  return (uint64_t)(v[0] * 65535.5f) | ((uint64_t)(v[1] * 65535.5f) << 16) | ((uint64_t)(v[2] * 65535.5f) << 32);
}
GS_FMT uint32_t enc_norm11(const float v[3]) {
  return (uint32_t)(v[0] * 2047.5f) | ((uint32_t)(v[1] * 1023.5f) << 11) | ((uint32_t)(v[2] * 2047.5f) << 21);
}
GS_FMT uint32_t enc_norm655(const float v[3]) {
  return ((uint32_t)(v[0] * 63.5f) | ((uint32_t)(v[1] * 31.5f) << 6) | ((uint32_t)(v[2] * 31.5f) << 11)) & 0xffffu;
}
GS_FMT uint32_t enc_norm565(const float v[3]) {
  return ((uint32_t)(v[0] * 31.5f) | ((uint32_t)(v[1] * 63.5f) << 5) | ((uint32_t)(v[2] * 31.5f) << 11)) & 0xffffu;
}
GS_FMT uint32_t enc_quat10(const float v[4]) {
  return (uint32_t)(v[0] * 1023.5f) | ((uint32_t)(v[1] * 1023.5f) << 10) | ((uint32_t)(v[2] * 1023.5f) << 20) |
         ((uint32_t)(v[3] * 3.5f) << 30);
}
GS_FMT uint32_t enc_norm8x4(const float v[4]) {   // Norm8x4 colour, saturated (E/...:661-703)
  return (uint32_t)(saturate(v[0]) * 255.5f) | ((uint32_t)(saturate(v[1]) * 255.5f) << 8) |
         ((uint32_t)(saturate(v[2]) * 255.5f) << 16) | ((uint32_t)(saturate(v[3]) * 255.5f) << 24);
}

// ---- one splat's records (E/...:705-1066) -----------------------------------------------------------------------------
// Stores at 2-byte-aligned addresses: every `other` stride is even but not always a multiple of 4.
GS_FMT void put16(uint8_t *p, uint32_t v) {
#ifdef __CUDA_ARCH__
  *(uint16_t *)p = (uint16_t)v;
#else
  const uint16_t h = (uint16_t)v;
  memcpy(p, &h, 2);
#endif
}
GS_FMT void put32(uint8_t *p, uint32_t v) {
#ifdef __CUDA_ARCH__
  put16(p, v & 0xffffu);
  put16(p + 2, v >> 16);
#else
  memcpy(p, &v, 4);
#endif
}
GS_FMT void put_texel(float *image, size_t texel, const float pix[4]) {   // image: 16-byte aligned float RGBA
#ifdef __CUDA_ARCH__
  reinterpret_cast<float4 *>(image)[texel] = make_float4(pix[0], pix[1], pix[2], pix[3]);
#else
  memcpy(image + texel * 4, pix, 16);
#endif
}

// E/...:727-758
GS_FMT void emit_vector(const float v[3], uint8_t *dst, uint32_t fmt) {
  if (fmt == 0) {
    for (int k = 0; k < 3; ++k) put32(dst + 4 * k, f32_bits(v[k]));
    return;
  }
  const float s[3] = {saturate(v[0]), saturate(v[1]), saturate(v[2])};
  if (fmt == 1) {
    const uint64_t e = enc_norm16(s);
    put32(dst, (uint32_t)e);
    put16(dst + 4, (uint32_t)(e >> 32));
  } else if (fmt == 2) {
    put32(dst, enc_norm11(s));
  } else {
    put16(dst, enc_norm655(s));
  }
}

// Where emit_splat writes: the blobs (zeroed beforehand, so padding stays zero) and, for BC7 colour, the float image the
// blocks are encoded from.  `sh` is not written for clustered SH, whose blob is the palette.
struct EmitTarget {
  uint8_t *pos, *other, *color, *sh;
  float *image;
  uint32_t pf, sf, cf, shf;
};
// Splat i (record `s`, after the Morton reorder and the chunk normalisation): position, the `other` record (rotation
// 10.10.10.2, scale, and for clustered SH its palette index `label`), the colour texel or BC7 image value, the SH item.
GS_FMT void emit_splat(const EmitTarget &t, uint32_t i, const float *s, uint32_t label) {
  emit_vector(s, t.pos + (size_t)i * vec_stride(t.pf), t.pf);
  const uint32_t ostride = other_stride(t.sf, t.shf);
  uint8_t *o = t.other + (size_t)i * ostride;
  put32(o, enc_quat10(s + kOffRot));   // E/...:776-805
  emit_vector(s + kOffScale, o + 4, t.sf);
  if (t.shf > 3) put16(o + ostride - 2, label & 0xffffu);   // E/...:801-803
  // colour, Morton-swizzled (E/...:873-885, 661-703)
  const size_t texel = splat_index_to_texel(i);
  const float pix[4] = {s[kOffDc0], s[kOffDc0 + 1], s[kOffDc0 + 2], s[kOffOpacity]};
  if (t.cf == 3) {
    put_texel(t.image, texel, pix);
  } else if (t.cf == 0) {
    for (int k = 0; k < 4; ++k) put32(t.color + texel * 16 + 4 * k, f32_bits(pix[k]));
  } else if (t.cf == 1) {
    for (int k = 0; k < 4; ++k) put16(t.color + texel * 8 + 2 * k, unity_f32tof16(pix[k]));
  } else {
    put32(t.color + texel * 4, enc_norm8x4(pix));
  }
  // SH table item (E/...:934-1037)
  if (t.shf > 3) return;
  const float *h = s + kOffSh;
  uint8_t *d = t.sh + (size_t)i * sh_stride(t.shf);
  if (t.shf == 0) {
    for (int k = 0; k < 45; ++k) put32(d + 4 * k, f32_bits(h[k]));   // 12 bytes of padding stay zero
  } else if (t.shf == 1) {
    for (int k = 0; k < 45; ++k) put16(d + 2 * k, unity_f32tof16(h[k]));
  } else if (t.shf == 2) {
    for (int j = 0; j < 15; ++j) put32(d + 4 * j, enc_norm11(h + j * 3));   // no saturate in the reference (E/...:990-1008)
  } else {
    for (int j = 0; j < 15; ++j) put16(d + 2 * j, enc_norm565(h + j * 3));
  }
}

// The chunk header (E/...:520-639) from its 13 (min, max) pairs, max already widened to at least min + 1e-5:
// 0..2 position, 3..5 scale, 6..9 colour (dc0 rgb, opacity), 10..12 SH channel
GS_FMT uint32_t f16_pair(float lo, float hi) { return unity_f32tof16(lo) | (unity_f32tof16(hi) << 16); }
GS_FMT ChunkInfo encode_chunk(const float *mn, const float *mx) {
  ChunkInfo c;
  c.posX[0] = mn[0]; c.posX[1] = mx[0];
  c.posY[0] = mn[1]; c.posY[1] = mx[1];
  c.posZ[0] = mn[2]; c.posZ[1] = mx[2];
  c.sclX = f16_pair(mn[3], mx[3]); c.sclY = f16_pair(mn[4], mx[4]); c.sclZ = f16_pair(mn[5], mx[5]);
  c.colR = f16_pair(mn[6], mx[6]); c.colG = f16_pair(mn[7], mx[7]); c.colB = f16_pair(mn[8], mx[8]);
  c.colA = f16_pair(mn[9], mx[9]);
  c.shR = f16_pair(mn[10], mx[10]); c.shG = f16_pair(mn[11], mx[11]); c.shB = f16_pair(mn[12], mx[12]);
  return c;
}

// ---- BC7 -------------------------------------------------------------------------------------------------------------
// One 4x4 block of float RGBA (raster order) -> one BC7 mode-6 block (one subset, 7.7.7.7 endpoints + p-bits, 4-bit
// indices) as two little-endian words.  Endpoints: extremes of the block's pixels (clamped to [0, 1], NaN -> 0) along their
// principal axis (power iteration on the 4x4 covariance), then one least-squares refit against the chosen indices.
struct Bc7Block { uint64_t lo, hi; };
GS_FMT int bc7_weight4(int i) { return (i * 64 + 7) / 15; }   // the 4-bit index weights {0, 4, 9, ..., 60, 64}: round(64 i / 15)
GS_FMT void bc7_put(Bc7Block &b, int &pos, uint32_t v, int n) {
  if (pos < 64) {
    b.lo |= (uint64_t)v << pos;
    if (pos + n > 64) b.hi |= (uint64_t)v >> (64 - pos);
  } else {
    b.hi |= (uint64_t)v << (pos - 64);
  }
  pos += n;
}
GS_FMT Bc7Block bc7_encode_block(const float *rgba) {
  float px[16][4], mean[4] = {0, 0, 0, 0};
  for (int i = 0; i < 16; ++i)
    for (int c = 0; c < 4; ++c) {
      float v = rgba[i * 4 + c];
      v = (v > 0.0f) ? (v < 1.0f ? v : 1.0f) : 0.0f;
      px[i][c] = v * 255.0f;
      mean[c] += px[i][c] * (1.0f / 16.0f);
    }
  float cov[4][4] = {};
  for (int i = 0; i < 16; ++i)
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) cov[r][c] += (px[i][r] - mean[r]) * (px[i][c] - mean[c]);
  float axis[4] = {1.0f, 1.0f, 1.0f, 1.0f};
  for (int it = 0; it < 8; ++it) {
    float nv[4] = {0, 0, 0, 0}, len = 0;
    for (int r = 0; r < 4; ++r) { for (int c = 0; c < 4; ++c) nv[r] += cov[r][c] * axis[c]; len += nv[r] * nv[r]; }
    if (len < 1e-12f) break;
    len = 1.0f / sqrtf(len);
    for (int r = 0; r < 4; ++r) axis[r] = nv[r] * len;
  }
  float tmin = 1e30f, tmax = -1e30f;
  for (int i = 0; i < 16; ++i) {
    float tt = 0;
    for (int c = 0; c < 4; ++c) tt += (px[i][c] - mean[c]) * axis[c];
    tmin = (tt < tmin) ? tt : tmin;
    tmax = (tmax < tt) ? tt : tmax;
  }
  float target[2][4];
  for (int c = 0; c < 4; ++c) { target[0][c] = mean[c] + axis[c] * tmin; target[1][c] = mean[c] + axis[c] * tmax; }
  int ep[2][4], pbit[2] = {0, 0}, idx[16];
  float best_total = 1e30f;
  int best_ep[2][4] = {}, best_p[2] = {0, 0}, best_idx[16] = {};
  for (int round = 0; round < 2; ++round) {
    // each endpoint: 7 bits per channel + one p-bit shared by its channels
    for (int e = 0; e < 2; ++e) {
      float best_err = 1e30f;
      for (int p = 0; p < 2; ++p) {
        int q[4];
        float err = 0;
        for (int c = 0; c < 4; ++c) {
          const float m0 = (0.0f < target[e][c]) ? target[e][c] : 0.0f;   // max(0, target)
          const float tc = (m0 < 255.0f) ? m0 : 255.0f;                     // min(255, .)
          int v = (int)lroundf((tc - (float)p) * 0.5f);
          v = v < 0 ? 0 : (v > 127 ? 127 : v);
          q[c] = (v << 1) | p;
          const float d = (float)q[c] - tc;
          err += d * d;
        }
        if (err < best_err) { best_err = err; pbit[e] = p; for (int c = 0; c < 4; ++c) ep[e][c] = q[c]; }
      }
    }
    int pal[16][4];
    for (int w = 0; w < 16; ++w)
      for (int c = 0; c < 4; ++c) pal[w][c] = ((64 - bc7_weight4(w)) * ep[0][c] + bc7_weight4(w) * ep[1][c] + 32) >> 6;
    float total = 0;
    for (int i = 0; i < 16; ++i) {
      float bst = 1e30f;
      int bi = 0;
      for (int w = 0; w < 16; ++w) {
        float err = 0;
        for (int c = 0; c < 4; ++c) { const float d = (float)pal[w][c] - px[i][c]; err += d * d; }
        if (err < bst) { bst = err; bi = w; }
      }
      idx[i] = bi;
      total += bst;
    }
    if (total < best_total) {
      best_total = total;
      for (int e = 0; e < 2; ++e) { best_p[e] = pbit[e]; for (int c = 0; c < 4; ++c) best_ep[e][c] = ep[e][c]; }
      for (int i = 0; i < 16; ++i) best_idx[i] = idx[i];
    }
    if (round == 1) break;
    // least squares for the two endpoints given the weights w_i = weight(idx_i) / 64: minimise sum |(1-w) A + w B - px|^2
    float saa = 0, sab = 0, sbb = 0, ra[4] = {0, 0, 0, 0}, rb[4] = {0, 0, 0, 0};
    for (int i = 0; i < 16; ++i) {
      const float w = (float)bc7_weight4(idx[i]) * (1.0f / 64.0f), u = 1.0f - w;
      saa += u * u; sab += u * w; sbb += w * w;
      for (int c = 0; c < 4; ++c) { ra[c] += u * px[i][c]; rb[c] += w * px[i][c]; }
    }
    const float det = saa * sbb - sab * sab;
    if (fabsf(det) < 1e-6f) break;
    for (int c = 0; c < 4; ++c) {
      target[0][c] = (ra[c] * sbb - rb[c] * sab) / det;
      target[1][c] = (rb[c] * saa - ra[c] * sab) / det;
    }
  }
  if (best_idx[0] >= 8) {   // the anchor (pixel 0) stores 3 bits: swap the endpoints so that its index has a zero top bit
    for (int c = 0; c < 4; ++c) { const int tmp = best_ep[0][c]; best_ep[0][c] = best_ep[1][c]; best_ep[1][c] = tmp; }
    const int tp = best_p[0]; best_p[0] = best_p[1]; best_p[1] = tp;
    for (int i = 0; i < 16; ++i) best_idx[i] = 15 - best_idx[i];
  }
  Bc7Block b = {0, 0};
  int pos = 0;
  bc7_put(b, pos, 1u << 6, 7);
  for (int c = 0; c < 4; ++c) { bc7_put(b, pos, (uint32_t)best_ep[0][c] >> 1, 7); bc7_put(b, pos, (uint32_t)best_ep[1][c] >> 1, 7); }
  bc7_put(b, pos, (uint32_t)best_p[0], 1); bc7_put(b, pos, (uint32_t)best_p[1], 1);
  bc7_put(b, pos, (uint32_t)best_idx[0], 3);
  for (int i = 1; i < 16; ++i) bc7_put(b, pos, (uint32_t)best_idx[i], 4);
  return b;
}

}  // namespace gs
