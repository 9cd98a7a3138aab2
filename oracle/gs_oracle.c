/* gs_oracle.c -- CPU ORACLE (test infrastructure; see gs_oracle.h for the contract).
 * Pinned against the reference's own shader source compiled for the CPU (oracle/refhlsl/, tests/test_reference_hlsl.py);
 * the reference ships no golden vectors for this path (SURVEY.md 8c).  See gs_oracle.h.
 * Build: gcc -O2 -ffp-contract=off -fopenmp -fPIC -shared (see oracle/Makefile).
 */
#define _GNU_SOURCE
#include "gs_oracle.h"

#include <math.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* ------------------------------------------------------------------ helpers */
static inline uint32_t as_u32(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float as_f32(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline float satf(float v) { return (v > 0.0f) ? ((v < 1.0f) ? v : 1.0f) : 0.0f; } /* NaN -> 0 like HLSL saturate */
static inline float lerpf(float a, float b, float t) { return fmaf(t, b - a, a); }
static inline uint32_t rd_u32(const void *base, uint64_t off) { uint32_t v; memcpy(&v, (const uint8_t *)base + off, 4); return v; }
static inline uint32_t rd_u16(const void *base, uint64_t off) { uint16_t v; memcpy(&v, (const uint8_t *)base + off, 2); return v; }
static inline float rd_f32(const void *base, uint64_t off) { float v; memcpy(&v, (const uint8_t *)base + off, 4); return v; }
#define M_(m, r, c) ((m)[(c) * 4 + (r)])

/* Threads worth using: OpenMP's default, capped by the CPUs this process may really use (affinity mask, cgroup CPU quota --
 * a container can show 128 cores and be allowed 16; oversubscribed OpenMP teams then run several times slower). */
int gso_max_threads(void) {
  long long t = 1;
#ifdef _OPENMP
  t = omp_get_max_threads();
#endif
#ifdef __linux__
  cpu_set_t set;
  if (sched_getaffinity(0, sizeof(set), &set) == 0 && CPU_COUNT(&set) > 0 && CPU_COUNT(&set) < t) t = CPU_COUNT(&set);
  long long quota = -1, period = -1;
  FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r");               /* cgroup v2: "<quota|max> <period>" */
  if (f) {
    char q[32];
    if (fscanf(f, "%31s %lld", q, &period) == 2 && strcmp(q, "max") != 0) quota = atoll(q);
    fclose(f);
  } else {                                                      /* cgroup v1 */
    f = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r");
    if (f) { if (fscanf(f, "%lld", &quota) != 1) quota = -1; fclose(f); }
    f = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r");
    if (f) { if (fscanf(f, "%lld", &period) != 1) period = -1; fclose(f); }
  }
  if (quota > 0 && period > 0 && (quota + period - 1) / period < t) t = (quota + period - 1) / period;
#endif
  return t < 1 ? 1 : (int)t;
}

uint32_t gso_f32tof16(float f) { /* IEEE binary32 -> binary16, round to nearest even */
  uint32_t x = as_u32(f);
  uint32_t sign = (x >> 16) & 0x8000u;
  uint32_t ax = x & 0x7fffffffu;
  if (ax >= 0x7f800000u) return sign | (ax > 0x7f800000u ? 0x7e00u : 0x7c00u);
  if (ax >= 0x477ff000u) return sign | 0x7c00u; /* >= 65520 rounds to inf */
  if (ax < 0x33000001u) return sign;            /* <= 2^-25 rounds to 0 */
  int32_t e = (int32_t)(ax >> 23) - 127;
  uint32_t m = (ax & 0x7fffffu) | 0x800000u;
  uint32_t shift, h;
  if (e < -14) { shift = (uint32_t)(13 + (-14 - e)); h = 0; }          /* subnormal half */
  else { shift = 13; h = (uint32_t)(e + 15) << 10; m &= 0x7fffffu; }
  uint32_t q = m >> shift, rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1);
  h += q;
  if (rem > half || (rem == half && (h & 1u))) h += 1;                  /* carries propagate into the exponent */
  return sign | h;
}

float gso_f16tof32(uint32_t h) {
  h &= 0xffffu;
  uint32_t sign = (h & 0x8000u) << 16, e = (h >> 10) & 31u, m = h & 0x3ffu;
  if (e == 0) {
    if (m == 0) return as_f32(sign);
    float v = (float)m * 5.9604644775390625e-08f; /* m * 2^-24, exact */
    return (sign ? -v : v);
  }
  if (e == 31) return as_f32(sign | 0x7f800000u | (m << 13));
  return as_f32(sign | ((e + 112u) << 23) | (m << 13));
}

float gso_exp_neg(float x) {
  /* exp(x) = 2^(x*log2e); n = rint via 1.5*2^23 magic; 2^f, |f|<=0.5 by a fixed polynomial */
  float t = x * 1.44269502f;
  if (!(t > -125.0f)) t = -125.0f;
  float m = t + 12582912.0f;
  float n = m - 12582912.0f;
  float f = t - n;
  float p = 0.0013276503887027502f;
  p = fmaf(p, f, 0.009675541892647743f);
  p = fmaf(p, f, 0.05550713092088699f);
  p = fmaf(p, f, 0.24022120237350464f);
  p = fmaf(p, f, 0.6931469440460205f);
  p = fmaf(p, f, 1.0000001192092896f);
  int32_t ni = (int32_t)(as_u32(m) - 0x4B400000u);
  return as_f32((uint32_t)((int32_t)as_u32(p) + ni * (1 << 23)));
}

uint32_t gso_float_to_sortable_uint(float f) { /* S/SplatUtilities.compute:52-57 */
  uint32_t fu = as_u32(f);
  uint32_t mask = (uint32_t)(-(int32_t)(fu >> 31)) | 0x80000000u;
  return fu ^ mask;
}

float gso_inv_square_centered01(float x) { /* S/GaussianSplatting.hlsl:5-11 */
  x -= 0.5f;
  x *= 0.5f;
  float s = (x > 0.0f) ? 1.0f : ((x < 0.0f) ? -1.0f : 0.0f);
  x = sqrtf(fabsf(x)) * s;
  return x + 0.5f;
}

static inline void decode_morton2d_16x16(uint32_t t, uint32_t *x, uint32_t *y) { /* :120-127 */
  t = (t & 0xFF) | ((t & 0xFE) << 7);
  t &= 0x5555;
  t = (t ^ (t >> 1)) & 0x3333;
  t = (t ^ (t >> 2)) & 0x0f0f;
  *x = t & 0xF;
  *y = t >> 8;
}

uint32_t gso_splat_index_to_pixel_index(uint32_t idx, uint32_t *px, uint32_t *py) { /* :183-194 */
  uint32_t mx, my;
  decode_morton2d_16x16(idx, &mx, &my);
  uint32_t width = 2048u / 16u;
  idx >>= 8;
  uint32_t x = (idx % width) * 16 + mx, y = (idx / width) * 16 + my;
  if (px) *px = x;
  if (py) *py = y;
  return y * 2048u + x;
}

/* ------------------------------------------------------------------ decoders */
static const float kInv63 = 1.0f / 63.0f, kInv31 = 1.0f / 31.0f, kInv2047 = 1.0f / 2047.0f,
                   kInv1023 = 1.0f / 1023.0f, kInv65535 = 1.0f / 65535.0f, kInv3 = 1.0f / 3.0f;

static inline void dec_6_5_5(uint32_t e, float o[3]) { /* :261-267 */
  o[0] = (float)(e & 63) * kInv63; o[1] = (float)((e >> 6) & 31) * kInv31; o[2] = (float)((e >> 11) & 31) * kInv31;
}
static inline void dec_5_6_5(uint32_t e, float o[3]) { /* :269-275 */
  o[0] = (float)(e & 31) * kInv31; o[1] = (float)((e >> 5) & 63) * kInv63; o[2] = (float)((e >> 11) & 31) * kInv31;
}
static inline void dec_11_10_11(uint32_t e, float o[3]) { /* :277-283 */
  o[0] = (float)(e & 2047) * kInv2047; o[1] = (float)((e >> 11) & 1023) * kInv1023; o[2] = (float)((e >> 21) & 2047) * kInv2047;
}
static inline void dec_16_16_16(uint32_t lo, uint32_t hi, float o[3]) { /* :285-291 */
  o[0] = (float)(lo & 65535) * kInv65535; o[1] = (float)((lo >> 16) & 65535) * kInv65535; o[2] = (float)(hi & 65535) * kInv65535;
}

static inline uint32_t vec_stride(uint32_t fmt) { return fmt == 0 ? 12u : fmt == 1 ? 6u : fmt == 2 ? 4u : 2u; }

/* LoadAndDecodeVector, :346-392 (the 16-bit-straddle shuffles there equal a plain
 * little-endian read at the unaligned byte address) */
static void load_vector(const void *buf, uint64_t addr, uint32_t fmt, float o[3]) {
  if (fmt == 0) { o[0] = rd_f32(buf, addr); o[1] = rd_f32(buf, addr + 4); o[2] = rd_f32(buf, addr + 8); }
  else if (fmt == 1) dec_16_16_16(rd_u32(buf, addr), rd_u16(buf, addr + 4), o);
  else if (fmt == 2) dec_11_10_11(rd_u32(buf, addr), o);
  else dec_6_5_5(rd_u16(buf, addr), o);
}

/* ------------------------------------------------------------------ BC7 (ColorFormat.BC7, R/GaussianSplatAsset.cs:56,169)
 * The reference samples a GraphicsFormat.RGBA_BC7_UNorm texture; the decode is done by the GPU's texture unit, i.e. by the
 * published BC7/BPTC block format (D3D11 functional spec 19.5 / Khronos Data Format "BPTC"), not by code in /root/reference.
 * Whole-block, spec-order restatement; pinned against an independent decoder (Pillow) by tests/golden/bc7_blocks.npz. */
#include "bc7_tables.h"
typedef struct Bc7Mode { uint8_t ns, pb, rb, isb, cb, ab, epb, spb, ib, ib2; } Bc7Mode;
static const Bc7Mode kBc7Modes[8] = {
    {3, 4, 0, 0, 4, 0, 1, 0, 3, 0}, {2, 6, 0, 0, 6, 0, 0, 1, 3, 0}, {3, 6, 0, 0, 5, 0, 0, 0, 2, 0}, {2, 6, 0, 0, 7, 0, 1, 0, 2, 0},
    {1, 0, 2, 1, 5, 6, 0, 0, 2, 3}, {1, 0, 2, 0, 7, 8, 0, 0, 2, 2}, {1, 0, 0, 0, 7, 7, 1, 0, 4, 0}, {2, 6, 0, 0, 5, 5, 1, 0, 2, 0}};
static const uint8_t kBc7W2[4] = {0, 21, 43, 64}, kBc7W3[8] = {0, 9, 18, 27, 37, 46, 55, 64},
                     kBc7W4[16] = {0, 4, 9, 13, 17, 21, 26, 30, 34, 38, 43, 47, 51, 55, 60, 64};
typedef struct Bc7Bits { const uint8_t *b; uint32_t pos; } Bc7Bits;
static uint32_t bc7_get(Bc7Bits *r, uint32_t n) {
  uint32_t v = 0;
  for (uint32_t i = 0; i < n; ++i, ++r->pos) v |= (uint32_t)((r->b[r->pos >> 3] >> (r->pos & 7)) & 1u) << i;
  return v;
}
void gso_bc7_decode_block(const uint8_t block[16], uint8_t out[64]) {
  Bc7Bits r = {block, 0};
  uint32_t mode = 0;
  while (mode < 8 && !bc7_get(&r, 1)) ++mode;
  if (mode == 8) { memset(out, 0, 64); return; } /* reserved: all channels 0 */
  const Bc7Mode m = kBc7Modes[mode];
  const uint32_t part = bc7_get(&r, m.pb), rot = bc7_get(&r, m.rb), isb = bc7_get(&r, m.isb);
  uint32_t ep[6][4];
  const uint32_t ne = m.ns * 2u;
  for (uint32_t ch = 0; ch < 3; ++ch) for (uint32_t e = 0; e < ne; ++e) ep[e][ch] = bc7_get(&r, m.cb);
  for (uint32_t e = 0; e < ne; ++e) ep[e][3] = m.ab ? bc7_get(&r, m.ab) : 0;
  uint32_t cb = m.cb, ab = m.ab;
  if (m.epb) {
    for (uint32_t e = 0; e < ne; ++e) { uint32_t p = bc7_get(&r, 1); for (uint32_t ch = 0; ch < (m.ab ? 4u : 3u); ++ch) ep[e][ch] = (ep[e][ch] << 1) | p; }
    cb += 1; if (m.ab) ab += 1;
  }
  if (m.spb) {
    for (uint32_t s = 0; s < m.ns; ++s) { uint32_t p = bc7_get(&r, 1); for (uint32_t e = 2 * s; e < 2 * s + 2; ++e) for (uint32_t ch = 0; ch < 3; ++ch) ep[e][ch] = (ep[e][ch] << 1) | p; }
    cb += 1;
  }
  for (uint32_t e = 0; e < ne; ++e) {
    for (uint32_t ch = 0; ch < 3; ++ch) { uint32_t x = ep[e][ch] << (8 - cb); ep[e][ch] = x | (x >> cb); }
    if (m.ab) { uint32_t x = ep[e][3] << (8 - ab); ep[e][3] = x | (x >> ab); } else ep[e][3] = 255;
  }
  uint32_t subset[16], anchor[3] = {0, 0, 0};
  for (uint32_t i = 0; i < 16; ++i) subset[i] = m.ns == 1 ? 0u : m.ns == 2 ? ((kBc7Part2[part] >> i) & 1u) : ((kBc7Part3[part] >> (2 * i)) & 3u);
  if (m.ns == 2) anchor[1] = kBc7Anchor2[part];
  if (m.ns == 3) { anchor[1] = kBc7Anchor3a[part]; anchor[2] = kBc7Anchor3b[part]; }
  uint32_t idx1[16], idx2[16];
  for (uint32_t i = 0; i < 16; ++i) idx1[i] = bc7_get(&r, (i == anchor[subset[i]]) ? m.ib - 1u : m.ib);
  for (uint32_t i = 0; i < 16; ++i) idx2[i] = m.ib2 ? bc7_get(&r, i == 0 ? m.ib2 - 1u : m.ib2) : 0;
  for (uint32_t i = 0; i < 16; ++i) {
    const uint32_t *e0 = ep[2 * subset[i]], *e1 = ep[2 * subset[i] + 1];
    uint32_t ci = idx1[i], cbits = m.ib, ai = idx1[i], abits = m.ib;
    if (m.ib2) { if (!isb) { ai = idx2[i]; abits = m.ib2; } else { ci = idx2[i]; cbits = m.ib2; } }
    const uint32_t wc = cbits == 2 ? kBc7W2[ci] : cbits == 3 ? kBc7W3[ci] : kBc7W4[ci];
    const uint32_t wa = abits == 2 ? kBc7W2[ai] : abits == 3 ? kBc7W3[ai] : kBc7W4[ai];
    uint32_t px[4];
    for (uint32_t ch = 0; ch < 3; ++ch) px[ch] = ((64 - wc) * e0[ch] + wc * e1[ch] + 32) >> 6;
    px[3] = ((64 - wa) * e0[3] + wa * e1[3] + 32) >> 6;
    if (rot) { uint32_t t = px[rot - 1]; px[rot - 1] = px[3]; px[3] = t; }
    for (uint32_t ch = 0; ch < 4; ++ch) out[i * 4 + ch] = (uint8_t)px[ch];
  }
}

typedef struct Chunk { /* SplatChunkInfo, :196-202 */
  uint32_t colR, colG, colB, colA;
  float posX[2], posY[2], posZ[2];
  uint32_t sclX, sclY, sclZ;
  uint32_t shR, shG, shB;
} Chunk;

static inline uint32_t chunk_count(const GsoAsset *a) { return a->chunks ? (uint32_t)(a->chunk_bytes / 64) : 0u; }

void gso_load_splat_pos(const GsoAsset *a, uint32_t idx, float pos[3]) { /* LoadSplatPos :409-421 */
  load_vector(a->pos, (uint64_t)idx * vec_stride(a->pos_format), a->pos_format, pos);
  uint32_t ci = idx / 256u;
  if (ci < chunk_count(a)) {
    const Chunk *c = (const Chunk *)a->chunks + ci;
    pos[0] = lerpf(c->posX[0], c->posX[1], pos[0]);
    pos[1] = lerpf(c->posY[0], c->posY[1], pos[1]);
    pos[2] = lerpf(c->posZ[0], c->posZ[1], pos[2]);
  }
}

void gso_load_splat_data(const GsoAsset *a, uint32_t idx, GsoSplat *s) { /* LoadSplatData :428-608 */
  memset(s, 0, sizeof(*s));
  const uint32_t scaleFmt = a->scale_format, shFmt = a->sh_format;
  uint32_t otherStride = 4 + vec_stride(scaleFmt);
  if (shFmt > 3) otherStride += 2;
  uint64_t otherAddr = (uint64_t)idx * otherStride;
  uint32_t shStride = shFmt == 0 ? 192u : (shFmt == 1 || shFmt > 3) ? 96u : shFmt == 2 ? 60u : 32u;

  load_vector(a->pos, (uint64_t)idx * vec_stride(a->pos_format), a->pos_format, s->pos);
  /* DecodeRotation(DecodePacked_10_10_10_2(..)), :219-229, :293-300 */
  {
    uint32_t e = rd_u32(a->other, otherAddr);
    float px = (float)(e & 1023) * kInv1023, py = (float)((e >> 10) & 1023) * kInv1023, pz = (float)((e >> 20) & 1023) * kInv1023;
    float pw = (float)((e >> 30) & 3) * kInv3;
    uint32_t qi = (uint32_t)roundf(pw * 3.0f);
    const float kSqrt2 = 1.41421354f, kInvSqrt2 = 0.707106769f;
    float x = fmaf(px, kSqrt2, -kInvSqrt2), y = fmaf(py, kSqrt2, -kInvSqrt2), z = fmaf(pz, kSqrt2, -kInvSqrt2);
    float w = sqrtf(1.0f - satf(fmaf(z, z, fmaf(y, y, x * x))));
    float q[4] = {x, y, z, w};
    if (qi == 0) { q[0] = w; q[1] = x; q[2] = y; q[3] = z; }      /* q.wxyz */
    if (qi == 1) { q[0] = x; q[1] = w; q[2] = y; q[3] = z; }      /* q.xwyz */
    if (qi == 2) { q[0] = x; q[1] = y; q[2] = w; q[3] = z; }      /* q.xywz */
    memcpy(s->rot, q, 16);
  }
  load_vector(a->other, otherAddr + 4, scaleFmt, s->scale);
  /* LoadSplatColTex(SplatIndexToPixelIndex(idx)) :423-426; the texture unit converts to float */
  float col[4];
  {
    uint64_t ti = gso_splat_index_to_pixel_index(idx, 0, 0);
    if (a->color_format == 0) { for (int k = 0; k < 4; ++k) col[k] = rd_f32(a->color, ti * 16 + 4 * k); }
    else if (a->color_format == 1) { for (int k = 0; k < 4; ++k) col[k] = gso_f16tof32(rd_u16(a->color, ti * 8 + 2 * k)); }
    else if (a->color_format == 2) { uint32_t e = rd_u32(a->color, ti * 4); for (int k = 0; k < 4; ++k) col[k] = (float)((e >> (8 * k)) & 255u) / 255.0f; }
    else { /* BC7: 4x4 blocks of 16 bytes, row-major over the 2048-wide image; UNORM8 result / 255 */
      uint32_t x, y; uint8_t px[64];
      gso_splat_index_to_pixel_index(idx, &x, &y);
      gso_bc7_decode_block((const uint8_t *)a->color + ((uint64_t)(y >> 2) * (2048u / 4u) + (x >> 2)) * 16u, px);
      for (int k = 0; k < 4; ++k) col[k] = (float)px[((y & 3u) * 4u + (x & 3u)) * 4u + k] / 255.0f;
    }
  }
  uint32_t shIndex = idx;
  if (shFmt > 3) shIndex = rd_u16(a->other, otherAddr + otherStride - 2);
  uint64_t shOff = (uint64_t)shIndex * shStride;
  for (int j = 0; j < 15; ++j) {
    float *d = &s->sh[j * 3];
    if (shFmt == 0) { for (int k = 0; k < 3; ++k) d[k] = rd_f32(a->sh, shOff + (uint64_t)(j * 3 + k) * 4); }
    else if (shFmt == 1 || shFmt > 3) { for (int k = 0; k < 3; ++k) d[k] = gso_f16tof32(rd_u16(a->sh, shOff + (uint64_t)(j * 3 + k) * 2)); }
    else if (shFmt == 2) dec_11_10_11(rd_u32(a->sh, shOff + (uint64_t)j * 4), d);
    else dec_5_6_5(rd_u16(a->sh, shOff + (uint64_t)j * 2), d);
  }
  uint32_t ci = idx / 256u;
  if (ci < chunk_count(a)) { /* :565-603 */
    const Chunk *c = (const Chunk *)a->chunks + ci;
    s->pos[0] = lerpf(c->posX[0], c->posX[1], s->pos[0]);
    s->pos[1] = lerpf(c->posY[0], c->posY[1], s->pos[1]);
    s->pos[2] = lerpf(c->posZ[0], c->posZ[1], s->pos[2]);
    const uint32_t sc[3] = {c->sclX, c->sclY, c->sclZ};
    for (int k = 0; k < 3; ++k) {
      float v = lerpf(gso_f16tof32(sc[k]), gso_f16tof32(sc[k] >> 16), s->scale[k]);
      v *= v; v *= v; v *= v;
      s->scale[k] = v;
    }
    const uint32_t cc[4] = {c->colR, c->colG, c->colB, c->colA};
    for (int k = 0; k < 4; ++k) col[k] = lerpf(gso_f16tof32(cc[k]), gso_f16tof32(cc[k] >> 16), col[k]);
    col[3] = gso_inv_square_centered01(col[3]);
    if (shFmt > 0 && shFmt <= 3) {
      const uint32_t hc[3] = {c->shR, c->shG, c->shB};
      for (int j = 0; j < 15; ++j)
        for (int k = 0; k < 3; ++k)
          s->sh[j * 3 + k] = lerpf(gso_f16tof32(hc[k]), gso_f16tof32(hc[k] >> 16), s->sh[j * 3 + k]);
    }
  }
  s->opacity = col[3];
  s->col[0] = col[0]; s->col[1] = col[1]; s->col[2] = col[2];
}

/* ------------------------------------------------------------------ host-side uniforms */
/* Matrix4x4 operator* as Unity evaluates it: out(r,c) = sum_k a(r,k)*b(k,c), plain float ops. */
static void mat_mul(const float *a, const float *b, float *o) {
  for (int c = 0; c < 4; ++c)
    for (int r = 0; r < 4; ++r)
      M_(o, r, c) = M_(a, r, 0) * M_(b, 0, c) + M_(a, r, 1) * M_(b, 1, c) + M_(a, r, 2) * M_(b, 2, c) + M_(a, r, 3) * M_(b, 3, c);
}
static inline float xf_row(const float *m, int r, const float p[3]) {
  return fmaf(M_(m, r, 2), p[2], fmaf(M_(m, r, 1), p[1], fmaf(M_(m, r, 0), p[0], M_(m, r, 3))));
}

void gso_set_indices(uint32_t *order, uint32_t n) { for (uint32_t i = 0; i < n; ++i) order[i] = i; }

void gso_calc_distances(const GsoAsset *a, const GsoFrame *f, const uint32_t *order, uint32_t *keys, int threads) {
  /* SortPoints: worldToCamera with row 2 negated, times localToWorld (R/GaussianSplatRenderer.cs:617-629) */
  float w2c[16], mv[16];
  memcpy(w2c, f->mat_view, 64);
  M_(w2c, 2, 0) *= -1.0f; M_(w2c, 2, 1) *= -1.0f; M_(w2c, 2, 2) *= -1.0f;
  mat_mul(w2c, f->mat_object_to_world, mv);
  if (threads < 1) threads = 1;
#pragma omp parallel for schedule(static) num_threads(threads)
  for (int64_t i = 0; i < (int64_t)a->splat_count; ++i) {
    float p[3];
    gso_load_splat_pos(a, order[i], p);
    keys[i] = gso_float_to_sortable_uint(xf_row(mv, 2, p));
  }
}

/* ------------------------------------------------------------------ sort */
void gso_sort_pairs(uint32_t *keys, uint32_t *payload, uint32_t n, int threads) {
  if (n == 0) return;
  if (threads < 1) threads = 1;
  if ((uint32_t)threads > n) threads = 1;
  uint32_t *k2 = (uint32_t *)malloc((size_t)n * 4), *p2 = (uint32_t *)malloc((size_t)n * 4);
  uint32_t *hist = (uint32_t *)malloc((size_t)threads * 256 * 4);
  uint32_t *src_k = keys, *src_p = payload, *dst_k = k2, *dst_p = p2;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = pass * 8;
    memset(hist, 0, (size_t)threads * 256 * 4);
#pragma omp parallel num_threads(threads)
    {
#ifdef _OPENMP
      int t = omp_get_thread_num(), T = omp_get_num_threads();
#else
      int t = 0, T = 1;
#endif
      uint64_t b = (uint64_t)n * t / T, e = (uint64_t)n * (t + 1) / T;
      uint32_t *h = hist + (size_t)t * 256;
      for (uint64_t i = b; i < e; ++i) h[(src_k[i] >> shift) & 255u]++;
#pragma omp barrier
#pragma omp single
      {
        uint32_t sum = 0;
        for (int d = 0; d < 256; ++d)
          for (int tt = 0; tt < T; ++tt) { uint32_t c = hist[(size_t)tt * 256 + d]; hist[(size_t)tt * 256 + d] = sum; sum += c; }
      }
      for (uint64_t i = b; i < e; ++i) {
        uint32_t d = (src_k[i] >> shift) & 255u, o = h[d]++;
        dst_k[o] = src_k[i]; dst_p[o] = src_p[i];
      }
    }
    uint32_t *tk = src_k; src_k = dst_k; dst_k = tk;
    uint32_t *tp = src_p; src_p = dst_p; dst_p = tp;
  }
  /* 4 passes: result is back in keys/payload (R/GpuSorting.cs:195-196) */
  free(k2); free(p2); free(hist);
}

/* ------------------------------------------------------------------ view calc */
static int is_splat_cut(const GsoFrame *f, const float pos[3]) { /* S/SplatUtilities.compute:164-187 */
  int finalCut = 0;
  for (uint32_t i = 0; i < f->cutout_count; ++i) {
    const GsoCutout *c = &f->cutouts[i];
    uint32_t type = c->type_and_flags & 0xFFu;
    if (type == 0xFFu) continue;
    int invert = (c->type_and_flags & 0xFF00u) != 0;
    float cp[3] = {xf_row(c->mat, 0, pos), xf_row(c->mat, 1, pos), xf_row(c->mat, 2, pos)};
    if (type == 0) { if (cp[0] * cp[0] + cp[1] * cp[1] + cp[2] * cp[2] <= 1.0f) return invert; }
    if (type == 1) { if (fabsf(cp[0]) <= 1.0f && fabsf(cp[1]) <= 1.0f && fabsf(cp[2]) <= 1.0f) return invert; }
    finalCut |= !invert;
  }
  return finalCut;
}

static const float SH_C1 = 0.4886025f;
static const float SH_C2[5] = {1.0925484f, -1.0925484f, 0.3153916f, -1.0925484f, 0.5462742f};
static const float SH_C3[7] = {-0.5900436f, 2.8906114f, -0.4570458f, 0.3731763f, -0.4570458f, 1.4453057f, -0.5900436f};

/* ShadeSH, S/GaussianSplatting.hlsl:139-179 (half == float32 on this path) */
static void shade_sh(const GsoSplat *s, const float dir_in[3], uint32_t shOrder, int onlySH, float res[3]) {
  float x = dir_in[0] * -1.0f, y = dir_in[1] * -1.0f, z = dir_in[2] * -1.0f;
  const float *sh = s->sh;
#define SH(j, k) sh[((j)-1) * 3 + (k)]
  for (int k = 0; k < 3; ++k) {
    float r = onlySH ? 0.5f : s->col[k];
    if (shOrder >= 1) {
      r += SH_C1 * (-SH(1, k) * y + SH(2, k) * z - SH(3, k) * x);
      if (shOrder >= 2) {
        float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
        r += (SH_C2[0] * xy) * SH(4, k) + (SH_C2[1] * yz) * SH(5, k) + (SH_C2[2] * (2.0f * zz - xx - yy)) * SH(6, k) +
             (SH_C2[3] * xz) * SH(7, k) + (SH_C2[4] * (xx - yy)) * SH(8, k);
        if (shOrder >= 3) {
          r += (SH_C3[0] * y * (3.0f * xx - yy)) * SH(9, k) + (SH_C3[1] * xy * z) * SH(10, k) +
               (SH_C3[2] * y * (4.0f * zz - xx - yy)) * SH(11, k) + (SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy)) * SH(12, k) +
               (SH_C3[4] * x * (4.0f * zz - xx - yy)) * SH(13, k) + (SH_C3[5] * z * (xx - yy)) * SH(14, k) +
               (SH_C3[6] * x * (xx - 3.0f * yy)) * SH(15, k);
        }
      }
    }
    res[k] = (r > 0.0f) ? r : 0.0f; /* max(res, 0); NaN -> 0 */
  }
#undef SH
}

/* CSExportData, S/SplatUtilities.compute:616-669 with _ExportTransformFlags == 0: LoadSplatData -> ExportSplatData
 * (= InputSplatData, 62 floats: pos, nor, dc0, sh R/G/B channel-major, opacity, scale, rot wxyz).  log() is libm's here and
 * the GPU's there: compared with a tolerance, the one place on this path where that is so. */
void gso_export_data(const GsoAsset *a, const GsoFrame *f, float *out, int threads) {
  (void)threads;
#pragma omp parallel for schedule(static) num_threads(threads > 0 ? threads : 1)
  for (int64_t ii = 0; ii < (int64_t)a->splat_count; ++ii) {
    GsoSplat s;
    gso_load_splat_data(a, (uint32_t)ii, &s);
    const int cut = f ? is_splat_cut(f, s.pos) : 0;
    float *d = out + (size_t)ii * 62;
    memcpy(d, s.pos, 12);
    d[3] = d[4] = d[5] = cut ? 1.0f : 0.0f;
    for (int k = 0; k < 3; ++k) d[6 + k] = (s.col[k] - 0.5f) / 0.2820948f;         /* ColorToSH0 :537-540 */
    for (int ch = 0; ch < 3; ++ch)
      for (int j = 0; j < 15; ++j) d[9 + ch * 15 + j] = s.sh[j * 3 + ch];
    d[54] = logf(s.opacity / fmaxf(1.0f - s.opacity, 1.0e-6f));                  /* InvSigmoid :541-544 */
    for (int k = 0; k < 3; ++k) d[55 + k] = logf(s.scale[k]);
    d[58] = s.rot[3]; d[59] = s.rot[0]; d[60] = s.rot[1]; d[61] = s.rot[2];        /* rot.wxyz */
  }
}

void gso_calc_view(const GsoAsset *a, const GsoFrame *f, GsoView *view, int threads) {
  /* uniforms, R/GaussianSplatRenderer.cs:586-606 */
  float mv[16], vp[16];
  mat_mul(f->mat_view, f->mat_object_to_world, mv);
  mat_mul(f->mat_proj_gpu, f->mat_view, vp); /* UNITY_MATRIX_VP */
  const float *P = f->mat_proj_gpu;
  const float p00 = M_(P, 0, 0), p11 = M_(P, 1, 1);
  /* CalcCovariance2D constants, S/GaussianSplatting.hlsl:62-70 (tanFovY == tanFovX: reference quirk) */
  const float aspect = p00 / p11;
  const float tanFovX = 1.0f / p00;
  const float tanFovY = 1.0f / (p11 * aspect);
  const float limX = 1.3f * tanFovX, limY = 1.3f * tanFovY;
  const float focal = f->screen_w * p00 / 2.0f;
  const float splatScale2 = f->splat_scale * f->splat_scale;
  if (threads < 1) threads = 1;
#pragma omp parallel for schedule(static) num_threads(threads)
  for (int64_t ii = 0; ii < (int64_t)a->splat_count; ++ii) {
    uint32_t idx = (uint32_t)ii;
    GsoSplat s;
    gso_load_splat_data(a, idx, &s);
    GsoView v;
    memset(&v, 0, sizeof(v));
    const float *o2w = f->mat_object_to_world;
    float cw[3] = {xf_row(o2w, 0, s.pos), xf_row(o2w, 1, s.pos), xf_row(o2w, 2, s.pos)};
    float clip[4] = {xf_row(vp, 0, cw), xf_row(vp, 1, cw), xf_row(vp, 2, cw), xf_row(vp, 3, cw)};
    if (f->deleted_bits) { /* :205-214 */
      if (f->deleted_bits[idx / 32] & (1u << (idx & 31))) clip[3] = 0.0f;
    }
    if (is_splat_cut(f, s.pos)) clip[3] = 0.0f; /* :217-220 */
    memcpy(v.pos, clip, 16);
    int behindCam = clip[3] <= 0.0f;
    if (!behindCam) {
      /* CalcMatrixFromRotationScale :29-46 */
      float x = s.rot[0], y = s.rot[1], z = s.rot[2], w = s.rot[3];
      float mr[3][3] = {{1.0f - 2.0f * (y * y + z * z), 2.0f * (x * y - w * z), 2.0f * (x * z + w * y)},
                        {2.0f * (x * y + w * z), 1.0f - 2.0f * (x * x + z * z), 2.0f * (y * z - w * x)},
                        {2.0f * (x * z - w * y), 2.0f * (y * z + w * x), 1.0f - 2.0f * (x * x + y * y)}};
      float m[3][3];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) m[r][c] = mr[r][c] * s.scale[c];
      /* CalcCovariance3D :48-53, scaled by splatScale^2 (S/SplatUtilities.compute:233-235) */
      float sig[3][3];
      for (int r = 0; r < 3; ++r)
        for (int c = r; c < 3; ++c) sig[r][c] = sig[c][r] = (m[r][0] * m[c][0] + m[r][1] * m[c][1] + m[r][2] * m[c][2]) * splatScale2;
      /* CalcCovariance2D :56-90 */
      float vpz[3] = {xf_row(mv, 0, s.pos), xf_row(mv, 1, s.pos), xf_row(mv, 2, s.pos)};
      float tz = vpz[2];
      float cx = vpz[0] / tz, cy = vpz[1] / tz;
      cx = fminf(fmaxf(cx, -limX), limX); cy = fminf(fmaxf(cy, -limY), limY);
      float tx = cx * tz, ty = cy * tz;
      float j00 = focal / tz, j02 = -(focal * tx) / (tz * tz), j12 = -(focal * ty) / (tz * tz);
      float T[2][3];
      for (int c = 0; c < 3; ++c) {
        T[0][c] = j00 * M_(mv, 0, c) + j02 * M_(mv, 2, c);
        T[1][c] = j00 * M_(mv, 1, c) + j12 * M_(mv, 2, c);
      }
      float vt[3][2]; /* V * T^T */
      for (int k = 0; k < 3; ++k)
        for (int i = 0; i < 2; ++i) vt[k][i] = sig[k][0] * T[i][0] + sig[k][1] * T[i][1] + sig[k][2] * T[i][2];
      float cov00 = T[0][0] * vt[0][0] + T[0][1] * vt[1][0] + T[0][2] * vt[2][0];
      float cov01 = T[0][0] * vt[0][1] + T[0][1] * vt[1][1] + T[0][2] * vt[2][1];
      float cov11 = T[1][0] * vt[0][1] + T[1][1] * vt[1][1] + T[1][2] * vt[2][1];
      cov00 += 0.3f; cov11 += 0.3f;
      /* DecomposeCovariance, S/SplatUtilities.compute:149-159 */
      float mid = 0.5f * (cov00 + cov11);
      float hd = (cov00 - cov11) * 0.5f;
      float radius = sqrtf(hd * hd + cov01 * cov01);
      float lambda1 = mid + radius;
      float lambda2 = fmaxf(mid - radius, 0.1f);
      float dvx = cov01, dvy = lambda1 - cov00;
      float dl = sqrtf(dvx * dvx + dvy * dvy);
      dvx = dvx / dl; dvy = dvy / dl; /* normalize; (0,0) -> NaN exactly like 0*rsqrt(0) */
      dvy = -dvy;
      float l1 = fminf(sqrtf(2.0f * lambda1), 4096.0f), l2 = fminf(sqrtf(2.0f * lambda2), 4096.0f);
      v.axis1[0] = l1 * dvx; v.axis1[1] = l1 * dvy;
      v.axis2[0] = l2 * dvy; v.axis2[1] = l2 * -dvx;
      /* colour :240-248 */
      float wvd[3] = {f->cam_pos_world[0] - cw[0], f->cam_pos_world[1] - cw[1], f->cam_pos_world[2] - cw[2]};
      const float *w2o = f->mat_world_to_object;
      float od[3];
      for (int r = 0; r < 3; ++r) od[r] = fmaf(M_(w2o, r, 2), wvd[2], fmaf(M_(w2o, r, 1), wvd[1], M_(w2o, r, 0) * wvd[0]));
      float ol = sqrtf(od[0] * od[0] + od[1] * od[1] + od[2] * od[2]);
      od[0] = od[0] / ol; od[1] = od[1] / ol; od[2] = od[2] / ol;
      float rgb[3];
      shade_sh(&s, od, f->sh_order, f->sh_only != 0, rgb);
      float alpha = fminf(s.opacity * f->opacity_scale, 65000.0f);
      v.color[0] = (gso_f32tof16(rgb[0]) << 16) | gso_f32tof16(rgb[1]);
      v.color[1] = (gso_f32tof16(rgb[2]) << 16) | gso_f32tof16(alpha);
    }
    view[idx] = v;
  }
}

/* ------------------------------------------------------------------ draw + blend */
static inline float round_h(float v) { return gso_f16tof32(gso_f32tof16(v)); }
/* A blend that yields NaN (a NaN or inf in the loaded target, or inf * 0) stores the GPU's canonical NaN 0x7FFFFFFF whatever the
   operands' payloads: float arithmetic returns it, and the fp16 ROP's half NaN 0x7FFF widens to it. */
static inline float canonical_nan(float v) { return v == v ? v : as_f32(0x7fffffffu); }

/* band t covers rows [H*t/bands, H*(t+1)/bands): the band of row y is the largest t with H*t/bands <= y */
static inline int band_of_row(int32_t y, int bands, uint32_t H) {
  int t = (int)(((uint64_t)y * (uint64_t)bands) / H);
  while (t + 1 < bands && (int32_t)((uint64_t)H * (uint64_t)(t + 1) / (uint64_t)bands) <= y) ++t;
  while (t > 0 && (int32_t)((uint64_t)H * (uint64_t)t / (uint64_t)bands) > y) --t;
  return t;
}

typedef struct DrawRec { /* per-splat constants of the draw, computed once (phase 1) */
  float cx, cy, i1x, i1y, i2x, i2y, cr, cg, cb, ca;
  float z;                /* depth of every fragment of the (flat) quad: clip.z / clip.w */
  int32_t x0, x1, y0, y1; /* pixel rectangle to visit; x0 >= x1 marks "nothing to draw" */
} DrawRec;

void gso_render(const GsoView *view, const uint32_t *order, uint32_t n, uint32_t W, uint32_t H, uint32_t blend_mode,
                float *rt, int threads) {
  gso_render_sel(view, order, n, W, H, blend_mode, rt, threads, NULL);
}

void gso_render_sel(const GsoView *view, const uint32_t *order, uint32_t n, uint32_t W, uint32_t H, uint32_t blend_mode,
                    float *rt, int threads, const uint32_t *selected_bits) {
  gso_render_ex(view, order, n, W, H, blend_mode, rt, threads, selected_bits, NULL, 0);
}

void gso_render_ex(const GsoView *view, const uint32_t *order, uint32_t n, uint32_t W, uint32_t H, uint32_t blend_mode,
                   float *rt, int threads, const uint32_t *selected_bits, const float *scene_depth, int load) {
  if (!load) memset(rt, 0, (size_t)W * H * 16); /* ClearRenderTarget(0,0,0,0), R/GaussianSplatRenderer.cs:196 */
  if (threads < 1) threads = 1;
  const float fW = (float)W, fH = (float)H;
  DrawRec *recs = (DrawRec *)malloc((size_t)(n ? n : 1) * sizeof(DrawRec));
  /* phase 1: the vertex-shader part, one record per splat in draw order (instID = _OrderBuffer[instID], :38-39) */
#pragma omp parallel for schedule(static) num_threads(threads)
  for (int64_t k = 0; k < (int64_t)n; ++k) {
    const GsoView *v = &view[order[k]];
    DrawRec *r = &recs[k];
    r->x0 = 0; r->x1 = 0; r->y0 = 0; r->y1 = 0;
    if (!(v->pos[3] > 0.0f)) continue;            /* behindCam -> NaN vertex -> primitive dropped, :41-45 */
    float a1x = v->axis1[0], a1y = v->axis1[1], a2x = v->axis2[0], a2y = v->axis2[1];
    float cr = gso_f16tof32(v->color[0] >> 16), cg = gso_f16tof32(v->color[0]), cb = gso_f16tof32(v->color[1] >> 16),
          ca = gso_f16tof32(v->color[1]);          /* :48-51 */
    if (!(ca >= 0.0f)) continue;                   /* never produced by CSCalcViewData (opacity >= 0); NaN draws nothing */
    if (selected_bits && (selected_bits[order[k] >> 5] & (1u << (order[k] & 31)))) ca = -1.0f; /* :63-73: o.col.a = -1 */
    /* centre in pixels: D3D viewport transform of clip.xy / clip.w */
    float ndx = v->pos[0] / v->pos[3], ndy = v->pos[1] / v->pos[3];
    float cx = fmaf(ndx, 0.5f, 0.5f) * fW, cy = fmaf(ndy, -0.5f, 0.5f) * fH;
    /* the quad spans centre +- 2*axis1 +- 2*axis2 (:54-61); one NDC unit = W/2 (H/2) pixels, y down */
    float ex = 2.0f * (fabsf(a1x) + fabsf(a2x)), ey = 2.0f * (fabsf(a1y) + fabsf(a2y));
    if (!(ex < 1.0e6f) || !(ey < 1.0e6f) || !(fabsf(cx) < 1.0e7f) || !(fabsf(cy) < 1.0e7f)) continue; /* NaN/inf axes: no raster */
    float fx0 = floorf(cx - ex - 1.0f), fx1 = ceilf(cx + ex + 1.0f), fy0 = floorf(cy - ey - 1.0f), fy1 = ceilf(cy + ey + 1.0f);
    int32_t x0 = fx0 < 0.0f ? 0 : (int32_t)fx0, x1 = fx1 > fW ? (int32_t)W : (int32_t)fx1;
    int32_t y0 = fy0 < 0.0f ? 0 : (int32_t)fy0, y1 = fy1 > fH ? (int32_t)H : (int32_t)fy1;
    if (x0 >= x1 || y0 >= y1) continue;
    /* quad coordinates of a pixel: d = qa*axis1 + qb*axis2, axes orthogonal (SURVEY App. B) */
    float n1 = a1x * a1x + a1y * a1y, n2 = a2x * a2x + a2y * a2y;
    r->cx = cx; r->cy = cy;
    r->i1x = a1x / n1; r->i1y = a1y / n1; r->i2x = a2x / n2; r->i2y = a2y / n2;
    r->cr = cr; r->cg = cg; r->cb = cb; r->ca = ca;
    r->z = v->pos[2] / v->pos[3];
    r->x0 = x0; r->x1 = x1; r->y0 = y0; r->y1 = y1;
  }
  /* phase 2: rasterise + blend.  The image is cut into bands of rows; every band visits, in draw order, the records whose
     rows reach into it (a per-band index list built by a counting pass), so the result depends neither on the thread count
     nor on the band count, and no band walks records that cannot touch it. */
  int bands = threads * 4;
  if ((uint32_t)bands > H) bands = (int)H;
  if (bands < 1) bands = 1;
  uint64_t *band_start = (uint64_t *)calloc((size_t)bands + 1, sizeof(uint64_t));
  for (uint32_t k = 0; k < n; ++k) {
    const DrawRec *r = &recs[k];
    if (r->x0 >= r->x1) continue;
    int t0, t1;
    t0 = band_of_row(r->y0, bands, H);
    t1 = band_of_row(r->y1 - 1, bands, H);
    for (int t = t0; t <= t1; ++t) band_start[t + 1]++;
  }
  for (int t = 0; t < bands; ++t) band_start[t + 1] += band_start[t];
  uint32_t *band_list = (uint32_t *)malloc((size_t)(band_start[bands] ? band_start[bands] : 1) * sizeof(uint32_t));
  uint64_t *fill = (uint64_t *)malloc((size_t)bands * sizeof(uint64_t));
  for (int t = 0; t < bands; ++t) fill[t] = band_start[t];
  for (uint32_t k = 0; k < n; ++k) {            /* in draw order, so every band's list is in draw order */
    const DrawRec *r = &recs[k];
    if (r->x0 >= r->x1) continue;
    int t0, t1;
    t0 = band_of_row(r->y0, bands, H);
    t1 = band_of_row(r->y1 - 1, bands, H);
    for (int t = t0; t <= t1; ++t) band_list[fill[t]++] = k;
  }
  free(fill);
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (int t = 0; t < bands; ++t) {
    const int32_t row0 = (int32_t)((uint64_t)H * t / bands), row1 = (int32_t)((uint64_t)H * (t + 1) / bands);
    for (uint64_t e = band_start[t]; e < band_start[t + 1]; ++e) {
      const DrawRec *r = &recs[band_list[e]];
      const int32_t y0 = r->y0 < row0 ? row0 : r->y0, y1 = r->y1 > row1 ? row1 : r->y1;
      if (y0 >= y1) continue;
      const float cx = r->cx, cy = r->cy, i1x = r->i1x, i1y = r->i1y, i2x = r->i2x, i2y = r->i2y;
      const float cr = r->cr, cg = r->cg, cb = r->cb, ca = r->ca;
      for (int32_t py = y0; py < y1; ++py) {
        float dy = cy - ((float)py + 0.5f); /* pixel y grows downwards, NDC y upwards */
        for (int32_t px = r->x0; px < r->x1; ++px) {
          float dx = ((float)px + 0.5f) - cx;
          float qa = fmaf(dy, i1y, dx * i1x), qb = fmaf(dy, i2y, dx * i2x);
          if (!(fabsf(qa) <= 2.0f && fabsf(qb) <= 2.0f)) continue; /* outside the quad */
          float power = -fmaf(qb, qb, qa * qa);     /* -dot(i.pos, i.pos), :81 */
          float alpha = gso_exp_neg(power);         /* half alpha = exp(power), :82 */
          float pr = cr, pg = cg, pb = cb;
          if (ca >= 0.0f) {
            alpha = satf(alpha * ca);               /* :83-86 */
          } else {                                  /* "selected" splat: magenta outline, more opacity, magenta tint, :87-101 */
            if (alpha > 7.0f / 255.0f) {
              if (alpha < 10.0f / 255.0f) { alpha = 1.0f; pr = 1.0f; pg = 0.0f; pb = 1.0f; }
              alpha = satf(alpha + 0.3f);
            }
            pr = lerpf(pr, 1.0f, 0.5f); pg = lerpf(pg, 0.0f, 0.5f); pb = lerpf(pb, 1.0f, 0.5f);
          }
          if (alpha < 0.003921569f) continue;       /* discard, :103-104 */
          if (scene_depth && !(r->z >= scene_depth[(size_t)py * W + px])) continue; /* ZTest LEqual under reversed Z */
          float *d = &rt[((size_t)py * W + px) * 4];
          /* a zero blend factor contributes nothing (the D3D convention, as in gso_composite): a pixel with dst.a == 1
             ignores every later splat, even one whose colour is inf (inf * 0 would be NaN) */
          if (d[3] == 1.0f) continue;
          float om = 1.0f - d[3];                   /* Blend OneMinusDstAlpha One, :11 */
          float r0 = fmaf(pr * alpha, om, d[0]), r1 = fmaf(pg * alpha, om, d[1]), r2 = fmaf(pb * alpha, om, d[2]),
                r3 = fmaf(alpha, om, d[3]);
          if (blend_mode == 0) { r0 = round_h(r0); r1 = round_h(r1); r2 = round_h(r2); r3 = round_h(r3); }
          d[0] = canonical_nan(r0); d[1] = canonical_nan(r1); d[2] = canonical_nan(r2); d[3] = canonical_nan(r3);
        }
      }
    }
  }
  free(band_list);
  free(band_start);
  free(recs);
}

/* ------------------------------------------------------------------ composite */
static inline float gamma_to_linear(float x) { /* UnityCG.cginc GammaToLinearSpace (Unity 2022.3 built-in shaders; not vendored) */
  return x * fmaf(x, fmaf(x, 0.305306011f, 0.682171111f), 0.012522878f);
}

void gso_composite(const float *rt, float *target, uint32_t W, uint32_t H, int target_fp16) {
  for (size_t i = 0; i < (size_t)W * H; ++i) {
    const float *c = &rt[i * 4];
    float *d = &target[i * 4];
    float a = c[3];
    if (!(a > 0.0f)) continue; /* SrcAlpha == 0: D3D blend treats 0 * (NaN from rgb/0) as 0 -> target unchanged */
    float om = 1.0f - a;
    float o[4];
    for (int k = 0; k < 3; ++k) o[k] = fmaf(gamma_to_linear(c[k] / a), a, d[k] * om);
    o[3] = fmaf(a, a, d[3] * om);
    for (int k = 0; k < 4; ++k) d[k] = target_fp16 ? round_h(o[k]) : o[k];
  }
}
