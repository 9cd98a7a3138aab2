// gs_packed_float.cuh -- the unsigned 11- and 10-bit floats of a GS_PIX_B10G11R11_UFLOAT texel (Unity B10G11R11_UFloatPack32,
// VK_FORMAT_B10G11R11_UFLOAT_PACK32, DXGI_FORMAT_R11G11B10_FLOAT): R in bits 0-10, G in 11-21 (float11: 5 exponent bits, bias
// 15, 6 mantissa bits), B in 22-31 (float10: 5 mantissa bits); no sign, no alpha.  Shared by the composite kernel and the
// codec's own test, so it compiles for the host as well.
//   decode: exact; exponent 0 is a denormal (mantissa * 2^-14 / 2^M), exponent 31 is +Inf (mantissa 0) or a NaN.
//   encode: NaN -> all ones; every value <= 0 (-0 and -Inf included) -> 0; +Inf -> +Inf; anything else rounds to nearest, ties
//           to even, over the whole value set (denormals included), and overflows to +Inf as IEEE rounding does (float11:
//           x >= 65280, float10: x >= 65024).
#pragma once
#include <cstdint>
#include <cstring>

namespace gs {

__host__ __device__ __forceinline__ uint32_t pf_bits(float f) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
#endif
}
__host__ __device__ __forceinline__ float pf_float(uint32_t u) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}

// float32 -> unsigned float of 5 exponent bits and M mantissa bits (M = 6: float11, M = 5: float10)
template <int M>
__host__ __device__ __forceinline__ uint32_t f32_to_ufloat(float f) {
  const uint32_t x = pf_bits(f), inf = 31u << M;
  if ((x & 0x7fffffffu) > 0x7f800000u) return inf | ((1u << M) - 1u);   // NaN
  if ((x >> 31) || x == 0) return 0;                                   // negative, -0, +0
  if (x == 0x7f800000u) return inf;
  const int32_t e = (int32_t)(x >> 23) - 127;   // a float32 denormal (e = -127) lies far below the smallest code
  if (e < -15 - M) return 0;                    // below half the smallest denormal (exactly half is a tie to 0)
  uint32_t m = x & 0x7fffffu, shift, h;
  if (e < -14) { m |= 0x800000u; shift = (uint32_t)(23 - M + (-14 - e)); h = 0; }   // a denormal code
  else { shift = (uint32_t)(23 - M); h = (uint32_t)(e + 15) << M; }
  const uint32_t rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1);
  h += m >> shift;
  if (rem > half || (rem == half && (h & 1u))) h += 1;   // a carry moves into the exponent
  return h >= inf ? inf : h;
}

template <int M>
__host__ __device__ __forceinline__ float ufloat_to_f32(uint32_t c) {
  const uint32_t e = (c >> M) & 31u, m = c & ((1u << M) - 1u);
  if (e == 0) return (float)m * pf_float((uint32_t)(127 - 14 - M) << 23);   // m * 2^(-14-M), exact
  if (e == 31) return pf_float(m ? 0x7fc00000u | (m << (23 - M)) : 0x7f800000u);
  return pf_float(((e + 112u) << 23) | (m << (23 - M)));
}

__host__ __device__ __forceinline__ uint32_t pack_b10g11r11(float r, float g, float b) {
  return f32_to_ufloat<6>(r) | (f32_to_ufloat<6>(g) << 11) | (f32_to_ufloat<5>(b) << 22);
}
__host__ __device__ __forceinline__ void unpack_b10g11r11(uint32_t v, float *r, float *g, float *b) {
  *r = ufloat_to_f32<6>(v & 0x7ffu);
  *g = ufloat_to_f32<6>((v >> 11) & 0x7ffu);
  *b = ufloat_to_f32<5>(v >> 22);
}

}  // namespace gs
