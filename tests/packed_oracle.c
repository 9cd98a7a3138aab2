/* packed_oracle.c -- see packed_oracle.h.  Built with -ffp-contract=off, like the CPU oracle: FMA only where fmaf is written.
 *
 * The codec is stated through the value, not the bits: x is scaled by the quantum of its binade (the denormal quantum
 * 2^(-14 - mbits) below 2^-14), rounded to an integer by nearbyint (round to nearest, ties to even: the default rounding mode),
 * and that integer plus the binade's offset is the code; a rounding that reaches the next binade carries into the exponent by
 * itself. */
#include "packed_oracle.h"

#include <math.h>
#include <stddef.h>
#include <string.h>

static float as_f32(uint32_t u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}

static uint32_t to_ufloat(float x, int mbits) {
  const uint32_t inf = 31u << mbits;
  if (isnan(x)) return inf | ((1u << mbits) - 1u);
  if (!(x > 0.0f)) return 0;
  if (isinf(x)) return inf;
  int e2;
  frexp((double)x, &e2);                 /* x = f * 2^e2, f in [0.5, 1): the binade of x is 2^(e2 - 1) */
  const int e = e2 - 1 < -14 ? -14 : e2 - 1;
  const double n = nearbyint(ldexp((double)x, mbits - e));   /* x / 2^(e - mbits), exact in double */
  const double code = (double)((uint32_t)(e + 15) << mbits) + n - (double)(1u << mbits);   /* below 2^-13 this is n */
  return code >= (double)inf ? inf : (uint32_t)code;
}

static float from_ufloat(uint32_t c, int mbits) {
  const uint32_t e = (c >> mbits) & 31u, m = c & ((1u << mbits) - 1u);
  if (e == 31) return m ? as_f32(0x7fc00000u | (m << (23 - mbits))) : as_f32(0x7f800000u);
  if (e == 0) return ldexpf((float)m, -14 - mbits);
  return ldexpf((float)(m + (1u << mbits)), (int)e - 15 - mbits);
}

uint32_t gso_f32_to_uf11(float x) { return to_ufloat(x, 6); }
uint32_t gso_f32_to_uf10(float x) { return to_ufloat(x, 5); }
float gso_uf11_to_f32(uint32_t c) { return from_ufloat(c & 0x7ffu, 6); }
float gso_uf10_to_f32(uint32_t c) { return from_ufloat(c & 0x3ffu, 5); }

static float gamma_to_linear(float x) { /* UnityCG.cginc GammaToLinearSpace, as the CPU oracle states it */
  return x * fmaf(x, fmaf(x, 0.305306011f, 0.682171111f), 0.012522878f);
}

void gso_composite_b10g11r11(const float *rt, uint32_t *target, uint32_t W, uint32_t H) {
  for (size_t i = 0; i < (size_t)W * H; ++i) {
    const float *c = &rt[i * 4];
    const float a = c[3];
    if (!(a > 0.0f)) continue;   /* SrcAlpha == 0: the texel keeps its bits */
    const float om = 1.0f - a;
    const uint32_t t = target[i];
    const float d[3] = {gso_uf11_to_f32(t), gso_uf11_to_f32(t >> 11), gso_uf10_to_f32(t >> 22)};
    float o[3];
    for (int k = 0; k < 3; ++k) o[k] = fmaf(gamma_to_linear(c[k] / a), a, d[k] * om);
    target[i] = gso_f32_to_uf11(o[0]) | (gso_f32_to_uf11(o[1]) << 11) | (gso_f32_to_uf10(o[2]) << 22);
  }
}
