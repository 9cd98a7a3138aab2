/* srgb8_oracle.c -- see srgb8_oracle.h.  Built with -ffp-contract=off, like the CPU oracle: FMA only where fmaf is written. */
#include "srgb8_oracle.h"

#include <math.h>
#include <stddef.h>

static double oetf(double x) { return x <= 0.0031308 ? 12.92 * x : 1.055 * pow(x, 1.0 / 2.4) - 0.055; }
static double eotf(double v) { return v <= 0.04045 ? v / 12.92 : pow((v + 0.055) / 1.055, 2.4); }

uint32_t gso_srgb8_encode(float x) {
  if (isnan(x) || x <= 0.0f) return 0;
  if (x >= 1.0f) return 255;
  const double n = floor(255.0 * oetf((double)x) + 0.5);
  return n < 0.0 ? 0 : n > 255.0 ? 255 : (uint32_t)n;
}

uint32_t gso_unorm8_encode(float x) {
  if (isnan(x) || x <= 0.0f) return 0;
  if (x >= 1.0f) return 255;
  return (uint32_t)floor(255.0 * (double)x + 0.5);   /* 255 x is exact in double */
}

float gso_srgb8_decode(uint32_t c) { return (float)eotf((double)(c & 0xffu) / 255.0); }
float gso_unorm8_decode(uint32_t c) { return (float)(c & 0xffu) / 255.0f; }

static float gamma_to_linear(float x) { /* UnityCG.cginc GammaToLinearSpace, as the CPU oracle states it */
  return x * fmaf(x, fmaf(x, 0.305306011f, 0.682171111f), 0.012522878f);
}

void gso_composite_srgb8(const float *rt, uint8_t *target, uint32_t W, uint32_t H) {
  for (size_t i = 0; i < (size_t)W * H; ++i) {
    const float *c = &rt[i * 4];
    uint8_t *t = &target[i * 4];
    const float a = c[3];
    if (!(a > 0.0f)) continue;   /* SrcAlpha == 0: the texel keeps its bytes */
    const float om = 1.0f - a;
    float o[4];
    for (int k = 0; k < 3; ++k) o[k] = fmaf(gamma_to_linear(c[k] / a), a, gso_srgb8_decode(t[k]) * om);
    o[3] = fmaf(a, a, gso_unorm8_decode(t[3]) * om);
    for (int k = 0; k < 3; ++k) t[k] = (uint8_t)gso_srgb8_encode(o[k]);
    t[3] = (uint8_t)gso_unorm8_encode(o[3]);
  }
}
