/* srgb8_oracle.h -- the CPU restatement of GS_PIX_R8G8B8A8_SRGB camera targets the sRGB8 tests compare the library with
 * (tests/srgb8_oracle.c; test infrastructure, compiled by tests/srgb8_oracle.py).  It shares no code with the library.
 *
 * Four bytes per pixel, R, G, B, A in memory order (R in bits 0-7 of the little-endian word); RGB sRGB-encoded, A linear UNorm,
 * after IEC 61966-2-1.  The codec is stated through the value, in double precision:
 *   decode  RGB: c -> (float) EOTF(c / 255);  A: a -> (float) a / 255.0f;
 *   encode  RGB: NaN and x <= 0 -> 0, x >= 1 -> 255, else floor(255 OETF(x) + 0.5), the number of j in 1..255 with
 *           255 OETF(x) >= j - 0.5;  A: NaN -> 0, else floor(255 clamp(x, 0, 1) + 0.5), exact in double.
 * Double evaluation of the transfer functions is exact enough wherever a float32 lies farther than 1e-15 (relative) from a
 * decision boundary or a float32 rounding midpoint; the tests check the tables' entries and both floats beside every
 * threshold against 50-digit decimal arithmetic, which covers the places where it could not be.
 * The composite is GaussianComposite's blend, as the CPU oracle's gso_composite states it onto an RGBA32F target, on the decoded
 * texel, then the encode; a pixel whose alpha is not > 0 keeps its bytes. */
#ifndef SRGB8_ORACLE_H
#define SRGB8_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

uint32_t gso_srgb8_encode(float x);        /* linear RGB channel -> code */
uint32_t gso_unorm8_encode(float x);       /* linear alpha -> code */
float gso_srgb8_decode(uint32_t c);        /* the low 8 bits of c */
float gso_unorm8_decode(uint32_t c);       /* the low 8 bits of c */
/* rt: W*H*4 floats (premultiplied RGBA); target: W*H*4 bytes, read-modify-write */
void gso_composite_srgb8(const float *rt, uint8_t *target, uint32_t width, uint32_t height);

#ifdef __cplusplus
}
#endif
#endif
