/* packed_oracle.h -- the CPU restatement of GS_PIX_B10G11R11_UFLOAT camera targets the packed-target tests compare the library
 * with (tests/packed_oracle.c; test infrastructure, compiled by tests/packed_oracle.py).  It shares no code with the library.
 *
 * One uint32 per pixel: R bits 0-10 and G 11-21 unsigned float11, B 22-31 unsigned float10 (5 exponent bits, bias 15; 6 or 5
 * mantissa bits), after the format definitions of the Vulkan and D3D11 specifications.
 *   decode  exact: exponent 0 denormal, 31 +Inf (mantissa 0) or a quiet NaN that keeps the mantissa (0x7FC00000 | m << (23 - M));
 *   encode  NaN -> all ones, <= 0 (-0, -Inf) -> 0, +Inf -> Inf, else round to nearest, ties to even, with IEEE overflow.
 * The composite is GaussianComposite's blend, as the CPU oracle's gso_composite states it, on the decoded r, g, b, with alpha
 * dropped; a pixel whose alpha is not > 0 keeps its bits. */
#ifndef PACKED_ORACLE_H
#define PACKED_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

uint32_t gso_f32_to_uf11(float x);
uint32_t gso_f32_to_uf10(float x);
float gso_uf11_to_f32(uint32_t c);   /* the low 11 bits of c */
float gso_uf10_to_f32(uint32_t c);   /* the low 10 bits of c */
/* rt: W*H*4 floats (premultiplied RGBA); target: W*H texels, read-modify-write */
void gso_composite_b10g11r11(const float *rt, uint32_t *target, uint32_t width, uint32_t height);

#ifdef __cplusplus
}
#endif
#endif
