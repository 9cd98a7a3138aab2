// The device codec of GS_PIX_R8G8B8A8_SRGB texels (csrc/gs_srgb8.cuh, as the composite kernel runs it) against the sRGB8
// oracle's restatement (tests/srgb8_oracle.c): the RGB and alpha encoders over every one of the 2^32 float32 bit patterns, and
// the decoders over every code, bit for bit.  Built with the library's nvcc flags and linked against that restatement's shared
// library; exit status 0 when everything agrees.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <thread>
#include <vector>

#include "srgb8_oracle.h"
#include "gs_srgb8.cuh"

constexpr uint64_t kChunk = 1ull << 26;

__global__ void k_encode(uint32_t base, uint8_t *rgb, uint8_t *alpha) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const float f = __uint_as_float(base + i);
  rgb[i] = (uint8_t)gs::srgb8_encode(f);
  alpha[i] = (uint8_t)gs::unorm8_encode(f);
}

__global__ void k_decode(uint32_t *rgb, uint32_t *alpha) {
  const uint32_t c = threadIdx.x;   // 256 threads: every code, as the composite unpacks it
  float r, g, b, a;
  gs::unpack_srgb8(c * 0x01010101u, &r, &g, &b, &a);
  rgb[c] = (r == g && g == b) ? __float_as_uint(r) : 0xffffffffu;
  alpha[c] = __float_as_uint(a);
}

static uint32_t bits(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}
static float from_bits(uint32_t u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e_ = (x);                                                                  \
    if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 2; } \
  } while (0)

int main() {
  // decoders: every code
  uint32_t *drgb, *dalpha;
  CK(cudaMalloc(&drgb, 256 * 4));
  CK(cudaMalloc(&dalpha, 256 * 4));
  k_decode<<<1, 256>>>(drgb, dalpha);
  CK(cudaGetLastError());
  std::vector<uint32_t> hrgb(256), halpha(256);
  CK(cudaMemcpy(hrgb.data(), drgb, 256 * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(halpha.data(), dalpha, 256 * 4, cudaMemcpyDeviceToHost));
  long bad = 0;
  for (uint32_t c = 0; c < 256; ++c) bad += (hrgb[c] != bits(gso_srgb8_decode(c))) + (halpha[c] != bits(gso_unorm8_decode(c)));
  if (bad) { printf("decode: %ld codes differ from the oracle\n", bad); return 1; }

  // encoders: every float32 bit pattern, a chunk at a time; the host checks a chunk on every core
  uint8_t *ergb, *ealpha;
  CK(cudaMalloc(&ergb, kChunk));
  CK(cudaMalloc(&ealpha, kChunk));
  std::vector<uint8_t> grgb(kChunk), galpha(kChunk);
  const unsigned T = std::max(1u, std::thread::hardware_concurrency());
  std::vector<long> bad_t(T);
  std::vector<uint32_t> first_t(T), dev_t(T);
  for (uint64_t base = 0; base < (1ull << 32); base += kChunk) {
    k_encode<<<(unsigned)(kChunk / 256), 256>>>((uint32_t)base, ergb, ealpha);
    CK(cudaGetLastError());
    CK(cudaMemcpy(grgb.data(), ergb, kChunk, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(galpha.data(), ealpha, kChunk, cudaMemcpyDeviceToHost));
    std::vector<std::thread> th;
    for (unsigned t = 0; t < T; ++t)
      th.emplace_back([&, t] {
        for (uint64_t i = t; i < kChunk; i += T) {
          const float f = from_bits((uint32_t)(base + i));
          if (grgb[i] != gso_srgb8_encode(f) || galpha[i] != gso_unorm8_encode(f)) {
            if (!bad_t[t]) { first_t[t] = (uint32_t)(base + i); dev_t[t] = grgb[i] | ((uint32_t)galpha[i] << 8); }
            ++bad_t[t];
          }
        }
      });
    for (auto &x : th) x.join();
  }
  for (unsigned t = 0; t < T; ++t)
    if (bad_t[t]) {
      const float f = from_bits(first_t[t]);
      printf("encode: %ld patterns differ, e.g. 0x%08x: device %u / %u, oracle %u / %u\n", bad_t[t], first_t[t], dev_t[t] & 0xffu,
             dev_t[t] >> 8, gso_srgb8_encode(f), gso_unorm8_encode(f));
      bad += bad_t[t];
    }
  cudaFree(drgb); cudaFree(dalpha); cudaFree(ergb); cudaFree(ealpha);
  if (bad) return 1;
  printf("sRGB8 codec: 2^32 encodes x 2 and 512 decodes agree with the oracle (%u host threads)\n", T);
  return 0;
}
