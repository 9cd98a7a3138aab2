// The device codec of GS_PIX_B10G11R11_UFLOAT texels (csrc/gs_packed_float.cuh, as the composite kernel runs it) against the
// packed-target oracle's restatement (tests/packed_oracle.c): the float11 and float10 encoders over every one of the 2^32 float32 bit
// patterns, and the decoders over every code, bit for bit.  Built with the library's nvcc flags and linked against
// that restatement's shared library; exit status 0 when everything agrees.
#include <cstdio>
#include <cstring>
#include <thread>
#include <vector>

#include "packed_oracle.h"
#include "gs_packed_float.cuh"

constexpr uint64_t kChunk = 1ull << 26;

__global__ void k_encode(uint32_t base, uint16_t *out11, uint16_t *out10) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const float f = __uint_as_float(base + i);
  out11[i] = (uint16_t)gs::f32_to_ufloat<6>(f);
  out10[i] = (uint16_t)gs::f32_to_ufloat<5>(f);
}

__global__ void k_decode(uint32_t *out11, uint32_t *out10) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;   // 2048 threads
  out11[c] = __float_as_uint(gs::ufloat_to_f32<6>(c));
  if (c < 1024) out10[c] = __float_as_uint(gs::ufloat_to_f32<5>(c));
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
  uint32_t *d11, *d10;
  CK(cudaMalloc(&d11, 2048 * 4));
  CK(cudaMalloc(&d10, 1024 * 4));
  k_decode<<<8, 256>>>(d11, d10);
  CK(cudaGetLastError());
  std::vector<uint32_t> h11(2048), h10(1024);
  CK(cudaMemcpy(h11.data(), d11, 2048 * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(h10.data(), d10, 1024 * 4, cudaMemcpyDeviceToHost));
  long bad = 0;
  for (uint32_t c = 0; c < 2048; ++c) bad += h11[c] != bits(gso_uf11_to_f32(c));
  for (uint32_t c = 0; c < 1024; ++c) bad += h10[c] != bits(gso_uf10_to_f32(c));
  if (bad) { printf("decode: %ld codes differ from the oracle\n", bad); return 1; }

  // encoders: every float32 bit pattern, a chunk at a time; the host checks a chunk on every core
  uint16_t *e11, *e10;
  CK(cudaMalloc(&e11, kChunk * 2));
  CK(cudaMalloc(&e10, kChunk * 2));
  std::vector<uint16_t> g11(kChunk), g10(kChunk);
  const unsigned T = std::max(1u, std::thread::hardware_concurrency());
  std::vector<long> bad_t(T);
  std::vector<uint32_t> first_t(T), dev_t(T);
  for (uint64_t base = 0; base < (1ull << 32); base += kChunk) {
    k_encode<<<(unsigned)(kChunk / 256), 256>>>((uint32_t)base, e11, e10);
    CK(cudaGetLastError());
    CK(cudaMemcpy(g11.data(), e11, kChunk * 2, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(g10.data(), e10, kChunk * 2, cudaMemcpyDeviceToHost));
    std::vector<std::thread> th;
    for (unsigned t = 0; t < T; ++t)
      th.emplace_back([&, t] {
        for (uint64_t i = t; i < kChunk; i += T) {
          const float f = from_bits((uint32_t)(base + i));
          if (g11[i] != gso_f32_to_uf11(f) || g10[i] != gso_f32_to_uf10(f)) {
            if (!bad_t[t]) { first_t[t] = (uint32_t)(base + i); dev_t[t] = g11[i] | ((uint32_t)g10[i] << 16); }
            ++bad_t[t];
          }
        }
      });
    for (auto &x : th) x.join();
  }
  for (unsigned t = 0; t < T; ++t)
    if (bad_t[t]) {
      const float f = from_bits(first_t[t]);
      printf("encode: %ld patterns differ, e.g. 0x%08x: device %u / %u, oracle %u / %u\n", bad_t[t], first_t[t],
             dev_t[t] & 0xffffu, dev_t[t] >> 16, gso_f32_to_uf11(f), gso_f32_to_uf10(f));
      bad += bad_t[t];
    }
  cudaFree(d11); cudaFree(d10); cudaFree(e11); cudaFree(e10);
  if (bad) return 1;
  printf("packed float codec: 2^32 encodes x 2 and 3072 decodes agree with the oracle (%u host threads)\n", T);
  return 0;
}
