// gs::Buffer (csrc/gs_buffer.cuh) on its own: a reserve that fails leaves the buffer empty and the runtime's last error
// clear, so neither a stale size nor a stale error outlives the failed call.
//   buffer_test no-device   without a CUDA device: every reserve fails and leaves the buffer empty
//   buffer_test device      on a GPU: growth, a refused 2^50-byte request, recovery, and the pinned variant
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <utility>

#include "gs_buffer.cuh"

using gs::Buffer;

#define CHECK(cond)                                                  \
  do {                                                               \
    if (!(cond)) {                                                   \
      std::printf("buffer_test:%d: check failed: %s\n", __LINE__, #cond); \
      return 1;                                                      \
    }                                                                \
  } while (0)

static int no_device() {
  Buffer<uint32_t> b;
  CHECK(b.reserve(16, {}) != cudaSuccess);
  CHECK(b.get() == nullptr && b.size() == 0);
  CHECK(b.reserve(8, {}) != cudaSuccess);   // a smaller request is not "already there"
  CHECK(b.get() == nullptr && b.size() == 0);
  return 0;
}

static int device() {
  cudaStream_t s = nullptr;
  CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess);
  {
    Buffer<uint32_t> b;
    CHECK(b.reserve(16, {s}) == cudaSuccess);
    uint32_t *p = b.get();
    CHECK(p != nullptr && b.size() == 16);
    CHECK(b.reserve(8, {s}) == cudaSuccess);   // fits: kept
    CHECK(b.get() == p && b.size() == 16);

    // refused by the allocator up front: nothing is taken from the device
    CHECK(b.reserve((size_t(1) << 50) / sizeof(uint32_t), {s}) == cudaErrorMemoryAllocation);
    CHECK(b.get() == nullptr && b.size() == 0);
    CHECK(cudaGetLastError() == cudaSuccess);
    CHECK(b.reserve(8, {s}) == cudaSuccess);   // the old size is gone with the old allocation: this allocates again
    CHECK(b.get() != nullptr && b.size() == 8);
    CHECK(cudaMemsetAsync(b.get(), 0, 8 * sizeof(uint32_t), s) == cudaSuccess);

    Buffer<uint32_t> moved(std::move(b));
    CHECK(b.get() == nullptr && b.size() == 0);
    CHECK(moved.get() != nullptr && moved.size() == 8);
    moved.reset();
    CHECK(moved.get() == nullptr && moved.size() == 0);
  }
  {
    Buffer<uint32_t, true> h;
    CHECK(h.reserve(16, {s}) == cudaSuccess);
    uint32_t *p = h.get();
    CHECK(p != nullptr && h.size() == 16);
    for (uint32_t i = 0; i < 16; ++i) p[i] = i;   // host memory
    cudaPointerAttributes attr;
    CHECK(cudaPointerGetAttributes(&attr, p) == cudaSuccess && attr.type == cudaMemoryTypeHost);
    CHECK(h.reserve(8, {s}) == cudaSuccess);
    CHECK(h.get() == p && h.size() == 16 && p[15] == 15);
    CHECK(h.reserve(64, {s}) == cudaSuccess);
    CHECK(h.get() != nullptr && h.size() == 64);
    h.reset();
    CHECK(h.get() == nullptr && h.size() == 0);
  }
  CHECK(cudaStreamSynchronize(s) == cudaSuccess);
  CHECK(cudaStreamDestroy(s) == cudaSuccess);
  CHECK(cudaGetLastError() == cudaSuccess);
  return 0;
}

int main(int argc, char **argv) {
  if (argc == 2 && std::strcmp(argv[1], "no-device") == 0) return no_device();
  if (argc == 2 && std::strcmp(argv[1], "device") == 0) return device();
  std::printf("usage: buffer_test no-device|device\n");
  return 2;
}
