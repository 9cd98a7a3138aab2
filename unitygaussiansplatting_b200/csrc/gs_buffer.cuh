// gs_buffer.cuh -- the owner of every scratch allocation a context or group member keeps between calls: one pointer and its
// size in one object, so a buffer is either allocated at its recorded size or empty.
#pragma once
#include <cstddef>
#include <initializer_list>

#include <cuda_runtime.h>

namespace gs {

// A device allocation (PINNED: pinned host memory, cudaMallocHost) of size() elements of T, or nothing (get() == nullptr,
// size() == 0).  Move-only.  The destructor frees it: the owner drains every stream that uses it first, and makes the
// allocation's device current.
template <class T, bool PINNED = false>
class Buffer {
 public:
  Buffer() = default;
  Buffer(const Buffer &) = delete;
  Buffer &operator=(const Buffer &) = delete;
  Buffer(Buffer &&o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
  Buffer &operator=(Buffer &&o) noexcept {
    if (this != &o) {
      reset();
      p_ = o.p_; n_ = o.n_;
      o.p_ = nullptr; o.n_ = 0;
    }
    return *this;
  }
  ~Buffer() { reset(); }

  T *get() const { return p_; }
  size_t size() const { return n_; }

  // Room for at least n elements; the contents are not kept.  Reallocates only when n > size(): every stream in `users` (the
  // streams that may still use the old allocation; never the null stream) is synchronized, then the old allocation is freed.
  // On failure the buffer is empty, the runtime's last error is cleared (the next call's cudaGetLastError does not report
  // it again), and the error is returned.
  cudaError_t reserve(size_t n, std::initializer_list<cudaStream_t> users) {
    if (n <= n_) return cudaSuccess;
    if (p_) {
      for (cudaStream_t s : users) cudaStreamSynchronize(s);
      reset();
    }
    void *p = nullptr;
    const cudaError_t e = PINNED ? cudaMallocHost(&p, n * sizeof(T)) : cudaMalloc(&p, n * sizeof(T));
    if (e != cudaSuccess) {
      cudaGetLastError();
      return e;
    }
    p_ = static_cast<T *>(p);
    n_ = n;
    return cudaSuccess;
  }

  // Frees the allocation now.
  void reset() {
    if (p_) {
      if (PINNED) cudaFreeHost(p_);
      else cudaFree(p_);
    }
    p_ = nullptr;
    n_ = 0;
  }

 private:
  T *p_ = nullptr;
  size_t n_ = 0;
};

}  // namespace gs
