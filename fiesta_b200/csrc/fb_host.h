// fiesta_b200 -- host-side ownership of device and pinned host memory, and the one error channel of the C ABI.
//
// Every buffer the library keeps is an FbDevBuf / FbHostBuf member: the destructor frees it, so an owner (map, query plan,
// host mirror, order-exact state) needs no free list and a creation that fails part-way cleans up by destruction.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <utility>
#include "../../include/fiesta_b200.h"

// printf-style; sets the calling thread's fiesta_last_error() message (defined in fb_map.cu)
void fb_set_error(const char *fmt, ...);
#define CK(call)                                                                                                        \
  do {                                                                                                                  \
    cudaError_t e__ = (call);                                                                                           \
    if (e__ != cudaSuccess) { fb_set_error("%s failed: %s", #call, cudaGetErrorString(e__)); return FIESTA_ERR_CUDA; } \
  } while (0)

// Move-only array of `cap` elements in device memory (HOST = false) or pinned host memory (HOST = true).
template <typename T, bool HOST>
struct FbBuf {
  T *p = nullptr;
  size_t cap = 0;

  FbBuf() = default;
  FbBuf(const FbBuf &) = delete;
  FbBuf &operator=(const FbBuf &) = delete;
  FbBuf(FbBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  FbBuf &operator=(FbBuf &&o) noexcept {
    std::swap(p, o.p);
    std::swap(cap, o.cap);
    return *this;
  }
  ~FbBuf() {
    if (p) { if (HOST) cudaFreeHost(p); else cudaFree(p); }
  }
  operator T *() const { return p; }
  T *operator->() const { return p; }

  // Exactly n elements; the previous block (and its contents) is released first.
  cudaError_t alloc(size_t n) {
    *this = FbBuf();
    void *q = nullptr;
    const cudaError_t e = HOST ? cudaMallocHost(&q, n * sizeof(T)) : cudaMalloc(&q, n * sizeof(T));
    if (e != cudaSuccess) return e;
    p = static_cast<T *>(q);
    cap = n;
    return cudaSuccess;
  }
  // At least `need` elements, with room to grow: need + need/2 + 4096.  The first `keep` elements are copied on the
  // stream `s`, which is synchronised before the old block is released.
  cudaError_t grow(size_t need, cudaStream_t s, size_t keep = 0) {
    if (need <= cap) return cudaSuccess;
    FbBuf nb;
    cudaError_t e = nb.alloc(need + need / 2 + 4096);
    if (e == cudaSuccess && keep && p) e = cudaMemcpyAsync(nb.p, p, keep * sizeof(T), cudaMemcpyDefault, s);
    if (e == cudaSuccess && keep && p) e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) *this = std::move(nb);
    return e;
  }
};
template <typename T> using FbDevBuf = FbBuf<T, false>;
template <typename T> using FbHostBuf = FbBuf<T, true>;
