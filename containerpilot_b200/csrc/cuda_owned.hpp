// cuda_owned.hpp — move-only owners of the CUDA memory, events and streams that a bus creates (DESIGN.md §5, "What
// the bus owns").
//
// An owner frees what it holds when it is destroyed or reset, and never throws.  A buffer converts to its pointer: the
// device pointer for device memory, the host pointer for pinned and mapped memory; dev() is the pointer a kernel takes.
//
// Failure rule: an allocation or creation the runtime refuses leaves the owner empty ({nullptr, 0}), whatever the runtime
// wrote into its out-parameter, and consumes the runtime's last error, so that the next, unrelated launch check does not
// report it.  The caller gets the error as the return value.
#pragma once

#include <cuda_runtime_api.h>

#include <cstddef>
#include <utility>

namespace cuda_owned {

enum class Mem {
  Device,   // cudaMalloc
  Pinned,   // cudaMallocHost
  Mapped,   // cudaHostAlloc(cudaHostAllocMapped): pinned host memory that kernels reach through its device alias
};

template <class T, Mem M>
class Buffer {
 public:
  Buffer() = default;
  Buffer(Buffer&& o) noexcept
      : h_(std::exchange(o.h_, nullptr)), d_(std::exchange(o.d_, nullptr)), n_(std::exchange(o.n_, 0)) {}
  Buffer& operator=(Buffer&& o) noexcept {
    if (this != &o) {
      reset();
      h_ = std::exchange(o.h_, nullptr); d_ = std::exchange(o.d_, nullptr); n_ = std::exchange(o.n_, 0);
    }
    return *this;
  }
  Buffer(const Buffer&) = delete;
  Buffer& operator=(const Buffer&) = delete;
  ~Buffer() { reset(); }

  T* get() const { return h_; }
  operator T*() const { return h_; }
  T* operator->() const { return h_; }
  T* dev() const { return d_; }
  size_t size() const { return n_; }   // in elements of T

  // Exactly n elements, in place of what the buffer held.
  cudaError_t alloc(size_t n) {
    reset();
    void *h = nullptr, *d = nullptr;
    cudaError_t e = cudaSuccess;
    if constexpr (M == Mem::Device) { e = cudaMalloc(&h, n * sizeof(T)); d = h; }
    else if constexpr (M == Mem::Pinned) { e = cudaMallocHost(&h, n * sizeof(T)); d = h; }
    else if ((e = cudaHostAlloc(&h, n * sizeof(T), cudaHostAllocMapped)) == cudaSuccess &&
             (e = cudaHostGetDevicePointer(&d, h, 0)) != cudaSuccess)
      cudaFreeHost(h);
    if (e != cudaSuccess) { cudaGetLastError(); return e; }
    h_ = static_cast<T*>(h); d_ = static_cast<T*>(d); n_ = n;
    return cudaSuccess;
  }

  // At least n elements: nothing happens while n fits; otherwise the buffer is freed and max(n, floor) are allocated.  The
  // contents are not kept, and the caller makes sure that no copy or kernel still uses the old memory.
  cudaError_t grow(size_t n, size_t floor = 0) { return n <= n_ ? cudaSuccess : alloc(n < floor ? floor : n); }

  void reset() {
    if (h_) M == Mem::Device ? cudaFree(h_) : cudaFreeHost(h_);
    h_ = d_ = nullptr; n_ = 0;
  }

 private:
  T* h_ = nullptr;   // what the buffer converts to
  T* d_ = nullptr;   // its device alias (the same pointer unless mapped)
  size_t n_ = 0;
};

template <class T> using DeviceBuf = Buffer<T, Mem::Device>;
template <class T> using PinnedBuf = Buffer<T, Mem::Pinned>;
template <class T> using MappedBuf = Buffer<T, Mem::Mapped>;

// A CUDA event or stream that the owner created (with the one flag every bus uses for its kind).
template <class H, cudaError_t (*Create)(H*, unsigned int), cudaError_t (*Destroy)(H), unsigned int Flags>
class Handle {
 public:
  Handle() = default;
  Handle(Handle&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  Handle& operator=(Handle&& o) noexcept {
    if (this != &o) { reset(); h_ = std::exchange(o.h_, nullptr); }
    return *this;
  }
  Handle(const Handle&) = delete;
  Handle& operator=(const Handle&) = delete;
  ~Handle() { reset(); }

  operator H() const { return h_; }

  cudaError_t create() {
    reset();
    H h{};
    const cudaError_t e = Create(&h, Flags);
    if (e != cudaSuccess) { cudaGetLastError(); return e; }
    h_ = h;
    return cudaSuccess;
  }

  void reset() { if (h_) Destroy(h_); h_ = nullptr; }

 private:
  H h_ = nullptr;
};

using CudaEvent = Handle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy, cudaEventDisableTiming>;
using CudaStream = Handle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy, cudaStreamNonBlocking>;

}  // namespace cuda_owned
