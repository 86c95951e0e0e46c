// owners.cuh -- move-only owners of the CUDA resources of a handle and its lanes: device memory, pinned host memory, streams
// and events.  An owner starts empty; alloc / create releases what it held, acquires a new resource and stays empty when that
// fails; the destructor releases the resource.  It converts to the raw pointer or handle, so launches and copies take it as
// they took the raw value; get() serves casts and template arguments.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace qb {

// H: the raw pointer or handle; Api::acquire(H*, args...) creates one, Api::release(H) gives it back
template <class H, class Api>
class Owner {
 public:
  Owner() = default;
  Owner(const Owner&) = delete;
  Owner& operator=(const Owner&) = delete;
  Owner(Owner&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
  Owner& operator=(Owner&& o) noexcept {
    if (this != &o) {
      reset();
      h_ = o.h_;
      o.h_ = nullptr;
    }
    return *this;
  }
  ~Owner() { reset(); }

  void reset() {
    if (h_) Api::release(h_);
    h_ = nullptr;
  }
  H get() const { return h_; }
  operator H() const { return h_; }

 protected:
  template <class... A>
  cudaError_t acquire(A... args) {
    reset();
    H h = nullptr;
    const cudaError_t e = Api::acquire(&h, args...);
    if (e == cudaSuccess) h_ = h;
    return e;
  }

 private:
  H h_ = nullptr;
};

struct DeviceApi {
  template <class T>
  static cudaError_t acquire(T** p, size_t bytes) { return cudaMalloc((void**)p, bytes); }
  static void release(const void* p) { cudaFree(const_cast<void*>(p)); }
};
struct PinnedApi {
  template <class T>
  static cudaError_t acquire(T** p, size_t bytes) { return cudaMallocHost((void**)p, bytes); }
  static void release(const void* p) { cudaFreeHost(const_cast<void*>(p)); }
};
struct StreamApi {
  static cudaError_t acquire(cudaStream_t* s, unsigned flags) { return cudaStreamCreateWithFlags(s, flags); }
  static void release(cudaStream_t s) { cudaStreamDestroy(s); }
};
struct EventApi {
  static cudaError_t acquire(cudaEvent_t* e, unsigned flags) { return cudaEventCreateWithFlags(e, flags); }
  static void release(cudaEvent_t e) { cudaEventDestroy(e); }
};

// count elements of T (alloc) or a byte count (alloc_bytes, also for T = void)
template <class T, class Api>
struct Memory : Owner<T*, Api> {
  cudaError_t alloc(size_t count) { return this->acquire(count * sizeof(T)); }
  cudaError_t alloc_bytes(size_t bytes) { return this->acquire(bytes); }
};
template <class T>
using DeviceMem = Memory<T, DeviceApi>;
template <class T>
using PinnedMem = Memory<T, PinnedApi>;

struct Stream : Owner<cudaStream_t, StreamApi> {
  cudaError_t create(unsigned flags) { return acquire(flags); }
};
struct Event : Owner<cudaEvent_t, EventApi> {
  cudaError_t create(unsigned flags = cudaEventDefault) { return acquire(flags); }
};

}  // namespace qb
