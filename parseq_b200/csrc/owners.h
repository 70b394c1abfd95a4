// Owners of the engine's device resources (engine.cu): every device buffer, stream, event and graph exec of an engine
// or a lexicon has one owner here, which releases it when destroyed or assigned over.
//
// Each release must run with the owner's device current.  Owners are destroyed or replaced only inside
// parseq_destroy, parseq_lexicon_destroy, the resize path of parseq_set_option, DevBuf::grow and the entry points after
// their cudaSetDevice, which all set the device first.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <utility>

#include "../../include/parseq_b200.h"

// Process-wide counts of what the owners hold: parseq_debug_int(NULL, "live_device_bytes" | "live_cuda_objects")
inline std::atomic<long long> g_live_bytes{0}, g_live_objects{0};

// One cudaMalloc allocation of n elements of T.  It converts to T*, so that launch sites pass it as a pointer.
template <typename T>
class DevBuf {
 public:
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) {
      reset();
      p_ = std::exchange(o.p_, nullptr);
      n_ = std::exchange(o.n_, 0);
    }
    return *this;
  }
  ~DevBuf() { reset(); }
  operator T*() const { return p_; }
  T* get() const { return p_; }
  long long size() const { return n_; }

  // n elements in place of what the buffer held; a PARSEQ_* status, the error message through fail() (engine.cu)
  int alloc(long long n);
  // n elements on first use only; adds the bytes it allocates to *counted
  int reserve(long long n, long long* counted = nullptr) {
    if (p_ != nullptr) return PARSEQ_OK;
    const int r = alloc(n);
    if (r == PARSEQ_OK && counted != nullptr) *counted += bytes();
    return r;
  }
  // A buffer of a call's inputs that grows on demand to n elements.  The kernels of the previous call, on the engine's
  // `main` or `copy` stream, may still read the old one: both streams are drained before it is freed.
  int grow(const parseq_engine* e, long long n);

 private:
  long long bytes() const { return n_ * static_cast<long long>(sizeof(T)); }
  void reset() {
    if (p_ == nullptr) return;
    cudaFree(p_);
    g_live_bytes -= bytes();
    p_ = nullptr;
    n_ = 0;
  }
  T* p_ = nullptr;
  long long n_ = 0;
};

// A stream, event or graph exec, released by Destroy
template <typename H, cudaError_t (*Destroy)(H)>
class CudaHandle {
 public:
  CudaHandle() = default;
  explicit CudaHandle(H h) : h_(h) { if (h_ != nullptr) ++g_live_objects; }
  CudaHandle(CudaHandle&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  CudaHandle& operator=(CudaHandle&& o) noexcept {
    if (this != &o) {
      reset();
      h_ = std::exchange(o.h_, nullptr);
    }
    return *this;
  }
  ~CudaHandle() { reset(); }
  operator H() const { return h_; }

 private:
  void reset() {
    if (h_ == nullptr) return;
    Destroy(h_);
    --g_live_objects;
    h_ = nullptr;
  }
  H h_ = nullptr;
};
using Stream = CudaHandle<cudaStream_t, cudaStreamDestroy>;
using Event = CudaHandle<cudaEvent_t, cudaEventDestroy>;
using GraphExec = CudaHandle<cudaGraphExec_t, cudaGraphExecDestroy>;
