// Shared plumbing for the b200slam library: error reporting, CUDA call checking, small RAII
// wrappers for device / pinned-host buffers.  No compute lives here.
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>

#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <exception>
#include <functional>
#include <new>
#include <string>

#include "../../include/b200slam.h"

namespace b200 {

void set_last_error(const std::string & s);

struct CudaFail {
  int code;
};

#define B200_CUDA(expr)                                                                       \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      ::b200::set_last_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" +      \
                             __FILE__ + ":" + std::to_string(__LINE__) + ")");                \
      throw ::b200::CudaFail{B200_ERR_CUDA};                                                  \
    }                                                                                         \
  } while (0)

// Around the body of a C ABI entry: a failed CUDA call, an exhausted host heap or any other exception becomes its error
// code (and the last error message) instead of crossing the C boundary.
#define B200_GUARD_BEGIN try {
#define B200_GUARD_END                                                     \
  }                                                                        \
  catch (const b200::CudaFail & f) { return f.code; }                      \
  catch (const std::bad_alloc &) { b200::set_last_error("out of host memory"); return B200_ERR_CUDA; } \
  catch (const std::exception & e) { b200::set_last_error(e.what()); return B200_ERR_CUDA; }

// Fails loudly (B200_ERR_CUDA) when there is no sm_90 device: there is no CPU fallback.
void require_device();

// NVTX range (shows up in Nsight Systems / ncu --nvtx; a no-op without an attached tool): upload / run / fetch of a sweep,
// single matches, LM iterations of a solve (SURVEY.md 5, "tracing")
struct NvtxRange {
  explicit NvtxRange(const char * name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange &) = delete;
  NvtxRange & operator=(const NvtxRange &) = delete;
};

// A small persistent pool of host threads for the table building on the host side of the ABI (lookup tables per angle,
// FindValidPoints per base scan, descriptor lists per angle): parallel_for(n, fn) runs fn(0..n-1), the caller takes part.
// B200_HOST_THREADS sets the size (default: up to 8, at most half the cores; 1 = everything on the calling thread).
void host_parallel_for(int n, const std::function<void(int)> & fn);
int host_pool_threads();

template <class T>
struct DevBuf {
  T * p = nullptr;
  size_t cap = 0;
  ~DevBuf() { release(); }
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf & operator=(const DevBuf &) = delete;
  void release()
  {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  // grow-only; contents are NOT preserved
  void reserve(size_t n)
  {
    if (n <= cap) return;
    release();
    size_t want = n + n / 4 + 16;
    B200_CUDA(cudaMalloc(reinterpret_cast<void **>(&p), want * sizeof(T)));
    cap = want;
  }
};

template <class T>
struct PinBuf {
  T * p = nullptr;
  size_t cap = 0;
  ~PinBuf() { release(); }
  PinBuf() = default;
  PinBuf(const PinBuf &) = delete;
  PinBuf & operator=(const PinBuf &) = delete;
  void release()
  {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
  void reserve(size_t n)
  {
    if (n <= cap) return;
    release();
    size_t want = n + n / 4 + 16;
    B200_CUDA(cudaMallocHost(reinterpret_cast<void **>(&p), want * sizeof(T)));
    cap = want;
  }
};

}  // namespace b200
