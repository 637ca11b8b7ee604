// Shared host-side helpers for libt2h.so: error reporting and launch checks.
#pragma once
#include <cstdlib>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/t2h.h"

namespace t2h {

// printf-style; stores the message for t2h_last_error() and returns `code`.
int fail(int code, const char* fmt, ...);
int num_sms();

#define T2H_CHECK_ARG(cond, ...)                        \
  do {                                                  \
    if (!(cond)) return ::t2h::fail(T2H_EINVAL, __VA_ARGS__); \
  } while (0)

#define T2H_CUDA(expr)                                                              \
  do {                                                                              \
    cudaError_t e__ = (expr);                                                       \
    if (e__ != cudaSuccess)                                                         \
      return ::t2h::fail(T2H_ECUDA, "%s failed: %s (%s:%d)", #expr,                  \
                         cudaGetErrorString(e__), __FILE__, __LINE__);              \
  } while (0)

// launch-error check that does not synchronise
#define T2H_LAUNCH_OK() T2H_CUDA(cudaPeekAtLastError())

static inline cudaStream_t as_stream(t2h_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

// T2H_PDL=0 turns programmatic dependent launch off (A/B measurements)
static inline bool pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("T2H_PDL");
    on = (e && e[0] == '0') ? 0 : 1;
  }
  return on == 1;
}

// T2H_DEBUG bits; bit 16: CTA 0 of every tap-GEMM / attention launch records a globaltimer trace (t2h_debug_read)
static inline int debug_bits() {
  static int bits = -1;
  if (bits < 0) {
    const char* e = getenv("T2H_DEBUG");
    bits = e ? atoi(e) : 0;
  }
  return bits;
}

// Launch a kernel that calls pdl_wait() before its first dependent global access, allowing it to overlap its
// prologue with the previous kernel's tail (also inside CUDA-graph capture, where it becomes a programmatic edge).
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  int n = 0;
  if (pdl_enabled()) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = at;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

}  // namespace t2h
