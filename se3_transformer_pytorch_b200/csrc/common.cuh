// Shared helpers for the se3b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include "../../include/se3b200.h"

namespace se3 {

void set_error(const char* fmt, ...);

#define SE3_REQUIRE(cond, ...)                                   \
  do {                                                           \
    if (!(cond)) { ::se3::set_error(__VA_ARGS__); return SE3_EINVAL; } \
  } while (0)

#define SE3_CUDA_OK(expr)                                                                   \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      ::se3::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return SE3_ECUDA;                                                                     \
    }                                                                                       \
  } while (0)

#define SE3_LAUNCH_OK() SE3_CUDA_OK(cudaGetLastError())

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace se3
