// Shared helpers for libb2pc (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b2pc.h"

namespace b2pc {

constexpr int kNumSMs = 132;  // H100 SXM

void set_error(const char* fmt, ...);
void count_launches(int n);  // kernels launched by this library (b2pc_launch_count)

#define B2PC_CHECK_ARG(cond, ...)                 \
  do {                                            \
    if (!(cond)) {                                \
      ::b2pc::set_error(__VA_ARGS__);             \
      return B2PC_ERR_INVALID_ARG;                \
    }                                             \
  } while (0)

#define B2PC_CHECK_LAUNCH(what)                                                         \
  do {                                                                                  \
    cudaError_t e__ = cudaGetLastError();                                               \
    if (e__ != cudaSuccess) {                                                           \
      ::b2pc::set_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e__));   \
      return B2PC_ERR_CUDA;                                                             \
    }                                                                                   \
  } while (0)

__host__ __device__ static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
__host__ __device__ static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- dtype <-> float ------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

}  // namespace b2pc
