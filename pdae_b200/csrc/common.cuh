// Shared helpers for the pdae_b200 kernels (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "pdae_b200.h"

namespace pdae {

void set_error(const char* fmt, ...);
// Deterministic statistics (norm_elementwise.cu): per-channel (sum, sum^2) partials [B][P][C][2], written with plain stores by
// P producers per image, summed over P in ascending order into [B][C][2].
cudaError_t launch_stat_parts_reduce(const float* part, int B, int P, int C, float* chs, cudaStream_t s);
// out[i] = sum over s = 0..S-1, in that order, of part[s * n + i] (backward_simt.cu): the reduction of deterministic slots
cudaError_t launch_slot_sum(const float* part, int S, long long n, float* out, cudaStream_t s);

#define PDAE_REQUIRE(cond, ...)             \
  do {                                      \
    if (!(cond)) {                          \
      ::pdae::set_error(__VA_ARGS__);       \
      return PDAE_EINVAL;                   \
    }                                       \
  } while (0)

#define PDAE_CUDA(expr)                                                                   \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      ::pdae::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                        __LINE__);                                                        \
      return PDAE_ECUDA;                                                                  \
    }                                                                                     \
  } while (0)

#define PDAE_LAUNCH_CHECK(name)                                                       \
  do {                                                                                \
    cudaError_t _e = cudaPeekAtLastError();                                           \
    if (_e != cudaSuccess) {                                                          \
      (void)cudaGetLastError();                                                       \
      ::pdae::set_error("launch of %s failed: %s", name, cudaGetErrorString(_e));     \
      return PDAE_ECUDA;                                                              \
    }                                                                                 \
  } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }

template <typename T>
__device__ __forceinline__ float4 load4(const T* p);
template <>
__device__ __forceinline__ float4 load4<float>(const float* p) {
  return *reinterpret_cast<const float4*>(p);
}
template <>
__device__ __forceinline__ float4 load4<__nv_bfloat16>(const __nv_bfloat16* p) {
  uint2 u = *reinterpret_cast<const uint2*>(p);
  __nv_bfloat162 lo = *reinterpret_cast<__nv_bfloat162*>(&u.x);
  __nv_bfloat162 hi = *reinterpret_cast<__nv_bfloat162*>(&u.y);
  float2 a = __bfloat1622float2(lo), b = __bfloat1622float2(hi);
  return make_float4(a.x, a.y, b.x, b.y);
}
template <typename T>
__device__ __forceinline__ void store4(T* p, float4 v);
template <>
__device__ __forceinline__ void store4<float>(float* p, float4 v) {
  *reinterpret_cast<float4*>(p) = v;
}
template <>
__device__ __forceinline__ void store4<__nv_bfloat16>(__nv_bfloat16* p, float4 v) {
  __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y);
  __nv_bfloat162 hi = __floats2bfloat162_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&lo);
  u.y = *reinterpret_cast<uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(p) = u;
}
template <typename T>
__device__ __forceinline__ float load1(const T* p);
template <>
__device__ __forceinline__ float load1<float>(const float* p) {
  return *p;
}
template <>
__device__ __forceinline__ float load1<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat162float(*p);
}
__device__ __forceinline__ void store1(float* p, float v) { *p = v; }
__device__ __forceinline__ void store1(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

}  // namespace pdae
