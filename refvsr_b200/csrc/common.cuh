// Shared helpers for the refvsr_b200 kernels (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdio>
#include <string>

#include "../../include/refvsr_b200.h"

namespace rv {

extern thread_local std::string g_last_error;
extern std::atomic<uint64_t> g_launches;

int fail(int code, const char* fmt, ...);

#define RV_REQUIRE(cond, ...)                           \
  do {                                                  \
    if (!(cond)) return rv::fail(RV_E_INVALID, __VA_ARGS__); \
  } while (0)

#define RV_CUDA_OK(expr)                                                                  \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      (void)cudaGetLastError(); /* do not leave a sticky error for the next launch */     \
      return rv::fail(RV_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),  \
                      __FILE__, __LINE__);                                                \
    }                                                                                     \
  } while (0)

// call after every kernel launch
#define RV_LAUNCH_CHECK(name)                                                             \
  do {                                                                                    \
    rv::g_launches.fetch_add(1, std::memory_order_relaxed);                               \
    cudaError_t _e = cudaGetLastError();                                                  \
    if (_e != cudaSuccess)                                                                \
      return rv::fail(RV_E_CUDA, "launch of %s failed: %s", name, cudaGetErrorString(_e)); \
  } while (0)

template <typename T>
struct DT;
template <>
struct DT<float> {
  static constexpr int code = RV_F32;
};
template <>
struct DT<__half> {
  static constexpr int code = RV_F16;
};
template <>
struct DT<__nv_bfloat16> {
  static constexpr int code = RV_BF16;
};

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__device__ __forceinline__ T from_f(float v);
template <>
__device__ __forceinline__ float from_f<float>(float v) {
  return v;
}
template <>
__device__ __forceinline__ __half from_f<__half>(float v) {
  return __float2half_rn(v);
}
template <>
__device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) {
  return __float2bfloat16_rn(v);
}

__host__ __device__ __forceinline__ int dtype_size(int dt) { return dt == RV_F32 ? 4 : 2; }

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case RV_ACT_RELU: return fmaxf(v, 0.f);
    case RV_ACT_LRELU01: return v > 0.f ? v : 0.1f * v;
    case RV_ACT_LRELU02: return v > 0.f ? v : 0.2f * v;
    case RV_ACT_CLAMP3: return fminf(fmaxf(v, -3.f), 3.f);
    default: return v;
  }
}

// Keys cubic convolution weights, A = -0.75 (aten UpSampleBicubic2d; SURVEY appendix A).
__device__ __forceinline__ void cubic_weights(float t, float w[4]) {
  const float A = -0.75f;
  float x = t + 1.f;
  w[0] = ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A;
  x = t;
  w[1] = ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f;
  x = 1.f - t;
  w[2] = ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f;
  x = 2.f - t;
  w[3] = ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A;
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// dispatch a templated launcher on a runtime dtype code
#define RV_DISPATCH_DTYPE(dt, T, ...)                                  \
  switch (dt) {                                                        \
    case RV_F32: { using T = float; __VA_ARGS__; } break;              \
    case RV_F16: { using T = __half; __VA_ARGS__; } break;             \
    case RV_BF16: { using T = __nv_bfloat16; __VA_ARGS__; } break;     \
    default: return rv::fail(RV_E_INVALID, "bad dtype code %d", (int)(dt)); \
  }

inline unsigned cdiv(long long a, long long b) { return (unsigned)((a + b - 1) / b); }

}  // namespace rv
