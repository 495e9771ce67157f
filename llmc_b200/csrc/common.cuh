// common.cuh — shared device/host helpers for libllmc_b200.so (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

#include <mutex>

#include "../../include/llmc_b200.h"

namespace llmc {

constexpr int kNumSMs = 132;  // H100 SXM

// ---- error plumbing --------------------------------------------------------------------
void set_last_error(const char* fmt, ...);

#define LLMC_CHECK_ARG(cond, ...)              \
  do {                                         \
    if (!(cond)) {                             \
      ::llmc::set_last_error(__VA_ARGS__);     \
      return LLMC_EINVAL;                      \
    }                                          \
  } while (0)

#define LLMC_CHECK_CUDA(expr)                                                        \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      ::llmc::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,           \
                             cudaGetErrorString(_e));                                \
      return LLMC_ECUDA;                                                             \
    }                                                                                \
  } while (0)

// every kernel launch of this library is counted (llmc_b200_launch_count(), used by bench.py)
void count_launch(int n);
#define LLMC_CHECK_LAUNCH()                 \
  do {                                      \
    ::llmc::count_launch(1);                \
    LLMC_CHECK_CUDA(cudaGetLastError());    \
  } while (0)

// Function attributes (opt-in dynamic shared memory) are per DEVICE: run `body` the first time
// this call site is reached on each device (a process normally drives one GPU, but nothing here
// should break when it drives several).  `body` may `return` an error code.
#define LLMC_ONCE_PER_DEVICE(body)                                   \
  do {                                                               \
    static std::mutex once_mutex_;                                   \
    static uint64_t once_mask_ = 0;                                  \
    int once_dev_ = 0;                                               \
    if (cudaGetDevice(&once_dev_) != cudaSuccess) once_dev_ = 0;     \
    std::lock_guard<std::mutex> once_guard_(once_mutex_);            \
    const uint64_t once_bit_ = 1ull << (once_dev_ & 63);             \
    if (!(once_mask_ & once_bit_)) {                                 \
      body;                                                          \
      once_mask_ |= once_bit_;                                       \
    }                                                                \
  } while (0)

// ---- dtype helpers ---------------------------------------------------------------------
// "T-faithful" arithmetic: torch eager evaluates every elementwise op on fp16/bf16 tensors
// in fp32 and rounds the result once to T.  rT<T>(x) is that rounding (identity for fp32).
template <int DT> struct DType;
template <> struct DType<LLMC_F32> {
  using type = float;
  static constexpr int bytes = 4;
  __device__ __forceinline__ static float rT(float x) { return x; }
  __device__ __forceinline__ static float load(const void* p, int64_t i) {
    return reinterpret_cast<const float*>(p)[i];
  }
  __device__ __forceinline__ static void store(void* p, int64_t i, float v) {
    reinterpret_cast<float*>(p)[i] = v;
  }
};
template <> struct DType<LLMC_F16> {
  using type = __half;
  static constexpr int bytes = 2;
  __device__ __forceinline__ static float rT(float x) {
    return __half2float(__float2half_rn(x));
  }
  __device__ __forceinline__ static float load(const void* p, int64_t i) {
    return __half2float(reinterpret_cast<const __half*>(p)[i]);
  }
  __device__ __forceinline__ static void store(void* p, int64_t i, float v) {
    reinterpret_cast<__half*>(p)[i] = __float2half_rn(v);
  }
};
template <> struct DType<LLMC_BF16> {
  using type = __nv_bfloat16;
  static constexpr int bytes = 2;
  __device__ __forceinline__ static float rT(float x) {
    return __bfloat162float(__float2bfloat16_rn(x));
  }
  __device__ __forceinline__ static float load(const void* p, int64_t i) {
    return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
  }
  __device__ __forceinline__ static void store(void* p, int64_t i, float v) {
    reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
  }
};

// 8 consecutive elements <-> 8 floats, vectorised (16 B for 2-byte types, 2x16 B for fp32).
template <int DT>
__device__ __forceinline__ void load8(const void* base, int64_t idx, float (&v)[8]) {
  if constexpr (DT == LLMC_F32) {
    const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + idx);
    float4 a = __ldg(p), b = __ldg(p + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    const uint4* p = reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(base) + idx);
    uint4 u = __ldg(p);
    uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if constexpr (DT == LLMC_BF16) {
        v[2 * i] = __uint_as_float(w[i] << 16);
        v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
      } else {
        __half2 h = *reinterpret_cast<__half2*>(&w[i]);
        float2 f = __half22float2(h);
        v[2 * i] = f.x;
        v[2 * i + 1] = f.y;
      }
    }
  }
}

template <int DT>
__device__ __forceinline__ void store8(void* base, int64_t idx, const float (&v)[8]) {
  if constexpr (DT == LLMC_F32) {
    float4* p = reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + idx);
    p[0] = make_float4(v[0], v[1], v[2], v[3]);
    p[1] = make_float4(v[4], v[5], v[6], v[7]);
  } else {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if constexpr (DT == LLMC_BF16) {
        __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
        w[i] = *reinterpret_cast<uint32_t*>(&h);
      } else {
        __half2 h = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
        w[i] = *reinterpret_cast<uint32_t*>(&h);
      }
    }
    *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(base) + idx) =
        make_uint4(w[0], w[1], w[2], w[3]);
  }
}

__device__ __forceinline__ float warp_max(float v, int width = 32) {
  for (int o = width >> 1; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_min(float v, int width = 32) {
  for (int o = width >> 1; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Non-template wrappers: the host pass of nvcc does not see the __f*_rn intrinsics, so calling
// them directly from templates fails two-phase lookup.
__device__ __forceinline__ float fdiv_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float fmul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fma_rn(float a, float b, float c) { return __fmaf_rn(a, b, c); }

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace llmc
