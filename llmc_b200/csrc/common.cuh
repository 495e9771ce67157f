// common.cuh — shared device/host helpers for libllmc_b200.so (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

#include <initializer_list>
#include <mutex>
#include <vector>

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

// Opts `kernel` in to `bytes` of dynamic shared memory beyond the default 48 KB.  Function
// attributes are per DEVICE, so this sets the attribute the first time each (device, kernel) is
// seen (a process normally drives one GPU, but nothing here should break when it drives several);
// `bytes` is the most any launch of the kernel uses.
int opt_in_smem(const void* kernel, int bytes);
template <class... P>
int opt_in_smem(void (*kernel)(P...), int bytes) {
  return opt_in_smem(reinterpret_cast<const void*>(kernel), bytes);
}

// A persistent kernel's CTAs take its `count` units of work in turn (u = blockIdx.x; u +=
// gridDim.x).  launch_persistent runs it on one CTA per SM, or on fewer when there are fewer units;
// cta_per_unit runs one CTA per unit instead (see tf32x3_update).
struct Units {
  int count;
  bool cta_per_unit;
  Units(int n, bool one_cta_each = false) : count(n), cta_per_unit(one_cta_each) {}
};
template <class... P, class... A>
int launch_persistent(void (*kernel)(P...), Units units, int threads, int smem, cudaStream_t st,
                      A... args) {
  if (int rc = opt_in_smem(kernel, smem)) return rc;
  const int grid = (units.cta_per_unit || units.count < kNumSMs) ? units.count : kNumSMs;
  kernel<<<grid, threads, smem, st>>>(args...);
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

// ---- side streams ------------------------------------------------------------------------
// The look-ahead schedules of the blocked Cholesky (chol.cu) and of the GPTQ / SpQR sweep
// (gptq.cu) run a latency-bound chain and the bulk updates off that chain on side streams of
// different priorities.  One set per device, created on first use, serves both.  Sharing it is
// sound only because every call forks from the caller's stream before its first side-stream
// launch and joins every side stream it used back into the caller's stream before it returns: its
// side-stream work starts after everything enqueued on the caller's stream before the call and
// ends before anything enqueued after it, so calls never overlap on a side stream.  Records and
// waits take effect at enqueue time, so one host thread per device is assumed, like everywhere in
// this library.
enum SideStream {
  kChain,          // greatest priority
  kInverse,        // the next priority: the Cholesky's inverse chain
  kBulk,           // least priority (the default priority of a stream)
  kInverseBulk,    // least priority
  kNumSideStreams
};
struct SideStreams {
  cudaStream_t stream[kNumSideStreams];
  cudaEvent_t fork_ev, join_ev[kNumSideStreams];
  std::vector<cudaEvent_t> ev[4];   // grow-only; each array serves one purpose within a call
  // `to` wait for everything enqueued on st so far
  int fork(cudaStream_t st, std::initializer_list<SideStream> to);
  // st waits for everything enqueued on `from` so far
  int join(cudaStream_t st, std::initializer_list<SideStream> from);
};
// This device's side streams, with at least n_events events in every ev[] array.
int side_streams(int64_t n_events, SideStreams** out);

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

// Run-time dtype versions of DType<>::load / store and store8 (an unknown dtype means bf16).
__device__ __forceinline__ float load_as(int dt, const void* p, int64_t i) {
  if (dt == LLMC_F32) return DType<LLMC_F32>::load(p, i);
  if (dt == LLMC_F16) return DType<LLMC_F16>::load(p, i);
  return DType<LLMC_BF16>::load(p, i);
}
__device__ __forceinline__ void store_as(int dt, void* p, int64_t i, float v) {
  if (dt == LLMC_F32) DType<LLMC_F32>::store(p, i, v);
  else if (dt == LLMC_F16) DType<LLMC_F16>::store(p, i, v);
  else DType<LLMC_BF16>::store(p, i, v);
}

// Host side: run CALL(DT) with DT the compile-time constant of the run-time dtype `dt`; an unknown
// dtype makes the enclosing entry point fail with LLMC_EINVAL.
#define LLMC_DISPATCH_DT(what, dt, CALL)                                            \
  do {                                                                              \
    if ((dt) == LLMC_F32) { CALL(LLMC_F32); }                                       \
    else if ((dt) == LLMC_F16) { CALL(LLMC_F16); }                                  \
    else if ((dt) == LLMC_BF16) { CALL(LLMC_BF16); }                                \
    else { ::llmc::set_last_error("%s: bad dtype %d", what, (dt)); return LLMC_EINVAL; } \
  } while (0)

// ---- 16-bit pairs ----------------------------------------------------------------------
// Two fp16 / bf16 (DT) values in one 32-bit word, the first in the low half.  Packing rounds each
// float once (cvt.rn.{f16,bf16}x2); widening is exact.
template <int DT>
__device__ __forceinline__ uint32_t pack_pair(float a, float b) {
  if constexpr (DT == LLMC_BF16) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  } else {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  }
}
// a lone 16-bit value (a bias element, a qparam in the activation dtype)
template <int DT>
__device__ __forceinline__ float widen16(uint16_t x) {
  if constexpr (DT == LLMC_BF16) return __uint_as_float(static_cast<uint32_t>(x) << 16);
  else return __half2float(__ushort_as_half(x));
}
template <int DT>
__device__ __forceinline__ float pair_lo(uint32_t w) {
  if constexpr (DT == LLMC_BF16) return __uint_as_float(w << 16);
  else return widen16<DT>(static_cast<uint16_t>(w & 0xffffu));
}
template <int DT>
__device__ __forceinline__ float pair_hi(uint32_t w) {
  if constexpr (DT == LLMC_BF16) return __uint_as_float(w & 0xffff0000u);
  else return widen16<DT>(static_cast<uint16_t>(w >> 16));
}

// 8 consecutive elements <-> 8 floats, vectorised (16 B for 2-byte types, 2x16 B for fp32).
// load8 writes its widening out rather than calling pair_lo / pair_hi: with the calls, ptxas
// allocates registers differently in callers (an 8-byte spill in quant_dynamic_warp_kernel<bf16>,
// three more registers in rope_kernel).
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
    for (int i = 0; i < 4; ++i) w[i] = pack_pair<DT>(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(base) + idx) =
        make_uint4(w[0], w[1], w[2], w[3]);
  }
}

__device__ __forceinline__ void store8_as(int dt, void* base, int64_t idx, const float (&v)[8]) {
  if (dt == LLMC_F32) store8<LLMC_F32>(base, idx, v);
  else if (dt == LLMC_F16) store8<LLMC_F16>(base, idx, v);
  else store8<LLMC_BF16>(base, idx, v);
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

// F.silu in fp32 (IEEE division), shared by llmc_silu_mul and the SwiGLU epilogue of the forward
// GEMM, which must agree bit for bit.
__device__ __forceinline__ float silu_f32(float x) { return x / (1.0f + expf(-x)); }
// F.sigmoid in fp32 (torch's sigmoid kernel: 1 / (1 + exp(-x)), IEEE division).
__device__ __forceinline__ float sigmoid_f32(float x) { return 1.0f / (1.0f + expf(-x)); }

// One element of F.silu(gate) * up on DT tensors: silu in fp32 rounded to DT, the product in fp32,
// which the caller's store rounds.  kRoundInputs: g and u are a GEMM epilogue's fp32 accumulators,
// rounded to DT first; else they are DT values already (llmc_silu_mul).  llmc_silu_mul and every
// SwiGLU epilogue compute it here, so they agree bit for bit.
template <int DT, bool kRoundInputs>
__device__ __forceinline__ float silu_mul_f32(float g, float u) {
  using T = DType<DT>;
  if constexpr (kRoundInputs) return fmul_rn(T::rT(silu_f32(T::rT(g))), T::rT(u));
  else return fmul_rn(T::rT(silu_f32(g)), u);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace llmc
