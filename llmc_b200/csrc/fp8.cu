// fp8.cu — FloatQuantizer (llmc/compression/quantization/quant.py:963-1229) for e4m3 / e5m2 with
// `use_qtorch: True`: symmetric scale = absmax / finfo.max, y = float_quantize(x / s) * s.
//
// PARITY UNPINNED: the rounding itself lives in the third-party `qtorch.quant.float_quantize`
// (unpinned in requirements/runtime.txt:29, absent from /root/reference and from this image;
// SURVEY.md §8c).  It is restated as IEEE round-to-nearest-even onto the e4m3fn / e5m2 grid with
// saturation to the finite maximum — the hardware `cvt.rn.satfinite.e4m3x2.f32` — which agrees
// with any correct nearest rounding for |x / s| <= finfo.max (always true for weights, since
// s = absmax / finfo.max).  Everything around it follows the reference's dtype flow: x / s is
// rounded to the tensor dtype T (quant.py:1063), the grid value is fp32 (the `.to(org_dtype)` on
// :1069 is a discarded no-op), dequant multiplies fp32 * T -> fp32 (:1075) and the result is cast
// back to T by the caller (:1154).
#include <cuda_fp8.h>

#include "common.cuh"
#include "fp8_math.cuh"

namespace llmc {

struct Fp8Args {
  const void* w;
  int64_t rows, cols, group, ng;
  int e5m2;
  float fmax;             // finfo.max: 448 / 57344
  void* scales;           // dynamic: out [rows*ng] T ; static: in
  int q_row_stride;       // static: ng, or 0 for one per-tensor scale
  int scale_f32;          // static per-tensor: scale is fp32 (torch CPU scalar-operand path)
  int out_mode;           // 0 none, 1 QDQ (T), 2 fp8 bytes
  void* out;
};

// The absmax propagates NaN, as the reference's amax / max / clamp do (quant.py:137-140, 550-551):
// a NaN anywhere in a group makes its scale, and so every output of the group, NaN.  fmaxf would
// drop it and quantise the rest of the group as if it were absent.
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float warp_max_nan(float v) {
  for (int o = 16; o > 0; o >>= 1) v = fmax_nan(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <int DT>
__device__ __forceinline__ void fp8_emit(const Fp8Args& a, int64_t idx, float x, float s, bool scalar) {
  // quant.py:1062: scales[scales == 0] = 1
  const float sq = (s == 0.f) ? 1.f : s;
  // quant.py:1063: y = x / s + z with z = 0.0 — the addition turns a -0.0 quotient into +0.0
  const float v = fadd_rn(DType<DT>::rT(fdiv_rn(x, sq)), 0.f);
  (void)scalar;
  if (a.out_mode == 2) {
    reinterpret_cast<uint8_t*>(a.out)[idx] = fp8_bits(v, a.e5m2);
  } else {
    const float q = fp8_round(v, a.e5m2);
    DType<DT>::store(a.out, idx, fmul_rn(q, sq));       // fp32 product, one rounding to T
  }
}

// one CTA per (row, group): absmax -> scale -> quantise (second pass from L1/L2)
template <int DT>
__global__ void __launch_bounds__(256)
fp8_dynamic_kernel(Fp8Args a) {
  __shared__ float red[8];
  __shared__ float s_sh;
  const int64_t total = a.rows * a.ng;
  for (int64_t g = blockIdx.x; g < total; g += gridDim.x) {
    const int64_t r = g / a.ng, j = g - r * a.ng;
    const int64_t base = r * a.cols + j * a.group;
    float mx = 0.f;
    for (int64_t i = threadIdx.x; i < a.group; i += blockDim.x)
      mx = fmax_nan(mx, fabsf(DType<DT>::load(a.w, base + i)));
    mx = warp_max_nan(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
      float v = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
      v = warp_max_nan(v);
      if (threadIdx.x == 0) {
        // quant.py:549-553: abs_max.clamp(min=1e-5) / qmax
        const float am = fmax_nan(v, DType<DT>::rT(1e-5f));
        s_sh = DType<DT>::rT(fdiv_rn(am, a.fmax));
        DType<DT>::store(a.scales, g, s_sh);
      }
    }
    __syncthreads();
    const float s = s_sh;
    if (a.out_mode != 0)
      for (int64_t i = threadIdx.x; i < a.group; i += blockDim.x)
        fp8_emit<DT>(a, base + i, DType<DT>::load(a.w, base + i), s, false);
    __syncthreads();
  }
}

template <int DT>
__global__ void __launch_bounds__(256)
fp8_static_kernel(Fp8Args a) {
  const int64_t total = a.rows * a.cols;
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = idx / a.cols, c = idx - r * a.cols;
    const int64_t qi = r * a.q_row_stride + (a.q_row_stride ? c / a.group : 0);
    const float s = a.scale_f32 ? reinterpret_cast<const float*>(a.scales)[qi]
                                : DType<DT>::load(a.scales, qi);
    fp8_emit<DT>(a, idx, DType<DT>::load(a.w, idx), s, a.scale_f32 != 0);
  }
}

}  // namespace llmc

using namespace llmc;

extern "C" int llmc_fp8_quant(const void* w, int64_t rows, int64_t cols, int dtype, int64_t group,
                              int e5m2, int dynamic, void* scales, int q_row_stride, int scale_f32,
                              int out_mode, void* out, void* stream) {
  LLMC_CHECK_ARG(rows >= 0 && cols >= 0, "fp8_quant: bad shape");
  if (rows == 0 || cols == 0) return LLMC_OK;
  LLMC_CHECK_ARG(w && scales, "fp8_quant: null pointer");
  LLMC_CHECK_ARG(group > 0 && cols % group == 0, "fp8_quant: cols %% group != 0");
  LLMC_CHECK_ARG(out_mode >= 0 && out_mode <= 2 && (out_mode == 0 || out), "fp8_quant: bad out_mode / out");
  LLMC_CHECK_ARG(dtype >= LLMC_F32 && dtype <= LLMC_BF16, "fp8_quant: bad dtype");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Fp8Args a{};
  a.w = w; a.rows = rows; a.cols = cols; a.group = group; a.ng = cols / group;
  a.e5m2 = e5m2; a.fmax = e5m2 ? 57344.f : 448.f;
  a.scales = scales; a.q_row_stride = q_row_stride; a.scale_f32 = scale_f32;
  a.out_mode = out_mode; a.out = out;
  if (dynamic) {
    int64_t blocks = rows * a.ng;
    if (blocks > kNumSMs * 32) blocks = kNumSMs * 32;
#define CALL(DT) fp8_dynamic_kernel<DT><<<(int)blocks, 256, 0, st>>>(a)
    LLMC_DISPATCH_DT("fp8_quant", dtype, CALL);
#undef CALL
  } else {
    LLMC_CHECK_ARG(out_mode != 0, "fp8_quant: static mode needs an output");
    int64_t blocks = (rows * cols + 255) / 256;
    if (blocks > kNumSMs * 32) blocks = kNumSMs * 32;
#define CALL(DT) fp8_static_kernel<DT><<<(int)blocks, 256, 0, st>>>(a)
    LLMC_DISPATCH_DT("fp8_quant", dtype, CALL);
#undef CALL
  }
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

// ---- 128 x 128 block FP8 (DeepSeek-V3 / R1 checkpoints; SURVEY 8a Q10) -----------------------------
// weight_cast_to_fp8 (quant.py:32-43) = FloatQuantizer(e4m3, per_block).real_quant_weight_dynamic:
//   reshape to [M/bs, bs, N/bs, bs] (zero padded), range = abs().float() amin/amax over dims (1, 3)
//   (quant.py:137-139), scale = max(absmax, 1e-5) / 448 in fp32, q = fp8(x.float() / scale) — the
//   fp32 scale promotes the division to fp32 (no rounding to the tensor dtype here).
// weight_cast_to_bf16 (quant.py:18-29): (w_fp8.float() - 0) * scale_inv -> bf16.
// One CTA per block; the block is read once for the absmax and once (L1/L2) for the conversion.
namespace llmc {

template <int DT>
__global__ void __launch_bounds__(256)
fp8_block_quant_kernel(const void* __restrict__ w, int64_t M, int64_t N, int bs, int e5m2, float fmax,
                       float* __restrict__ scales, int out_mode, void* __restrict__ out) {
  __shared__ float red[8];
  __shared__ float s_sh;
  const int64_t nbn = (N + bs - 1) / bs, nbm = (M + bs - 1) / bs;
  for (int64_t b = blockIdx.x; b < nbm * nbn; b += gridDim.x) {
    const int64_t bi = b / nbn, bj = b - bi * nbn;
    const int64_t r0 = bi * bs, c0 = bj * bs;
    float mx = 0.f;
    for (int e = threadIdx.x; e < bs * bs; e += blockDim.x) {
      const int64_t r = r0 + e / bs, c = c0 + e % bs;
      if (r < M && c < N) mx = fmax_nan(mx, fabsf(DType<DT>::load(w, r * N + c)));
    }
    mx = warp_max_nan(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
      float v = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
      v = warp_max_nan(v);
      if (threadIdx.x == 0) {
        s_sh = fdiv_rn(fmax_nan(v, 1e-5f), fmax);
        scales[b] = s_sh;
      }
    }
    __syncthreads();
    const float s = s_sh;
    if (out_mode != 0) {
      for (int e = threadIdx.x; e < bs * bs; e += blockDim.x) {
        const int64_t r = r0 + e / bs, c = c0 + e % bs;
        if (r < M && c < N) {
          const float v = fadd_rn(fdiv_rn(DType<DT>::load(w, r * N + c), s), 0.f);   // x / s + 0.0 (:1063)
          if (out_mode == 2) reinterpret_cast<uint8_t*>(out)[r * N + c] = fp8_bits(v, e5m2);
          else DType<DT>::store(out, r * N + c, fmul_rn(fp8_round(v, e5m2), s));
        }
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256)
fp8_block_dequant_kernel(const uint8_t* __restrict__ w, int64_t M, int64_t N, int bs, int e5m2,
                         const float* __restrict__ scale_inv, __nv_bfloat16* __restrict__ out) {
  const int64_t nbn = (N + bs - 1) / bs;
  const int64_t total = M * N;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / N, c = i - r * N;
    const float s = scale_inv[(r / bs) * nbn + c / bs];
    const float q = __half2float(__half(__nv_cvt_fp8_to_halfraw(w[i], e5m2 ? __NV_E5M2 : __NV_E4M3)));
    out[i] = __float2bfloat16_rn(fmul_rn(q, s));
  }
}

}  // namespace llmc

extern "C" int llmc_fp8_block_quant(const void* w, int64_t M, int64_t N, int dtype, int block, int e5m2,
                                    float* scales, int out_mode, void* out, void* stream) {
  LLMC_CHECK_ARG(w && scales && M > 0 && N > 0 && block > 0 && block <= 256, "fp8_block_quant: bad argument");
  LLMC_CHECK_ARG(out_mode >= 0 && out_mode <= 2 && (out_mode == 0 || out), "fp8_block_quant: bad out_mode / out");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t nb = ((M + block - 1) / block) * ((N + block - 1) / block);
  const int grid = static_cast<int>(nb < kNumSMs * 16 ? nb : kNumSMs * 16);
  const float fmax = e5m2 ? 57344.f : 448.f;
#define CALL(DT) fp8_block_quant_kernel<DT><<<grid, 256, 0, st>>>(w, M, N, block, e5m2, fmax, scales, out_mode, out)
  LLMC_DISPATCH_DT("fp8_block_quant", dtype, CALL);
#undef CALL
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

extern "C" int llmc_fp8_block_dequant(const void* w_fp8, int64_t M, int64_t N, int block, int e5m2,
                                      const float* scale_inv, void* out_bf16, void* stream) {
  LLMC_CHECK_ARG(w_fp8 && scale_inv && out_bf16 && M > 0 && N > 0 && block > 0, "fp8_block_dequant: bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t blocks = (M * N + 255) / 256;
  if (blocks > kNumSMs * 32) blocks = kNumSMs * 32;
  fp8_block_dequant_kernel<<<(int)blocks, 256, 0, st>>>(reinterpret_cast<const uint8_t*>(w_fp8), M, N, block, e5m2,
                                                        scale_inv, reinterpret_cast<__nv_bfloat16*>(out_bf16));
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

// ---- 1 x 128 activation quantiser: act_quant (kernel.py:7-53), the input side of fp8_gemm ----------
// Per contiguous group of 128 elements, in fp32: s = max|x| / 448, y = e4m3(x / s).  The reference's
// Triton kernel compiles both divisions on sm_90 to the approximate `div.full.f32` (<= 2 ulp), not
// IEEE div.rn, the max to `max.f32` and the cast to `cvt.rn.satfinite.e4m3x2.f32`; the same
// instructions are issued here, so scales and codes match the reference's bit for bit on the same
// hardware.  Reproduced quirk: unlike weight_cast_to_fp8 there is no clamp(min=1e-5), so an
// all-zero group gets s = 0 and NaN codes (0 / 0), which fp8_gemm spreads over its output row.
// max.f32 returns the other operand when one is NaN, so a NaN element does not reach the scale
// (its own code is NaN) unless the whole group is NaN; an infinite element makes s = inf, the
// group's finite codes +-0 and its infinite ones NaN.
// Half a warp per group, 8 elements per lane: one 16-byte load (two for fp32), one 8-byte store.
namespace llmc {

__device__ __forceinline__ float div_full(float a, float b) {
  float r;
  asm("div.full.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// two e4m3 codes in one 16-bit word, `lo` in the low byte (the lower address)
__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

template <int DT>
__global__ void __launch_bounds__(256)
fp8_act_quant_kernel(const void* __restrict__ x, int64_t groups, uint8_t* __restrict__ y,
                     float* __restrict__ scales) {
  // the loop bound is uniform across a warp (both halves shuffle together)
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  const int half = (threadIdx.x >> 4) & 1, sub = threadIdx.x & 15;
  for (int64_t g0 = 2 * warp; g0 < groups; g0 += 2 * nwarps) {
    const int64_t g = g0 + half;
    const bool live = g < groups;
    const int64_t base = g * 128 + sub * 8;
    float v[8];
    if (live) load8<DT>(x, base, v);
    else {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = 0.f;
    }
    // seeded with an element, not 0, so that an all-NaN group keeps a NaN max like the reference's
    float mx = fabsf(v[0]);
#pragma unroll
    for (int i = 1; i < 8; ++i) mx = fmaxf(mx, fabsf(v[i]));
    mx = warp_max(mx, 16);
    const float s = div_full(mx, 448.f);
    if (!live) continue;
    uint32_t w[2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
      w[h] = e4m3x2(div_full(v[4 * h], s), div_full(v[4 * h + 1], s)) |
             (e4m3x2(div_full(v[4 * h + 2], s), div_full(v[4 * h + 3], s)) << 16);
    *reinterpret_cast<uint2*>(y + base) = make_uint2(w[0], w[1]);
    if (sub == 0) scales[g] = s;
  }
}

}  // namespace llmc

extern "C" int llmc_fp8_act_quant(const void* x, int64_t rows, int64_t K, int dtype, void* y,
                                  float* scales, void* stream) {
  LLMC_CHECK_ARG(rows >= 0 && K >= 1, "fp8_act_quant: bad shape rows=%lld K=%lld", (long long)rows,
                 (long long)K);
  LLMC_CHECK_ARG(K % 128 == 0, "fp8_act_quant: K=%lld must be a multiple of 128", (long long)K);
  LLMC_CHECK_ARG(dtype >= LLMC_F32 && dtype <= LLMC_BF16, "fp8_act_quant: bad dtype %d", dtype);
  if (rows == 0) return LLMC_OK;
  LLMC_CHECK_ARG(x && y && scales, "fp8_act_quant: null pointer");
  if (!aligned16(x) || !aligned16(y)) {
    set_last_error("fp8_act_quant: x and y must be 16-byte aligned");
    return LLMC_EALIGN;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t groups = rows * (K / 128);
  int64_t blocks = (groups + 15) / 16;                 // 16 groups per 256-thread block
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
#define CALL(DT) fp8_act_quant_kernel<DT><<<(int)blocks, 256, 0, st>>>(x, groups, reinterpret_cast<uint8_t*>(y), scales)
  LLMC_DISPATCH_DT("fp8_act_quant", dtype, CALL);
#undef CALL
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}
