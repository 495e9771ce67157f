// range.cu — range search / observers beyond plain min-max (SURVEY.md 8a Q2, Q7):
//
//   llmc_mse_range  `calib_algo: mse` (quant.py:145-203): per quantisation group, shrink the
//                   [min, max] range over `steps` = int(maxshrink * mse_grid) levels p = 1 - i/grid,
//                   quantise-dequantise the group with the qparams of (p*min, p*max) and keep the
//                   range with the smallest sum |q - x|^norm.  ONE launch replaces 80 x (~20 eager
//                   kernels over the whole weight).
//   llmc_histc      torch.histc for the static histogram observer (quant.py:462-522): counts of
//                   fp32(x) in `bins` equal bins over [lo, hi] (x == hi -> last bin, values outside
//                   are ignored), counted exactly in 32-bit integers and rounded once to fp32.
//
// The reference evaluates the mse search on `tensor.float()`: fp32 arithmetic throughout.  One
// quirk is preserved on purpose (SURVEY App. E style): `best_min_val, best_max_val = _min_val,
// _max_val` ALIAS the running range (quant.py:165), so an improvement at level i overwrites the
// base range and every later level shrinks from the already shrunk range (xmin = p * _min_val).
#include "common.cuh"

namespace llmc {
namespace rg {

constexpr int kThreads = 128;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One CTA per row (= one quantisation group of the reshaped tensor).  The row is staged in shared
// memory as fp32 when it fits (cols <= cache_cols), else re-read from global at every level.
template <int DT>
__global__ void __launch_bounds__(kThreads)
mse_range_kernel(const void* __restrict__ w, int64_t rows, int64_t cols, int sym, float qmin,
                 float qmax, int steps, float grid, float norm, int cache_cols,
                 float* __restrict__ min_out, float* __restrict__ max_out) {
  extern __shared__ float cache[];
  __shared__ float red[3][kThreads / 32];
  __shared__ float bc[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const int64_t base = row * cols;
    const bool cached = cols <= cache_cols;
    float mn = INFINITY, mx = -INFINITY;
    for (int64_t c = tid; c < cols; c += kThreads) {
      const float x = DType<DT>::load(w, base + c);
      if (cached) cache[c] = x;
      mn = fminf(mn, x);
      mx = fmaxf(mx, x);
    }
    mn = warp_min(mn);
    mx = warp_max(mx);
    if (lane == 0) { red[0][warp] = mn; red[1][warp] = mx; }
    __syncthreads();
    if (tid == 0) {
      float a = red[0][0], b = red[1][0];
      for (int i = 1; i < kThreads / 32; ++i) { a = fminf(a, red[0][i]); b = fmaxf(b, red[1][i]); }
      bc[0] = a; bc[1] = b;
    }
    __syncthreads();
    float cur_min = bc[0], cur_max = bc[1];     // the ALIASED running range (see header)
    float best = INFINITY;
    for (int i = 0; i < steps; ++i) {
      // p = 1 - i / mse_grid is a Python double; `p * tensor` multiplies in fp32 by fl32(p)
      const float p = static_cast<float>(1.0 - static_cast<double>(i) / static_cast<double>(grid));
      const float xmin = p * cur_min, xmax = p * cur_max;
      float s, z;
      if (sym) {                                           // quant.py:549-552
        s = fmaxf(fmaxf(fabsf(xmax), fabsf(xmin)), 1e-5f) / qmax;
        z = 0.f;
      } else {                                             // quant.py:553-558
        s = fmaxf(xmax - xmin, 1e-5f) / (qmax - qmin);
        z = fminf(fmaxf(qmin - rintf(xmin / s), qmin), qmax);
      }
      float err = 0.f;
      for (int64_t c = tid; c < cols; c += kThreads) {
        const float x = cached ? cache[c] : DType<DT>::load(w, base + c);
        const float q = fminf(fmaxf(rintf(x / s) + z, qmin), qmax);       // quant.py:699-708
        // dequant (q - z) * s, then q_tensor -= x: two roundings, never one FMA
        const float d = fabsf(fsub_rn(fmul_rn(fsub_rn(q, z), s), x));
        err += powf(d, norm);
      }
      err = warp_sum(err);
      if (lane == 0) red[2][warp] = err;
      __syncthreads();
      float tot = 0.f;
#pragma unroll
      for (int k = 0; k < kThreads / 32; ++k) tot += red[2][k];
      __syncthreads();
      if (tot < best) {                                    // `err < best`, strict (quant.py:190)
        best = tot;
        cur_min = xmin;
        cur_max = xmax;
      }
    }
    if (tid == 0) { min_out[row] = cur_min; max_out[row] = cur_max; }
    __syncthreads();
  }
}

template <int DT>
__global__ void __launch_bounds__(256)
histc_kernel(const void* __restrict__ x, int64_t n, float lo, float hi, int bins,
             unsigned int* __restrict__ counts) {
  extern __shared__ unsigned int local[];
  for (int b = threadIdx.x; b < bins; b += blockDim.x) local[b] = 0u;
  __syncthreads();
  const float width = hi - lo;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float v = DType<DT>::load(x, i);
    if (v >= lo && v <= hi) {
      // ATen's linear binning: pos = (v - lo) * bins / (hi - lo), the right edge goes to the last bin
      int b = static_cast<int>((v - lo) * static_cast<float>(bins) / width);
      if (b >= bins) b = bins - 1;
      atomicAdd(&local[b], 1u);
    }
  }
  __syncthreads();
  // exact integer totals (n < 2^32): an fp32 sum of the blocks' counts would round, in completion
  // order, once a bin passes 2^24
  for (int b = threadIdx.x; b < bins; b += blockDim.x)
    if (local[b]) atomicAdd(&counts[b], local[b]);
}

// hist holds the uint32 totals bit for bit; replace each by the count rounded once to fp32, like
// torch.histc's
__global__ void __launch_bounds__(256)
histc_finish_kernel(float* __restrict__ hist, int bins) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < bins) hist[b] = __uint2float_rn(__float_as_uint(hist[b]));
}

}  // namespace rg
}  // namespace llmc

using namespace llmc;

extern "C" int llmc_mse_range(const void* w, int64_t rows, int64_t cols, int dtype, int sym,
                              int qmin, int qmax, int steps, float grid, float norm,
                              float* min_out, float* max_out, void* stream) {
  LLMC_CHECK_ARG(w && min_out && max_out && rows > 0 && cols > 0, "mse_range: bad argument");
  LLMC_CHECK_ARG(steps >= 1 && grid > 0.f && qmax > qmin, "mse_range: bad grid / range");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  constexpr int kCacheCols = 24 * 1024;                      // 96 KB of fp32
  const int smem = (cols <= kCacheCols ? static_cast<int>(cols) : 0) * 4;
  for (auto kern : {rg::mse_range_kernel<LLMC_F32>, rg::mse_range_kernel<LLMC_F16>, rg::mse_range_kernel<LLMC_BF16>})
    if (int rc = opt_in_smem(kern, kCacheCols * 4)) return rc;
  const int64_t grid_x = rows < static_cast<int64_t>(kNumSMs) * 16 ? rows : static_cast<int64_t>(kNumSMs) * 16;
#define CALL(DT)                                                                                  \
  rg::mse_range_kernel<DT><<<(int)grid_x, rg::kThreads, smem, st>>>(                              \
      w, rows, cols, sym, (float)qmin, (float)qmax, steps, grid, norm, kCacheCols, min_out, max_out)
  LLMC_DISPATCH_DT("mse_range", dtype, CALL);
#undef CALL
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

extern "C" int llmc_histc(const void* x, int64_t n, int dtype, int bins, float lo, float hi,
                          float* hist, void* stream) {
  LLMC_CHECK_ARG((x || n == 0) && hist && n >= 0 && bins > 0 && bins <= 8192, "histc: bad argument");
  LLMC_CHECK_ARG(n <= 0xffffffffll, "histc: n = %lld exceeds the 32-bit bin counts", (long long)n);
  LLMC_CHECK_ARG(hi >= lo, "histc: max < min");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LLMC_CHECK_CUDA(cudaMemsetAsync(hist, 0, bins * sizeof(float), st));   // 0.0f == 0u
  if (n == 0) return LLMC_OK;
  if (hi == lo) { lo -= 1.f; hi += 1.f; }                   // torch.histc's degenerate-range rule
  int64_t blocks = (n + 255) / 256;
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  const int smem = bins * 4;
  unsigned int* counts = reinterpret_cast<unsigned int*>(hist);   // counted in place, then converted
#define CALL(DT) rg::histc_kernel<DT><<<(int)blocks, 256, smem, st>>>(x, n, lo, hi, bins, counts)
  LLMC_DISPATCH_DT("histc", dtype, CALL);
#undef CALL
  LLMC_CHECK_LAUNCH();
  rg::histc_finish_kernel<<<(bins + 255) / 256, 256, 0, st>>>(hist, bins);
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}
