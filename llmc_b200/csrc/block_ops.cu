// block_ops.cu — the elementwise glue of a Llama-shaped decoder block during calibration
// (F2 of SURVEY.md §8(a): block_forward, base_blockwise_quantization.py:367-390).  The reference
// runs the HF module, i.e. ~12 eager kernels per norm / rotary / activation with fp32
// temporaries, i.e. several extra HBM round trips of the activations per op.
// Each op here is one pass.  Semantics are those of the HF modules the reference wraps:
//   rmsnorm : LlamaRMSNorm.forward  — x.float(); x * rsqrt(mean(x^2) + eps); weight * x.to(T)
//   rope    : apply_rotary_pos_emb  — q * cos + rotate_half(q) * sin, evaluated in T
//   silu_mul: LlamaMLP              — act_fn(gate) * up, silu in fp32 rounded to T, product in T
#include "common.cuh"

namespace llmc {

template <int DT>
__global__ void __launch_bounds__(256)
rmsnorm_kernel(const void* __restrict__ x, const void* __restrict__ w, void* __restrict__ y,
               int64_t rows, int64_t cols, float eps) {
  __shared__ float red[8];
  __shared__ float inv_sh;
  const int chunks = static_cast<int>(cols >> 3);
  for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
    float acc = 0.f;
    for (int ch = threadIdx.x; ch < chunks; ch += blockDim.x) {
      float v[8];
      load8<DT>(x, r * cols + ch * 8, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc = fmaf(v[i], v[i], acc);
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
      float t = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
      t = warp_sum(t);
      if (threadIdx.x == 0) inv_sh = rsqrtf(t / static_cast<float>(cols) + eps);
    }
    __syncthreads();
    const float inv = inv_sh;
    for (int ch = threadIdx.x; ch < chunks; ch += blockDim.x) {
      float v[8], g[8], o[8];
      load8<DT>(x, r * cols + ch * 8, v);       // second pass: L1/L2 hit
      load8<DT>(w, ch * 8, g);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = fmul_rn(g[i], DType<DT>::rT(fmul_rn(v[i], inv)));
      store8<DT>(y, r * cols + ch * 8, o);
    }
    __syncthreads();
  }
}

// x: [B, S, H, D] (tokens-major, as produced by the q/k projections), rotated in place.
// cos/sin: [S, D].  One thread per (token, head, 8-wide chunk of the first half) handles the pair
// (i, i + D/2):  out_i = x_i*cos_i - x_{i+D/2}*sin_i ;  out_{i+D/2} = x_{i+D/2}*cos_{i+D/2} + x_i*sin_{i+D/2}
template <int DT>
__global__ void __launch_bounds__(256)
rope_kernel(void* __restrict__ x, const void* __restrict__ cosv, const void* __restrict__ sinv,
            int64_t B, int64_t S, int64_t H, int64_t D) {
  const int64_t half_chunks = D >> 4;                   // 8-wide chunks in half a head
  const int64_t total = B * S * H * half_chunks;
  for (int64_t u = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < total;
       u += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t ch = u % half_chunks;
    const int64_t t = u / half_chunks;                 // (b, s, h) flattened
    const int64_t s = (t / H) % S;
    const int64_t base = t * D + ch * 8;
    float a[8], b[8], c1[8], s1[8], c2[8], s2[8], oa[8], ob[8];
    load8<DT>(x, base, a);
    load8<DT>(x, base + (D >> 1), b);
    load8<DT>(cosv, s * D + ch * 8, c1);
    load8<DT>(sinv, s * D + ch * 8, s1);
    load8<DT>(cosv, s * D + (D >> 1) + ch * 8, c2);
    load8<DT>(sinv, s * D + (D >> 1) + ch * 8, s2);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      using T = DType<DT>;
      // torch: (q * cos) + (rotate_half(q) * sin), each op rounded to T; rotate_half = (-x2, x1)
      oa[i] = T::rT(fadd_rn(T::rT(fmul_rn(a[i], c1[i])), T::rT(fmul_rn(-b[i], s1[i]))));
      ob[i] = T::rT(fadd_rn(T::rT(fmul_rn(b[i], c2[i])), T::rT(fmul_rn(a[i], s2[i]))));
    }
    store8<DT>(x, base, oa);
    store8<DT>(x, base + (D >> 1), ob);
  }
}

template <int DT>
__global__ void __launch_bounds__(256)
silu_mul_kernel(const void* __restrict__ g, const void* __restrict__ u, void* __restrict__ y,
                int64_t n8) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float a[8], b[8], o[8];
    load8<DT>(g, i << 3, a);
    load8<DT>(u, i << 3, b);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = silu_mul_f32<DT, false>(a[k], b[k]);     // store8 rounds
    store8<DT>(y, i << 3, o);
  }
}

// y = a + b (residual), T-faithful
template <int DT>
__global__ void __launch_bounds__(256)
add_kernel(const void* __restrict__ a, const void* __restrict__ b, void* __restrict__ y, int64_t n8) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float va[8], vb[8], o[8];
    load8<DT>(a, i << 3, va);
    load8<DT>(b, i << 3, vb);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = fadd_rn(va[k], vb[k]);
    store8<DT>(y, i << 3, o);
  }
}

}  // namespace llmc

using namespace llmc;

extern "C" int llmc_rmsnorm(const void* x, const void* weight, void* y, int64_t rows, int64_t cols,
                            float eps, int dtype, void* stream) {
  LLMC_CHECK_ARG(x && weight && y && rows >= 0 && cols > 0, "rmsnorm: bad argument");
  if (rows == 0) return LLMC_OK;
  LLMC_CHECK_ARG(cols % 8 == 0 && aligned16(x) && aligned16(y) && aligned16(weight),
                 "rmsnorm: cols %% 8 == 0 and 16-byte alignment required");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t blocks = rows < kNumSMs * 16 ? rows : kNumSMs * 16;
#define CALL(DT) rmsnorm_kernel<DT><<<(int)blocks, 256, 0, st>>>(x, weight, y, rows, cols, eps); LLMC_CHECK_LAUNCH()
  LLMC_DISPATCH_DT("rmsnorm", dtype, CALL);
#undef CALL
  return LLMC_OK;
}

extern "C" int llmc_rope(void* x, const void* cosv, const void* sinv, int64_t B, int64_t S, int64_t H,
                         int64_t D, int dtype, void* stream) {
  LLMC_CHECK_ARG(x && cosv && sinv && B >= 0 && S > 0 && H > 0 && D > 0, "rope: bad argument");
  if (B == 0) return LLMC_OK;
  LLMC_CHECK_ARG(D % 16 == 0 && aligned16(x) && aligned16(cosv) && aligned16(sinv),
                 "rope: head_dim %% 16 == 0 and 16-byte alignment required");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t total = B * S * H * (D >> 4);
  int64_t blocks = (total + 255) / 256;
  if (blocks > kNumSMs * 32) blocks = kNumSMs * 32;
#define CALL(DT) rope_kernel<DT><<<(int)blocks, 256, 0, st>>>(x, cosv, sinv, B, S, H, D); LLMC_CHECK_LAUNCH()
  LLMC_DISPATCH_DT("rope", dtype, CALL);
#undef CALL
  return LLMC_OK;
}

extern "C" int llmc_silu_mul(const void* gate, const void* up, void* y, int64_t n, int dtype,
                             void* stream) {
  LLMC_CHECK_ARG(gate && up && y && n >= 0, "silu_mul: bad argument");
  if (n == 0) return LLMC_OK;
  LLMC_CHECK_ARG(n % 8 == 0 && aligned16(gate) && aligned16(up) && aligned16(y),
                 "silu_mul: n %% 8 == 0 and 16-byte alignment required");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t blocks = ((n >> 3) + 255) / 256;
  if (blocks > kNumSMs * 32) blocks = kNumSMs * 32;
#define CALL(DT) silu_mul_kernel<DT><<<(int)blocks, 256, 0, st>>>(gate, up, y, n >> 3); LLMC_CHECK_LAUNCH()
  LLMC_DISPATCH_DT("silu_mul", dtype, CALL);
#undef CALL
  return LLMC_OK;
}

extern "C" int llmc_add(const void* a, const void* b, void* y, int64_t n, int dtype, void* stream) {
  LLMC_CHECK_ARG(a && b && y && n >= 0, "add: bad argument");
  if (n == 0) return LLMC_OK;
  LLMC_CHECK_ARG(n % 8 == 0 && aligned16(a) && aligned16(b) && aligned16(y),
                 "add: n %% 8 == 0 and 16-byte alignment required");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t blocks = ((n >> 3) + 255) / 256;
  if (blocks > kNumSMs * 32) blocks = kNumSMs * 32;
#define CALL(DT) add_kernel<DT><<<(int)blocks, 256, 0, st>>>(a, b, y, n >> 3); LLMC_CHECK_LAUNCH()
  LLMC_DISPATCH_DT("add", dtype, CALL);
#undef CALL
  return LLMC_OK;
}
