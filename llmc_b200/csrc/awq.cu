// awq.cu — K8/K9: the tensor-level pieces of AWQ's scale search and weight auto-clip.
//
//  * llmc_absmean_cols   get_act_scale            (awq.py:74-85):  mean_t |x[t, c]|
//  * llmc_div_cols       scaling_input            (base_blockwise_quantization.py:876-889): x / s[c]
//  * llmc_mse            calculate_loss           (awq.py:134-145): mean(((a - b) in T).float()^2)
//  * llmc_awq_clip_err + llmc_awq_clip_select     AutoClipper.auto_clip_layer (auto_clip.py:83-191)
//  (the scaled fake-quant W*s -> group qdq of awq.py:147-164 is llmc_quant_dynamic's col_scale)
//
// All are HBM / CUDA-core work: the reference evaluates them as chains of elementwise torch ops on
// fp16/bf16 tensors (auto-clip materialises [256, 512, ng, g] broadcast products, ~1 GiB per step);
// here nothing is materialised.  Arithmetic is T-faithful (common.cuh), reductions accumulate in
// fp32 like torch and round once.
#include "common.cuh"
#include "quant_math.cuh"

namespace llmc {

// ---- mean |x| over rows, per column ------------------------------------------------------------
template <int DT>
__global__ void __launch_bounds__(256)
absmean_stage1(const void* __restrict__ x, int64_t T, int64_t C, int rows_per_split,
               float* __restrict__ ws) {
  // grid (C/8 column-octets / 256, splits): thread owns 8 consecutive columns
  const int64_t oct = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (oct * 8 >= C) return;
  const int64_t t0 = static_cast<int64_t>(blockIdx.y) * rows_per_split;
  const int64_t t1 = min(t0 + rows_per_split, T);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int64_t t = t0; t < t1; ++t) {
    float v[8];
    load8<DT>(x, t * C + oct * 8, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] += fabsf(v[i]);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) ws[static_cast<int64_t>(blockIdx.y) * C + oct * 8 + i] = acc[i];
}

template <int DT>
__global__ void __launch_bounds__(256)
absmean_stage2(const float* __restrict__ ws, int splits, int64_t T, int64_t C, void* __restrict__ out) {
  const int64_t c = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float acc = 0.f;
  for (int s = 0; s < splits; ++s) acc += ws[static_cast<int64_t>(s) * C + c];
  DType<DT>::store(out, c, acc / static_cast<float>(T));
}

// ---- x / s[c] ------------------------------------------------------------------------------------
template <int DT>
__global__ void __launch_bounds__(256)
div_cols_kernel(const void* __restrict__ x, const void* __restrict__ s, int64_t T, int64_t C,
                void* __restrict__ out) {
  const int64_t octs_per_row = C >> 3;
  const int64_t total = T * octs_per_row;
  for (int64_t u = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < total;
       u += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t t = u / octs_per_row, o = u - t * octs_per_row;
    float v[8], sv[8], y[8];
    load8<DT>(x, t * C + o * 8, v);
    load8<DT>(s, o * 8, sv);
#pragma unroll
    for (int i = 0; i < 8; ++i) y[i] = fdiv_rn(v[i], sv[i]);     // store8 rounds to T
    store8<DT>(out, t * C + o * 8, y);
  }
}

// ---- mean(((a - b) rounded to T)^2) ------------------------------------------------------------------
template <int DT>
__global__ void __launch_bounds__(256)
mse_stage1(const void* __restrict__ a, const void* __restrict__ b, int64_t n, float* __restrict__ ws) {
  __shared__ float red[8];
  float acc = 0.f;
  const int64_t n8 = n >> 3;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float va[8], vb[8];
    load8<DT>(a, i << 3, va);
    load8<DT>(b, i << 3, vb);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float d = DType<DT>::rT(fsub_rn(va[k], vb[k]));
      acc = fmaf(d, d, acc);
    }
  }
  if (blockIdx.x == 0)
    for (int64_t i = (n8 << 3) + threadIdx.x; i < n; i += blockDim.x) {
      const float d = DType<DT>::rT(fsub_rn(DType<DT>::load(a, i), DType<DT>::load(b, i)));
      acc = fmaf(d, d, acc);
    }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) ws[blockIdx.x] = v;
  }
}

__global__ void __launch_bounds__(256)
mse_stage2(const float* __restrict__ ws, int nblocks, double n, float* __restrict__ out) {
  __shared__ double red[8];
  double acc = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) acc += static_cast<double>(ws[i]);
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += red[i];
    // t / n rounded to double and then to fp32 is t / n rounded once to fp32 (53 >= 2 * 24 + 2);
    // t * (1 / n) would round three times
    out[0] = static_cast<float>(t / n);
  }
}

// ---- auto-clip --------------------------------------------------------------------------------------
// One CTA per (group, row slice).  The group's sampled activations X_g [ns <= 512 tokens, g] sit in
// shared memory (padded pitch: lanes read different tokens of the same k without bank conflicts);
// a warp owns one weight row at a time: lanes = tokens (16 per lane), the 128 (clamped, fake-
// quantised) weights of the current shrink level are broadcast from a per-warp smem vector.
constexpr int kClipMaxTok = 256;           // tokens per pass (fp32 tile: 256 x 129 x 4 B = 132 KB)
constexpr int kClipLevels = 10;           // int(max_shrink 0.5 * n_grid 20), auto_clip.py:127
constexpr int kClipG = 128;               // max group size handled by this kernel

struct ClipArgs {
  const void* w;        // [R, C]
  const void* x;        // [ns_total, C] sampled tokens
  int64_t R, C;
  int group, ng;
  int tok0, ntok;       // token chunk [tok0, tok0 + ntok), ntok <= kClipMaxTok
  int sym, bit, clip_sym;
  float qmin, qmax;
  float* err;           // [R, ng, 10] fp32 sums over tokens (accumulated across chunks)
};

template <int DT>
__device__ __forceinline__ void group_qdq(const float (&cw)[4], int nk, int sym, float qmin, float qmax,
                                          float (&qw)[4], int lane) {
  // fake_quant_weight_dynamic on one group of g = 4 * 32 (or fewer) values held 4 per lane
  float mn = INFINITY, mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (lane * 4 + i < nk) { mn = fminf(mn, cw[i]); mx = fmaxf(mx, cw[i]); }
  mn = warp_min(mn);
  mx = warp_max(mx);
  float s, z;
  qparams<DType<DT>>(mn, mx, sym, 1, qmin, qmax, s, z);
#pragma unroll
  for (int i = 0; i < 4; ++i)
    qw[i] = dequant<DType<DT>>(quant_code<DType<DT>>(cw[i], IeeeDiv{s}, z, qmin, qmax), s, z);
}

template <int DT>
__global__ void __launch_bounds__(256, 1)
awq_clip_err_kernel(ClipArgs a) {
  extern __shared__ float csm[];
  constexpr int PITCH = kClipG + 1;                 // floats per token row (conflict-free)
  float* Xs = csm;                                  // [ntok][PITCH] activations of this group (fp32)
  float* Wv = csm + kClipMaxTok * PITCH;            // [8 warps][kClipG] current-level weights
  const int grp = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = a.group;
  // stage X_g
  for (int idx = threadIdx.x; idx < a.ntok * g; idx += blockDim.x) {
    const int t = idx / g, k = idx - t * g;
    Xs[t * PITCH + k] = DType<DT>::load(a.x, static_cast<int64_t>(a.tok0 + t) * a.C + grp * g + k);
  }
  __syncthreads();
  float* wv = Wv + warp * kClipG;
  const int rows_per_cta = (static_cast<int>(a.R) + gridDim.y - 1) / gridDim.y;
  const int r_begin = blockIdx.y * rows_per_cta;
  const int r_end = min(r_begin + rows_per_cta, static_cast<int>(a.R));
  for (int r = r_begin + warp; r < r_end; r += 8) {
    // this lane's 4 weights of the group
    float w4[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = lane * 4 + i;
      w4[i] = (k < g) ? DType<DT>::load(a.w, static_cast<int64_t>(r) * a.C + grp * g + k) : 0.f;
    }
    float omax = -INFINITY, omin = INFINITY;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (lane * 4 + i < g) {
        omax = fmaxf(omax, a.clip_sym ? fabsf(w4[i]) : w4[i]);
        omin = fminf(omin, w4[i]);
      }
    omax = warp_max(omax);
    omin = warp_min(omin);
    // org_out for this lane's tokens: sum_k rT(x * w), rounded once to T (auto_clip.py:149)
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 4; ++i) wv[lane * 4 + i] = w4[i];
    __syncwarp();
    float org[kClipMaxTok / 32];
#pragma unroll
    for (int j = 0; j < kClipMaxTok / 32; ++j) {
      const int t = lane + 32 * j;
      float acc = 0.f;
      if (t < a.ntok) {
        const float* xr = Xs + t * PITCH;
        for (int k = 0; k < g; ++k) acc += DType<DT>::rT(fmul_rn(xr[k], wv[k]));
      }
      org[j] = DType<DT>::rT(acc);
    }
    for (int lvl = 0; lvl < kClipLevels; ++lvl) {
      const float f = static_cast<float>(1.0 - static_cast<double>(lvl) / 20.0);
      const float maxv = DType<DT>::rT(fmul_rn(omax, f));
      const float minv = a.clip_sym ? -maxv : DType<DT>::rT(fmul_rn(omin, f));
      float cw[4], qw[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) cw[i] = fminf(fmaxf(w4[i], minv), maxv);
      group_qdq<DT>(cw, g, a.sym, a.qmin, a.qmax, qw, lane);
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 4; ++i) wv[lane * 4 + i] = qw[i];
      __syncwarp();
      float esum = 0.f;
#pragma unroll
      for (int j = 0; j < kClipMaxTok / 32; ++j) {
        const int t = lane + 32 * j;
        if (t < a.ntok) {
          const float* xr = Xs + t * PITCH;
          float acc = 0.f;
          for (int k = 0; k < g; ++k) acc += DType<DT>::rT(fmul_rn(xr[k], wv[k]));
          const float d = DType<DT>::rT(fsub_rn(DType<DT>::rT(acc), org[j]));
          esum += DType<DT>::rT(fmul_rn(d, d));
        }
      }
      esum = warp_sum(esum);
      if (lane == 0) a.err[(static_cast<int64_t>(r) * a.ng + grp) * kClipLevels + lvl] += esum;
    }
  }
}

template <int DT>
__global__ void __launch_bounds__(256)
awq_clip_select_kernel(const void* __restrict__ w, int64_t R, int64_t C, int group, int ng,
                       int clip_sym, const float* __restrict__ err, int ns,
                       void* __restrict__ best_max, void* __restrict__ best_min) {
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= R * ng) return;
  const int64_t r = idx / ng;
  const int grp = static_cast<int>(idx - r * ng);
  float omax = -INFINITY, omin = INFINITY;
  for (int k = 0; k < group; ++k) {
    const float v = DType<DT>::load(w, r * C + static_cast<int64_t>(grp) * group + k);
    omax = fmaxf(omax, clip_sym ? fabsf(v) : v);
    omin = fminf(omin, v);
  }
  float best_e = DType<DT>::rT(1e9f);       // torch.ones_like(org_max_val) * 1e9 in T
  float bmax = omax, bmin = omin;
  for (int lvl = 0; lvl < kClipLevels; ++lvl) {
    const float e = DType<DT>::rT(err[idx * kClipLevels + lvl] / static_cast<float>(ns));
    if (e < best_e) {                        // strict <: the earliest level wins ties
      const float f = static_cast<float>(1.0 - static_cast<double>(lvl) / 20.0);
      best_e = e;
      bmax = DType<DT>::rT(fmul_rn(omax, f));
      bmin = clip_sym ? -bmax : DType<DT>::rT(fmul_rn(omin, f));
    }
  }
  DType<DT>::store(best_max, idx, bmax);
  DType<DT>::store(best_min, idx, bmin);
}

}  // namespace llmc

using namespace llmc;

extern "C" int llmc_absmean_cols(const void* x, int64_t T, int64_t C, int dtype, void* out,
                                 float* workspace, int64_t workspace_floats, void* stream) {
  LLMC_CHECK_ARG(x && out && workspace && T > 0 && C > 0, "absmean_cols: bad argument");
  LLMC_CHECK_ARG(C % 8 == 0 && aligned16(x), "absmean_cols: C %% 8 == 0 and 16-byte alignment required");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int splits = static_cast<int>(T < 64 ? 1 : (T / 64 < 256 ? T / 64 : 256));
  while (static_cast<int64_t>(splits) * C > workspace_floats && splits > 1) splits /= 2;
  LLMC_CHECK_ARG(static_cast<int64_t>(splits) * C <= workspace_floats, "absmean_cols: workspace too small");
  const int rows_per_split = static_cast<int>((T + splits - 1) / splits);
  splits = static_cast<int>((T + rows_per_split - 1) / rows_per_split);
  dim3 grid(static_cast<unsigned>((C / 8 + 255) / 256), static_cast<unsigned>(splits));
#define CALL(DT)                                                                            \
  absmean_stage1<DT><<<grid, 256, 0, st>>>(x, T, C, rows_per_split, workspace);             \
  LLMC_CHECK_LAUNCH();                                                                      \
  absmean_stage2<DT><<<static_cast<unsigned>((C + 255) / 256), 256, 0, st>>>(workspace, splits, T, C, out); \
  LLMC_CHECK_LAUNCH()
  LLMC_DISPATCH_DT("absmean_cols", dtype, CALL);
#undef CALL
  return LLMC_OK;
}

extern "C" int llmc_div_cols(const void* x, const void* s, int64_t T, int64_t C, int dtype, void* out,
                             void* stream) {
  LLMC_CHECK_ARG(x && s && out && T >= 0 && C > 0, "div_cols: bad argument");
  if (T == 0) return LLMC_OK;
  LLMC_CHECK_ARG(C % 8 == 0 && aligned16(x) && aligned16(s) && aligned16(out),
                 "div_cols: C %% 8 == 0 and 16-byte alignment required");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t blocks = (T * (C / 8) + 255) / 256;
  if (blocks > kNumSMs * 32) blocks = kNumSMs * 32;
#define CALL(DT) div_cols_kernel<DT><<<(int)blocks, 256, 0, st>>>(x, s, T, C, out); LLMC_CHECK_LAUNCH()
  LLMC_DISPATCH_DT("div_cols", dtype, CALL);
#undef CALL
  return LLMC_OK;
}

extern "C" int llmc_mse(const void* a, const void* b, int64_t n, int dtype, float* out,
                        float* workspace, void* stream) {
  LLMC_CHECK_ARG(a && b && out && workspace && n > 0, "mse: bad argument (workspace >= 1024 floats)");
  LLMC_CHECK_ARG(aligned16(a) && aligned16(b), "mse: 16-byte alignment required");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t blocks = ((n >> 3) + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > 1024) blocks = 1024;
#define CALL(DT) mse_stage1<DT><<<(int)blocks, 256, 0, st>>>(a, b, n, workspace); LLMC_CHECK_LAUNCH()
  LLMC_DISPATCH_DT("mse", dtype, CALL);
#undef CALL
  mse_stage2<<<1, 256, 0, st>>>(workspace, (int)blocks, static_cast<double>(n), out);
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

extern "C" int llmc_awq_clip(const void* w, int64_t R, int64_t C, const void* x, int64_t ns, int dtype,
                             int64_t group, int bit, int sym, int clip_sym, void* best_max,
                             void* best_min, float* workspace, int64_t workspace_floats,
                             void* stream) {
  LLMC_CHECK_ARG(w && x && best_max && best_min && workspace && R > 0 && C > 0 && ns > 0,
                 "awq_clip: bad argument");
  LLMC_CHECK_ARG(group > 0 && C % group == 0, "awq_clip: C %% group != 0");
  if (group > kClipG) {
    set_last_error("awq_clip: group %lld > %d (per_channel clip) has no kernel yet", (long long)group, kClipG);
    return LLMC_EUNSUPPORTED;
  }
  LLMC_CHECK_ARG(bit >= 2 && bit <= 8, "awq_clip: bit %d outside 2..8", bit);
  const int ng = static_cast<int>(C / group);
  LLMC_CHECK_ARG(workspace_floats >= R * ng * kClipLevels, "awq_clip: workspace too small");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LLMC_CHECK_CUDA(cudaMemsetAsync(workspace, 0, R * ng * kClipLevels * sizeof(float), st));
  ClipArgs a{};
  a.w = w; a.x = x; a.R = R; a.C = C; a.group = static_cast<int>(group); a.ng = ng;
  a.sym = sym; a.bit = bit; a.clip_sym = clip_sym;
  int_range(bit, sym, a.qmin, a.qmax);
  a.err = workspace;
  const int smem = (kClipMaxTok * (kClipG + 1) + 8 * kClipG) * 4;
  for (auto kern : {awq_clip_err_kernel<LLMC_F32>, awq_clip_err_kernel<LLMC_F16>, awq_clip_err_kernel<LLMC_BF16>})
    if (int rc = opt_in_smem(kern, smem)) return rc;
  // row slices so that ng * slices ~ a few waves of kNumSMs CTAs
  int slices = (4 * kNumSMs + ng - 1) / ng;
  if (slices > (R + 7) / 8) slices = static_cast<int>((R + 7) / 8);
  if (slices < 1) slices = 1;
  dim3 grid(static_cast<unsigned>(ng), static_cast<unsigned>(slices));
  for (int64_t t0 = 0; t0 < ns; t0 += kClipMaxTok) {
    a.tok0 = static_cast<int>(t0);
    a.ntok = static_cast<int>(ns - t0 < kClipMaxTok ? ns - t0 : kClipMaxTok);
#define CALL(DT) awq_clip_err_kernel<DT><<<grid, 256, smem, st>>>(a); LLMC_CHECK_LAUNCH()
    LLMC_DISPATCH_DT("awq_clip", dtype, CALL);
#undef CALL
  }
  const int64_t total = R * ng;
#define CALL(DT)                                                                                   \
  awq_clip_select_kernel<DT><<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(          \
      w, R, C, static_cast<int>(group), ng, clip_sym, workspace, static_cast<int>(ns), best_max, best_min); \
  LLMC_CHECK_LAUNCH()
  LLMC_DISPATCH_DT("awq_clip", dtype, CALL);
#undef CALL
  return LLMC_OK;
}
