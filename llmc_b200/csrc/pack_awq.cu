// pack_awq.cu — K2-awq: AutoAWQ "gemm_pack" layout.
//
// Replaces AutoawqRealQuantLinear.gemm_pack (llmc/compression/quantization/module_utils.py:
// 1004-1065): a Python loop over every input column that recomputes
//   intweight[:, c] = round((W[:, c] + zeros*scales) / scales)      (no clamp, :1022-1029)
// transposes to [C, R] and ORs 8 nibbles per int32 along R in the order {0,2,4,6,1,3,5,7}.
//
// One CTA handles a 256(R) x 64(C) tile: coalesced 128-byte reads along C, a transposing
// shared-memory stage of int8 codes, coalesced 128-byte writes of 32 packed words along R/8.
#include "common.cuh"

namespace llmc {

constexpr int kTileR = 256;
constexpr int kTileC = 64;

// torch promotes (weight dtype, fp16 scales): fp16 stays fp16, bf16/fp32 compute in fp32.
template <int WT>
__global__ void __launch_bounds__(256)
pack_awq_kernel(const void* __restrict__ w, int64_t R, int64_t C, const void* __restrict__ scales,
                int s_dtype, const int32_t* __restrict__ zeros, int64_t group, int64_t ng,
                int32_t* __restrict__ qweight) {
  __shared__ int8_t codes[kTileC][kTileR + 4];
  const int64_t r0 = static_cast<int64_t>(blockIdx.y) * kTileR;
  const int64_t c0 = static_cast<int64_t>(blockIdx.x) * kTileC;
  // phase 1: thread t -> (row = r0 + t/64*?...) ; 256 threads cover 4 rows x 64 cols per step
  const int tc = threadIdx.x & 63;
  const int tr = threadIdx.x >> 6;
  for (int rr = tr; rr < kTileR; rr += 4) {
    const int64_t r = r0 + rr, c = c0 + tc;
    int v = 0;
    if (r < R && c < C) {
      const int64_t g = c / group;
      // scales.t().contiguous().to(torch.float16)  (:1008)
      const float s = DType<LLMC_F16>::rT(load_as(s_dtype, scales, r * ng + g));
      const float z = static_cast<float>(zeros[r * ng + g]);
      const float sz = DType<LLMC_F16>::rT(fmul_rn(z, s));  // int32 * fp16 -> fp16 (:1011)
      const float x = DType<WT>::load(w, r * C + c);
      float q;
      if constexpr (WT == LLMC_F16) {
        float a = DType<LLMC_F16>::rT(fadd_rn(x, sz));
        q = DType<LLMC_F16>::rT(fdiv_rn(a, s));
      } else {
        q = fdiv_rn(fadd_rn(x, sz), s);
      }
      v = static_cast<int>(rintf(q));
    }
    codes[tc][rr] = static_cast<int8_t>(v);
  }
  __syncthreads();
  // phase 2: 64 output rows (c) x 32 words (r/8); thread t -> word (c = t/32 + 8*k, wi = t%32)
  const int wi = threadIdx.x & 31;
  for (int cc = threadIdx.x >> 5; cc < kTileC; cc += 8) {
    const int64_t c = c0 + cc;
    const int64_t rbase = r0 + wi * 8;
    if (c < C && rbase < R) {
      const int order[8] = {0, 2, 4, 6, 1, 3, 5, 7};
      uint32_t word = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int v = codes[cc][wi * 8 + order[i]];
        word |= static_cast<uint32_t>(v) << (4 * i);  // int32 shift + OR, sign bits included
      }
      qweight[c * (R / 8) + (rbase >> 3)] = static_cast<int32_t>(word);
    }
  }
}

__global__ void __launch_bounds__(256)
pack_awq_qparams_kernel(const void* __restrict__ scales, int s_dtype,
                        const int32_t* __restrict__ zeros, int64_t R, int64_t ng,
                        int32_t* __restrict__ qzeros, __half* __restrict__ scales_out) {
  // scales_out [ng, R] fp16 ; qzeros [ng, R/8]
  const int64_t total = ng * R;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t g = i / R, r = i - g * R;
    scales_out[i] = __float2half_rn(load_as(s_dtype, scales, r * ng + g));
    if ((r & 7) == 0) {
      const int order[8] = {0, 2, 4, 6, 1, 3, 5, 7};
      uint32_t word = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        word |= static_cast<uint32_t>(zeros[(r + order[k]) * ng + g]) << (4 * k);
      qzeros[g * (R / 8) + (r >> 3)] = static_cast<int32_t>(word);
    }
  }
}

}  // namespace llmc

using namespace llmc;

extern "C" int llmc_pack_awq(const void* w, int64_t R, int64_t C, int dtype, const void* scales,
                             int s_dtype, const int32_t* zeros, int64_t group,
                             int32_t* qweight, int32_t* qzeros, void* scales_out_f16,
                             void* stream) {
  LLMC_CHECK_ARG(w && scales && zeros && qweight && qzeros && scales_out_f16,
                 "pack_awq: null pointer (AutoAWQ packing needs asymmetric zeros, module_utils.py:1006)");
  LLMC_CHECK_ARG(R > 0 && C > 0 && R % 32 == 0, "pack_awq: R=%lld must be a positive multiple of 32",
                 (long long)R);
  LLMC_CHECK_ARG(group > 0 && C % group == 0, "pack_awq: C=%lld not divisible by group %lld",
                 (long long)C, (long long)group);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t ng = C / group;
  dim3 grid((unsigned)((C + kTileC - 1) / kTileC), (unsigned)((R + kTileR - 1) / kTileR));
#define CALL(DT) pack_awq_kernel<DT><<<grid, 256, 0, st>>>(w, R, C, scales, s_dtype, zeros, group, ng, qweight)
  LLMC_DISPATCH_DT("pack_awq", dtype, CALL);
#undef CALL
  LLMC_CHECK_LAUNCH();
  int64_t total = ng * R;
  int64_t blocks = (total + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  pack_awq_qparams_kernel<<<(int)blocks, 256, 0, st>>>(scales, s_dtype, zeros, R, ng, qzeros,
                                                       reinterpret_cast<__half*>(scales_out_f16));
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}
