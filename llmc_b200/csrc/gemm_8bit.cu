// gemm_8bit.cu — the GEMMs on Hopper 8-bit tensor cores, both operands K-major 8-bit codes:
//
//   block-FP8 (llmc_gemm_fp8_block): the block-FP8 linear forward, fp8_gemm of the reference's
//   kernel.py:153-242 and the GEMM half of block_wise_fp8_forward_func (module_utils.py:40-45).
//     Y[m, n] = sum over 128-deep K blocks kb, ascending, of
//               acc = fma(dot_kb(m, n) * a_s[m, kb], b_s[n / 128, kb], acc)
//     A [M, K] e4m3 activations with a_s [M, K/128] fp32 (act_quant's 1 x 128 groups),
//     B [N, K] e4m3 weights with b_s [ceil(N/128), K/128] fp32 (the checkpoint's weight_scale_inv).
//     Epilogues: fp32 Y (fp8_gemm with the default dtype), or bf16 Y with an optional bias added
//     after the rounding, bf16(float(bf16(acc)) + float(bias)) — `y = fp8_gemm(...).to(bfloat16);
//     y += bias` of module_utils.py:42-44 in one pass.
//
//   W8A8 (llmc_gemm_w8a8_i8 / _fp8): the forward of the exported W8A8 linears (VllmRealQuantLinear
//   and its aliases), one scale per row of X and one per row of W (a per-tensor scale is a vector of
//   stride 0).
//     acc[m, n] = sum_k qx[m, k] * qw[n, k]
//     Y[m, n]   = rT(fmul(fmul(fp32(acc), s_w[n]), s_x[m]) (+ bias[n]))   fp32 ops, one rounding
//     INT8  wgmma m64n128k32 s32.s8.s8: the int32 sum is exact (K <= 131056 bounds it by 2^31 for
//           any int8 codes), fp32(acc) is cvt.rn.
//     FP8   a fresh dot per K block as in block-FP8, promoted by acc = fadd(acc, dot).
//   Grouped W8A8 (llmc_moe_gemm_w8a8_swiglu / _down): the same GEMM over a sparse-MoE layer's routed
//   rows, one launch per projection of every expert (MoeW8A8Operands below).
//
// One persistent, warp-specialised kernel template (1 CTA per SM, 3 warpgroups), the structure of
// gemm.cu's wgmma_gemm_kernel:
//   warpgroup 0     TMA producer (one thread) filling a ring of 128-byte-swizzled stages in the
//                   L2-grouped tile order; one stage is one 128-deep K block of a 128 x 128 tile:
//                   16 KB of A + 16 KB of B (a 128-element 8-bit row is exactly one swizzle span)
//   warpgroups 1-2  consumers: each owns 64 rows of the tile and issues four wgmma m64n128k32 per
//                   K block.
//     INT8  keeps one wgmma group in flight across stages (its accumulator needs no promotion).
//     FP8   the first wgmma of a K block has scale-d = 0 (a fresh dot); wait, free the stage, then
//           promote the dot into a second register accumulator — for block-FP8 with one mul.rn and
//           one fma.rn, the reference's `mul.f32` + `fma.rn.f32`.  The two consumers drift apart, so
//           one promotes while the other's wgmmas run.  (Issuing K block kb + 1 into a second dot
//           fragment before promoting kb, with the producer's registers handed over by setmaxnreg,
//           measured no faster on the shapes of scripts/microbench.py fp8 — H100 SXM at a 400 W
//           limit.)
// BN = 128 makes the block-FP8 weight scale one scalar per K block per tile.
//
// Every output element sees the same operations in the same order whatever the tile assignment,
// grid size or problem size: its dot per K block reads only its own row of A and column of B (rows
// and columns past M / N and the K tail past K are zero-filled by TMA and never stored), and the
// promotion and epilogue are element-wise.  Only the hardware's reduced-precision accumulation
// inside a 128-deep FP8 dot differs from an fp32 sum of exact products (kernel.py's own dot depends
// on the autotuned config).
#include <type_traits>

#include "tc.cuh"

namespace llmc {
namespace {

using namespace tc;

constexpr int kBM = 128, kBN = 128, kBK = 128;
constexpr int kStages = 6;
constexpr int kTileBytes = kBM * kBK;                  // 16 KB of 8-bit elements (kBN == kBM)
constexpr int kStageBytes = 2 * kTileBytes;            // 32 KB
constexpr int kSmemBytes = ring_smem_bytes(kStages * kStageBytes);
constexpr int kThreads = 384;
// largest K (a multiple of 16) for which K * 128 * 128 < 2^31: the INT8 sum is exact for any codes
constexpr int64_t kMaxKInt8 = ((1ll << 17) - 1) / 16 * 16;

enum Mode { kBlockFp8, kW8A8Int8, kW8A8Fp8 };

struct Fp8GemmParams {
  const float* a_s;         // [M, kb_total]
  const float* b_s;         // [n_tiles, kb_total]
  const void* bias;         // [N] of bias_dt, or null (bf16 output only)
  void* out;                // [M, N] fp32 or bf16
  int64_t M, N;
  int kb_total;
  int m_tiles, n_tiles, num_tiles;
  int gn;                   // L2 group width in n-tiles (tc::grouped_tile)
  int bias_dt;
};

struct W8A8Params {
  const float* s_x;         // [M] fp32, or one value (s_x_stride 0)
  const float* s_w;         // [N] fp32, or one value (s_w_stride 0)
  int64_t s_x_stride, s_w_stride;
  const void* bias;         // [N] of the output dtype, or null
  void* out;                // [M, N] bf16 / fp16
  int64_t M, N;
  int kb_total;
  int m_tiles, n_tiles, num_tiles;
  int gn;                   // L2 group width in n-tiles (tc::grouped_tile)
};

template <Mode kMode>
using Params = std::conditional_t<kMode == kBlockFp8, Fp8GemmParams, W8A8Params>;

// Grouped (sparse-MoE) mode of the W8A8 GEMM (tc::MoeMode, on 8-bit codes): A = the routed rows
// quantised in expert order, s_x one fp32 scale per A row (stride 1).  The gate/up B stage is two
// 64 x 128-byte boxes, whole 128-byte swizzle atoms, so the stage is byte for byte the plain
// kernel's; the epilogue writes act = silu(gate) * up for 64 columns (tc::store_swiglu_m64n64).
// Both projections scale the accumulator as the plain W8A8 epilogue does first (scale_moe_w8a8).
// The grouped operands of one launch, per expert linear (tc::moe_load_b's order): its codes' tensor
// map and its weight scales (N values, or one when W8A8Params::s_w_stride is 0).  A kernel argument
// of its own, after Params.
struct MoeW8A8Operands {
  CUtensorMap tmB[2 * LLMC_MOE_MAX_EXPERTS];
  const float* s_w[2 * LLMC_MOE_MAX_EXPERTS];
  MoeSegments seg;
};
// The whole argument list of the grouped kernel fits the 32,764-byte kernel-parameter space of
// CUDA 12.1+ (driver R530+) at LLMC_MOE_MAX_EXPERTS experts.
static_assert(2 * sizeof(CUtensorMap) + sizeof(W8A8Params) + sizeof(MoeW8A8Operands) <= 32764,
              "LLMC_MOE_MAX_EXPERTS exceeds the kernel-parameter space");

// Grouped mode: acc = fmul(fmul(acc, s_w[col]), s_x[row]) over this thread's part of an m64n128
// fragment (layout at wgmma_m64n128k16_bf16) whose first row is A row row0 — the plain W8A8
// epilogue's scaling, before the shared grouped stores round.  kSwiGLU: fragments j < 8 are w1
// column col0 + 8 j + ... (scales sw_a), fragments j >= 8 the same columns of w3 (sw_b); else
// fragment j is w2 column col0 + 8 j + ... (sw_a).  Rows past p.M and columns past p.N read the
// last row's / column's scale; their results are never stored.
template <bool kSwiGLU>
__device__ __forceinline__ void scale_moe_w8a8(float (&acc)[64], int64_t row0, int64_t col0, const W8A8Params& p,
                                               const float* sw_a, const float* sw_b) {
  const int tid = threadIdx.x & 127, lane = threadIdx.x & 31;
  const int64_t r_lo = row0 + (tid >> 5) * 16 + (lane >> 2);
  const float sx0 = __ldg(p.s_x + min(r_lo, p.M - 1));
  const float sx1 = __ldg(p.s_x + min(r_lo + 8, p.M - 1));
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float* sw = (kSwiGLU && j >= 8) ? sw_b : sw_a;
    const int64_t col = col0 + 8 * (kSwiGLU ? (j & 7) : j) + 2 * (lane & 3);
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float s = __ldg(sw + min(col + e, p.N - 1) * p.s_w_stride);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int x = 4 * j + 2 * i + e;
        acc[x] = fmul_rn(fmul_rn(acc[x], s), i ? sx1 : sx0);
      }
    }
  }
}

// Y = rT(fmul(fmul(acc, s_w[n]), s_x[m]) (+ bias[n])) for this thread's part of an m64n128
// fragment (layout at wgmma_m64n128k16_bf16) whose element (0, 0) is Y[row0][col0].
template <int DT>
__device__ __forceinline__ void store_w8a8_m64n128(const float (&acc)[64], int64_t row0, int64_t col0,
                                                   const W8A8Params& p) {
  const int tid = threadIdx.x & 127, lane = threadIdx.x & 31;
  const int64_t r_lo = row0 + (tid >> 5) * 16 + (lane >> 2);
  // rows past M read the scale of row M - 1; their results are never stored
  const float sx0 = __ldg(p.s_x + min(r_lo, p.M - 1) * p.s_x_stride);
  const float sx1 = __ldg(p.s_x + min(r_lo + 8, p.M - 1) * p.s_x_stride);
  const uint16_t* bs = static_cast<const uint16_t*>(p.bias);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int64_t col = col0 + 8 * j + 2 * (lane & 3);
    if (col >= p.N) continue;
    const bool pair = col + 1 < p.N;
    const float sw0 = __ldg(p.s_w + col * p.s_w_stride);
    const float sw1 = pair ? __ldg(p.s_w + (col + 1) * p.s_w_stride) : 0.f;
    float b0 = 0.f, b1 = 0.f;
    if (bs != nullptr) {
      b0 = widen16<DT>(bs[col]);
      if (pair) b1 = widen16<DT>(bs[col + 1]);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int64_t row = r_lo + 8 * i;
      if (row >= p.M) continue;
      const float sx = i ? sx1 : sx0;
      float v0 = fmul_rn(fmul_rn(acc[4 * j + 2 * i], sw0), sx);
      float v1 = fmul_rn(fmul_rn(acc[4 * j + 2 * i + 1], sw1), sx);
      if (bs != nullptr) { v0 = fadd_rn(v0, b0); v1 = fadd_rn(v1, b1); }
      store_pair16(static_cast<uint16_t*>(p.out) + row * p.N + col, pack_pair<DT>(v0, v1), pair, p.N);
    }
  }
}

// Y = bf16(float(bf16(acc)) + float(bias[n])) for this thread's part of an m64n128 fragment
// (layout at wgmma_m64n128k16_bf16) whose first row is r_lo and whose tile starts at column col0.
__device__ __forceinline__ void store_bf16_bias_m64n128(const float (&acc)[64], int64_t r_lo, int64_t col0,
                                                        const Fp8GemmParams& p) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int64_t col = col0 + 8 * j + 2 * (lane & 3);
    if (col >= p.N) continue;
    const bool pair = col + 1 < p.N;
    const float b0 = load_as(p.bias_dt, p.bias, col);
    const float b1 = pair ? load_as(p.bias_dt, p.bias, col + 1) : 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int64_t row = r_lo + 8 * i;
      if (row >= p.M) continue;
      const float v0 = fadd_rn(DType<LLMC_BF16>::rT(acc[4 * j + 2 * i]), b0);
      const float v1 = fadd_rn(DType<LLMC_BF16>::rT(acc[4 * j + 2 * i + 1]), b1);
      const uint32_t pk = pack_pair<LLMC_BF16>(v0, v1);
      store_pair16(static_cast<uint16_t*>(p.out) + row * p.N + col, pk, pair, p.N);
    }
  }
}

// DT is the output dtype: fp32 / bf16 for kBlockFp8, bf16 / fp16 for the W8A8 modes.
// Plain mode: tiles from grouped_tile, B from tmB.  Grouped mode (kMoe, W8A8 only): tiles from
// moe_segment_tile, B and the weight scales of the tile's expert from `moe`; tmB is unused.
template <Mode kMode, int DT, int kMoe = kMoeOff>
__global__ void __launch_bounds__(kThreads, 1)
gemm_8bit_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const Params<kMode> p, const __grid_constant__ MoeArg<kMoe, MoeW8A8Operands> moe) {
  static_assert(kMoe == kMoeOff || kMode != kBlockFp8, "the grouped mode runs the W8A8 GEMM");
  constexpr bool kInt8 = kMode == kW8A8Int8;
  // the tile of unit u (grouped mode: also its expert, first A row and segment end); false past
  // the last expert's tiles
  auto tile_of = [&](int u, int& e, int& m_blk, int& n_blk, int& row0, int& row_end) -> bool {
    if constexpr (kMoe != kMoeOff) {
      return moe_segment_tile<kBM>(moe.seg, u, p.n_tiles, p.gn, e, m_blk, n_blk, row0, row_end);
    } else {
      grouped_tile(u, p.m_tiles, p.n_tiles, p.gn, m_blk, n_blk);
      return true;
    }
  };
  extern __shared__ uint8_t smem_raw[];
  // The ring is reached only through TMA and wgmma descriptors, so the generic address costs
  // nothing here.  tc::ring_base and tc::Ring's init, waits and release are not used: with either,
  // ptxas schedules the descriptor setup between the fence and the first wgmma of each K block,
  // which the wgmma_wait<0> per FP8 K block serialises (5-13 % slower at M = 4096 / 16384 with
  // DeepSeek-V3 and Llama-3-8B widths, H100 SXM at 700 W).
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    if constexpr (kMoe != kMoeOff) {
      prefetch_moe_tmaps<kMoe>(moe.tmB, moe.seg);
    } else {
      prefetch_tmap(&tmB);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);    // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (tid == 0) {
      PipeState<kStages> ps;
      for (int u = blockIdx.x; u < p.num_tiles; u += gridDim.x) {
        int e, m_blk, n_blk, row0, row_end;
        if (!tile_of(u, e, m_blk, n_blk, row0, row_end)) break;
        for (int kb = 0; kb < p.kb_total; ++kb) {
          mbar_wait(&empty_bar[ps.stage], ps.phase ^ 1);
          uint8_t* a_dst = smem + ps.stage * kStageBytes;
          mbar_expect_tx(&full_bar[ps.stage], kStageBytes);
          if constexpr (kMoe != kMoeOff) {
            tma_load_2d(a_dst, &tmA, &full_bar[ps.stage], kb * kBK, row0);
            moe_load_b<kMoe>(a_dst + kTileBytes, moe.tmB, &full_bar[ps.stage], e, kb * kBK, n_blk, kBN, kTileBytes / 2);
          } else {
            tma_load_2d(a_dst, &tmA, &full_bar[ps.stage], kb * kBK, m_blk * kBM);
            tma_load_2d(a_dst + kTileBytes, &tmB, &full_bar[ps.stage], kb * kBK, n_blk * kBN);
          }
          ps.advance();
        }
      }
    }
    return;
  }

  // ===================== consumers (warpgroups 1, 2): tile rows 64 c .. 64 c + 63 =====================
  const int c = wg - 1;
  const int lane = tid & 31;
  PipeState<kStages> ps;
  for (int u = blockIdx.x; u < p.num_tiles; u += gridDim.x) {
    int e, m_blk, n_blk, row0, row_end;
    if (!tile_of(u, e, m_blk, n_blk, row0, row_end)) break;
    // block-FP8: this thread's first fragment row (layout at wgmma_m64n128k16_bf16) and the scales
    // of its two rows; rows past M read the scale of row M - 1 — their results are never stored
    int64_t r_lo = 0;
    const float *as_lo = nullptr, *as_hi = nullptr, *bs = nullptr;
    if constexpr (kMode == kBlockFp8) {
      r_lo = static_cast<int64_t>(m_blk) * kBM + c * 64 + (tid >> 5) * 16 + (lane >> 2);
      as_lo = p.a_s + min(r_lo, p.M - 1) * p.kb_total;
      as_hi = p.a_s + min(r_lo + 8, p.M - 1) * p.kb_total;
      bs = p.b_s + static_cast<int64_t>(n_blk) * p.kb_total;
    }
    float acc[64];
    std::conditional_t<kInt8, int32_t, float> d[64];   // INT8: the tile's sum; FP8: one K block's dot
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      if constexpr (!kInt8) acc[i] = 0.f;
      d[i] = 0;
    }
    int prev = -1;                               // INT8: the stage the in-flight group reads
    for (int kb = 0; kb < p.kb_total; ++kb) {
      float sa0, sa1, sb;
      if constexpr (kMode == kBlockFp8) {
        sa0 = __ldg(as_lo + kb); sa1 = __ldg(as_hi + kb); sb = __ldg(bs + kb);
      }
      mbar_wait(&full_bar[ps.stage], ps.phase);
      wgmma_fence();
      const uint32_t a_addr = smem_u32(smem + ps.stage * kStageBytes);
      const uint32_t b_addr = a_addr + kTileBytes;
#pragma unroll
      for (int k = 0; k < kBK / 32; ++k) {
        const uint64_t adesc = make_smem_desc(a_addr + c * 64 * 128 + k * 32, 16, 1024);
        const uint64_t bdesc = make_smem_desc(b_addr + k * 32, 16, 1024);
        if constexpr (kInt8) wgmma_m64n128k32_s8(d, adesc, bdesc, (kb > 0 || k > 0) ? 1u : 0u);
        else wgmma_m64n128k32_e4m3(d, adesc, bdesc, k > 0 ? 1u : 0u);
      }
      wgmma_commit();
      if constexpr (kInt8) {
        wgmma_wait<1>();                         // the group that read stage `prev` has retired
        if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);
        prev = ps.stage;
        ps.advance();
      } else {
        wgmma_wait<0>();
        fence_acc(d);
        if (tid == 0) mbar_arrive(&empty_bar[ps.stage]);
        ps.advance();
        if constexpr (kMode == kBlockFp8) {
          // promotion: d[4 j + 2 i + e] belongs to row r_lo + 8 i
#pragma unroll
          for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float sa = i ? sa1 : sa0;
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int x = 4 * j + 2 * i + e;
                acc[x] = fma_rn(fmul_rn(d[x], sa), sb, acc[x]);
              }
            }
          }
        } else {
#pragma unroll
          for (int i = 0; i < 64; ++i) acc[i] = fadd_rn(acc[i], d[i]);
        }
      }
    }
    if constexpr (kInt8) {
      wgmma_wait<0>();
      fence_acc(d);
      if (tid == 0) mbar_arrive(&empty_bar[prev]);   // kb_total >= 1
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = __int2float_rn(d[i]);
    }

    // ---- epilogue straight from the registers ----
    const int64_t r0 = static_cast<int64_t>(m_blk) * kBM + c * 64;
    const int64_t col0 = static_cast<int64_t>(n_blk) * kBN;
    if constexpr (kMoe == kMoeSwiGLU) {
      const int64_t rg = static_cast<int64_t>(row0) + c * 64, cg = static_cast<int64_t>(n_blk) * (kBN / 2);
      scale_moe_w8a8<true>(acc, rg, cg, p, moe.s_w[2 * e], moe.s_w[2 * e + 1]);
      store_swiglu_m64n64<DT>(acc, rg, cg, row_end, p.N, p.out);
    } else if constexpr (kMoe == kMoeDown) {
      const int64_t rg = static_cast<int64_t>(row0) + c * 64;
      scale_moe_w8a8<false>(acc, rg, col0, p, moe.s_w[e], nullptr);
      store_routed_m64n128<DT>(acc, rg, col0, row_end, p.N, p.N, p.out, moe.seg.w_route);
    } else if constexpr (kMode != kBlockFp8) {
      store_w8a8_m64n128<DT>(acc, r0, col0, p);
    } else if constexpr (DT == LLMC_F32) {
      store_f32_m64n128(acc, r0, col0, p.M, p.N, p.N, static_cast<float*>(p.out));
    } else if (p.bias == nullptr) {
      store_linear_m64n128<LLMC_BF16>(acc, r0, col0, p.M, p.N, p.N, nullptr, p.out);
    } else {
      store_bf16_bias_m64n128(acc, r_lo, col0, p);
    }
  }
}

// Encodes the two K-major 8-bit operand maps, completes p with the shape and the tile plan, and
// launches the persistent kernel with bf16 output (dt == LLMC_BF16) or the mode's other dtype.
template <Mode kMode>
int launch_gemm_8bit(const void* a, const void* b, int64_t M, int64_t N, int64_t K, int kb_total, int dt,
                     Params<kMode> p, void* stream) {
  CUtensorMap tmA, tmB;
  if (int rc = encode_tmap_2d(&tmA, a, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, M, K, K, kBM, kBK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  if (int rc = encode_tmap_2d(&tmB, b, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, N, K, K, kBN, kBK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  p.M = M; p.N = N;
  p.kb_total = kb_total;
  p.m_tiles = static_cast<int>((M + kBM - 1) / kBM);
  p.n_tiles = static_cast<int>((N + kBN - 1) / kBN);
  p.num_tiles = p.m_tiles * p.n_tiles;
  p.gn = l2_group_width(static_cast<int64_t>(kBN) * K, p.n_tiles);   // one n-tile's weight bytes
  constexpr int kOtherDt = kMode == kBlockFp8 ? LLMC_F32 : LLMC_F16;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return launch_persistent(dt == LLMC_BF16 ? gemm_8bit_kernel<kMode, LLMC_BF16>
                                           : gemm_8bit_kernel<kMode, kOtherDt>,
                           p.num_tiles, kThreads, kSmemBytes, st, tmA, tmB, p, static_cast<const void*>(nullptr));
}

template <bool kFp8>
int gemm_w8a8(const char* what, const void* x, const float* s_x, int64_t s_x_stride, const void* w,
              const float* s_w, int64_t s_w_stride, const void* bias, void* y, int64_t M, int64_t N,
              int64_t K, int dtype, void* stream) {
  LLMC_CHECK_ARG(M >= 0 && N >= 1 && K >= 1, "%s: bad shape M=%lld N=%lld K=%lld", what, (long long)M,
                 (long long)N, (long long)K);
  LLMC_CHECK_ARG(dtype == LLMC_BF16 || dtype == LLMC_F16, "%s: dtype %d must be bf16 or fp16", what, dtype);
  LLMC_CHECK_ARG(s_x_stride == 0 || s_x_stride == 1, "%s: s_x_stride %lld must be 0 or 1", what,
                 (long long)s_x_stride);
  LLMC_CHECK_ARG(s_w_stride == 0 || s_w_stride == 1, "%s: s_w_stride %lld must be 0 or 1", what,
                 (long long)s_w_stride);
  LLMC_CHECK_ARG(K % 16 == 0, "%s: K=%lld must be a multiple of 16", what, (long long)K);
  LLMC_CHECK_ARG(kFp8 || K <= kMaxKInt8, "%s: K=%lld > %lld overflows the int32 sum", what, (long long)K,
                 (long long)kMaxKInt8);
  const int64_t m_tiles = (M + kBM - 1) / kBM, n_tiles = (N + kBN - 1) / kBN;
  LLMC_CHECK_ARG(m_tiles * n_tiles < (1ll << 31), "%s: too many tiles", what);
  if (M == 0) return LLMC_OK;
  LLMC_CHECK_ARG(x && s_x && w && s_w && y, "%s: null pointer", what);
  if (!aligned16(x) || !aligned16(w) || !aligned16(y)) {
    set_last_error("%s: x, w and y must be 16-byte aligned", what);
    return LLMC_EALIGN;
  }
  W8A8Params p{};
  p.s_x = s_x; p.s_w = s_w; p.s_x_stride = s_x_stride; p.s_w_stride = s_w_stride;
  p.bias = bias; p.out = y;
  const int kb_total = static_cast<int>((K + kBK - 1) / kBK);   // TMA zero-fills the K tail
  return launch_gemm_8bit<kFp8 ? kW8A8Fp8 : kW8A8Int8>(x, w, M, N, K, kb_total, dtype, p, stream);
}

// Checks and launches the grouped W8A8 GEMM over m.rows quantised rows, s_x one scale per row;
// s_a / s_b the per-expert weight scales of w_a / w_b.
template <int kMoe>
int moe_w8a8(const MoeLaunch<kMoe>& m, const float* s_x, int fp8, const float* const* s_a, const float* const* s_b,
             int64_t s_w_stride, void* stream) {
  int n_tiles, units;
  if (int rc = m.check_values(kBM, kBN)) return rc;
  LLMC_CHECK_ARG(m.K % 16 == 0, "%s: K=%lld must be a multiple of 16", m.what, (long long)m.K);
  LLMC_CHECK_ARG(fp8 || m.K <= kMaxKInt8, "%s: K=%lld > %lld overflows the int32 sum", m.what, (long long)m.K,
                 (long long)kMaxKInt8);
  LLMC_CHECK_ARG(s_w_stride == 0 || s_w_stride == 1, "%s: s_w_stride %lld must be 0 or 1", m.what,
                 (long long)s_w_stride);
  if (int rc = m.plan(kBM, kBN, n_tiles, units)) return rc;
  if (m.rows == 0) return LLMC_OK;
  if (int rc = m.check_pointers()) return rc;
  LLMC_CHECK_ARG(s_x && s_a && (!m.kSwiGLU || s_b), "%s: null pointer", m.what);
  MoeW8A8Operands g{};
  for (int i = 0; i < m.linears(); ++i) {
    g.s_w[i] = m.linear(s_a, s_b, i);
    LLMC_CHECK_ARG(g.s_w[i], "%s: null codes or scales of expert %d", m.what, m.expert_of(i));
  }
  CUtensorMap tmA;
  if (int rc = encode_tmap_2d(&tmA, m.a, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, m.rows, m.K, m.K, kBM, kBK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  if (int rc = m.encode_tmaps(g.tmB, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, m.K, kBN, kBK, CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  g.seg = m.segments();
  W8A8Params p{};
  p.s_x = s_x; p.s_x_stride = 1; p.s_w_stride = s_w_stride;
  p.out = m.out;
  p.M = m.rows; p.N = m.N;
  p.kb_total = static_cast<int>((m.K + kBK - 1) / kBK);   // TMA zero-fills the K tail
  p.n_tiles = n_tiles;
  p.num_tiles = units;
  p.gn = l2_group_width(static_cast<int64_t>(kBN) * m.K, n_tiles);   // one n-tile's weight bytes
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto kernel = fp8 ? (m.dtype == LLMC_BF16 ? gemm_8bit_kernel<kW8A8Fp8, LLMC_BF16, kMoe>
                                            : gemm_8bit_kernel<kW8A8Fp8, LLMC_F16, kMoe>)
                    : (m.dtype == LLMC_BF16 ? gemm_8bit_kernel<kW8A8Int8, LLMC_BF16, kMoe>
                                            : gemm_8bit_kernel<kW8A8Int8, LLMC_F16, kMoe>);
  return launch_persistent(kernel, p.num_tiles, kThreads, kSmemBytes, st, tmA, CUtensorMap{}, p, g);
}

}  // namespace
}  // namespace llmc

using namespace llmc;

extern "C" int llmc_gemm_fp8_block(const void* a, const float* a_s, const void* b, const float* b_s,
                                   const void* bias, int bias_dtype, void* out, int out_dtype,
                                   int64_t M, int64_t N, int64_t K, void* stream) {
  LLMC_CHECK_ARG(M >= 0 && N >= 1 && K >= 1, "gemm_fp8_block: bad shape M=%lld N=%lld K=%lld",
                 (long long)M, (long long)N, (long long)K);
  LLMC_CHECK_ARG(K % kBK == 0, "gemm_fp8_block: K=%lld must be a multiple of 128", (long long)K);
  LLMC_CHECK_ARG(out_dtype == LLMC_F32 || out_dtype == LLMC_BF16,
                 "gemm_fp8_block: out dtype %d must be fp32 or bf16", out_dtype);
  LLMC_CHECK_ARG(bias == nullptr || out_dtype == LLMC_BF16,
                 "gemm_fp8_block: a bias needs the bf16 output");
  LLMC_CHECK_ARG(bias == nullptr || (bias_dtype >= LLMC_F32 && bias_dtype <= LLMC_BF16),
                 "gemm_fp8_block: bad bias dtype %d", bias_dtype);
  if (M == 0) return LLMC_OK;
  LLMC_CHECK_ARG(a && a_s && b && b_s && out, "gemm_fp8_block: null pointer");
  if (!aligned16(a) || !aligned16(b) || !aligned16(out)) {
    set_last_error("gemm_fp8_block: a, b and out must be 16-byte aligned");
    return LLMC_EALIGN;
  }
  const int64_t m_tiles = (M + kBM - 1) / kBM, n_tiles = (N + kBN - 1) / kBN;
  LLMC_CHECK_ARG(m_tiles * n_tiles < (1ll << 31) && K / kBK < (1ll << 31),
                 "gemm_fp8_block: too many tiles");
  Fp8GemmParams p{};
  p.a_s = a_s; p.b_s = b_s; p.bias = bias; p.out = out;
  p.bias_dt = bias_dtype;
  return launch_gemm_8bit<kBlockFp8>(a, b, M, N, K, static_cast<int>(K / kBK), out_dtype, p, stream);
}

extern "C" int llmc_gemm_w8a8_i8(const void* x, const float* s_x, int64_t s_x_stride, const void* w,
                                 const float* s_w, int64_t s_w_stride, const void* bias, void* y, int64_t M,
                                 int64_t N, int64_t K, int dtype, void* stream) {
  return gemm_w8a8<false>("gemm_w8a8_i8", x, s_x, s_x_stride, w, s_w, s_w_stride, bias, y, M, N, K, dtype,
                          stream);
}

extern "C" int llmc_gemm_w8a8_fp8(const void* x, const float* s_x, int64_t s_x_stride, const void* w,
                                  const float* s_w, int64_t s_w_stride, const void* bias, void* y, int64_t M,
                                  int64_t N, int64_t K, int dtype, void* stream) {
  return gemm_w8a8<true>("gemm_w8a8_fp8", x, s_x, s_x_stride, w, s_w, s_w_stride, bias, y, M, N, K, dtype,
                         stream);
}

extern "C" int llmc_moe_gemm_w8a8_swiglu(const void* xq, const float* s_x, int fp8, const void* const* w1,
                                         const void* const* w3, const float* const* s_w1,
                                         const float* const* s_w3, int64_t s_w_stride, const int32_t* offsets,
                                         void* act, int64_t rows, int64_t inter, int64_t K, int64_t n_experts,
                                         int dtype, void* stream) {
  return moe_w8a8<kMoeSwiGLU>({"moe_gemm_w8a8_swiglu", xq, act, w1, w3, offsets, nullptr, rows, inter, K, n_experts,
                               dtype, "codes or scales"}, s_x, fp8, s_w1, s_w3, s_w_stride, stream);
}

extern "C" int llmc_moe_gemm_w8a8_down(const void* actq, const float* s_x, int fp8, const void* const* w2,
                                       const float* const* s_w2, int64_t s_w_stride, const int32_t* offsets,
                                       const void* w_route, void* y, int64_t rows, int64_t N, int64_t inter,
                                       int64_t n_experts, int dtype, void* stream) {
  return moe_w8a8<kMoeDown>({"moe_gemm_w8a8_down", actq, y, w2, nullptr, offsets, w_route, rows, N, inter, n_experts,
                             dtype, "codes or scales"}, s_x, fp8, s_w2, nullptr, s_w_stride, stream);
}
