// gemm_fp8.cu — the block-FP8 linear forward on Hopper FP8 tensor cores: fp8_gemm of the
// reference's kernel.py:153-242 and the GEMM half of block_wise_fp8_forward_func
// (module_utils.py:40-45).
//
//   Y[m, n] = sum over 128-deep K blocks kb, ascending, of
//             acc = fma(dot_kb(m, n) * a_s[m, kb], b_s[n / 128, kb], acc)
//   A [M, K] e4m3 activations with a_s [M, K/128] fp32 (act_quant's 1 x 128 groups),
//   B [N, K] e4m3 weights with b_s [ceil(N/128), K/128] fp32 (the checkpoint's weight_scale_inv).
//
// One persistent, warp-specialised kernel (1 CTA per SM, 3 warpgroups), the structure of
// gemm.cu's wgmma_gemm_kernel:
//   warpgroup 0     TMA producer (one thread) filling a ring of 128-byte-swizzled stages; one
//                   stage is one 128-deep K block of a 128 x 128 tile: 16 KB of A + 16 KB of B
//                   (a 128-element e4m3 row is exactly one swizzle span)
//   warpgroups 1-2  consumers: each owns 64 rows of the tile.  Per K block four
//                   wgmma m64n128k32 e4m3 (the first with scale-d = 0: a fresh dot), wait, free
//                   the stage, then promote the dot into a second register accumulator with one
//                   mul.rn and one fma.rn — the reference's `mul.f32` + `fma.rn.f32`.  The two
//                   consumers drift apart, so one promotes while the other's wgmmas run.  (Issuing
//                   K block kb + 1 into a second dot fragment before promoting kb, with the
//                   producer's registers handed over by setmaxnreg, measured no faster on the
//                   shapes of scripts/microbench.py fp8 — H100 SXM at a 400 W limit.)
// BN = 128 makes the weight scale one scalar per K block per tile.
//
// Every output element sees the same operations in the same order whatever the tile assignment,
// grid size or problem size: its dot per K block reads only its own row of A and column of B
// (rows and columns past M / N are zero-filled by TMA and never stored), and the promotion is
// element-wise.  Only the hardware's reduced-precision accumulation inside the 128-deep dot
// differs from an fp32 dot of exact products (kernel.py's own dot depends on the autotuned config).
//
// Epilogues: fp32 Y (fp8_gemm with the default dtype), or bf16 Y with an optional bias added
// after the rounding, bf16(float(bf16(acc)) + float(bias)) — `y = fp8_gemm(...).to(bfloat16);
// y += bias` of module_utils.py:42-44 in one pass.
#include "tc.cuh"

namespace llmc {
namespace {

using namespace tc;

constexpr int kBM = 128, kBN = 128, kBK = 128;
constexpr int kStages = 6;
constexpr int kTileBytes = kBM * kBK;                  // 16 KB of e4m3 (kBN == kBM)
constexpr int kStageBytes = 2 * kTileBytes;            // 32 KB
constexpr int kSmemBytes = ring_smem_bytes(kStages * kStageBytes);
constexpr int kThreads = 384;

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

template <bool kBf16Out>
__global__ void __launch_bounds__(kThreads, 1)
fp8_block_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const Fp8GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  // The ring is reached only through TMA and wgmma descriptors, so the generic address costs
  // nothing here.  tc::ring_base and tc::Ring's init, waits and release are not used: with either,
  // ptxas schedules the descriptor setup between the fence and the first wgmma of each K block,
  // which the wgmma_wait<0> per K block serialises (5-13 % slower at M = 4096 / 16384 with
  // DeepSeek-V3 and Llama-3-8B widths, H100 SXM at 700 W).
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
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
        int m_blk, n_blk;
        grouped_tile(u, p.m_tiles, p.n_tiles, p.gn, m_blk, n_blk);
        for (int kb = 0; kb < p.kb_total; ++kb) {
          mbar_wait(&empty_bar[ps.stage], ps.phase ^ 1);
          uint8_t* a_dst = smem + ps.stage * kStageBytes;
          mbar_expect_tx(&full_bar[ps.stage], kStageBytes);
          tma_load_2d(a_dst, &tmA, &full_bar[ps.stage], kb * kBK, m_blk * kBM);
          tma_load_2d(a_dst + kTileBytes, &tmB, &full_bar[ps.stage], kb * kBK, n_blk * kBN);
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
  float d[64];                                   // the dot of one K block
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  for (int u = blockIdx.x; u < p.num_tiles; u += gridDim.x) {
    int m_blk, n_blk;
    grouped_tile(u, p.m_tiles, p.n_tiles, p.gn, m_blk, n_blk);
    const int64_t row0 = static_cast<int64_t>(m_blk) * kBM + c * 64;
    // this thread's two fragment rows (layout at wgmma_m64n128k16_bf16); rows past M read the
    // scale of row M - 1 — their results are never stored
    const int64_t r_lo = row0 + (tid >> 5) * 16 + (lane >> 2);
    const float* as_lo = p.a_s + min(r_lo, p.M - 1) * p.kb_total;
    const float* as_hi = p.a_s + min(r_lo + 8, p.M - 1) * p.kb_total;
    const float* bs = p.b_s + static_cast<int64_t>(n_blk) * p.kb_total;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < p.kb_total; ++kb) {
      const float sa0 = __ldg(as_lo + kb), sa1 = __ldg(as_hi + kb), sb = __ldg(bs + kb);
      mbar_wait(&full_bar[ps.stage], ps.phase);
      wgmma_fence();
      const uint32_t a_addr = smem_u32(smem + ps.stage * kStageBytes);
      const uint32_t b_addr = a_addr + kTileBytes;
#pragma unroll
      for (int k = 0; k < kBK / 32; ++k) {
        const uint64_t adesc = make_smem_desc(a_addr + c * 64 * 128 + k * 32, 16, 1024);
        const uint64_t bdesc = make_smem_desc(b_addr + k * 32, 16, 1024);
        wgmma_m64n128k32_e4m3(d, adesc, bdesc, k > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_acc(d);
      if (tid == 0) mbar_arrive(&empty_bar[ps.stage]);
      ps.advance();
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
    }

    // ---- epilogue straight from the registers ----
    const int64_t col0 = static_cast<int64_t>(n_blk) * kBN;
    if constexpr (kBf16Out) {
      if (p.bias == nullptr) {
        store_linear_m64n128<LLMC_BF16>(acc, row0, col0, p.M, p.N, p.N, nullptr, p.out);
      } else {
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
    } else {
      store_f32_m64n128(acc, row0, col0, p.M, p.N, p.N, static_cast<float*>(p.out));
    }
  }
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
  CUtensorMap tmA, tmB;
  if (int rc = encode_tmap_2d(&tmA, a, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, M, K, K, kBM, kBK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  if (int rc = encode_tmap_2d(&tmB, b, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, N, K, K, kBN, kBK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  Fp8GemmParams p{};
  p.a_s = a_s; p.b_s = b_s; p.bias = bias; p.out = out;
  p.M = M; p.N = N;
  p.kb_total = static_cast<int>(K / kBK);
  p.m_tiles = static_cast<int>(m_tiles);
  p.n_tiles = static_cast<int>(n_tiles);
  p.num_tiles = static_cast<int>(m_tiles * n_tiles);
  p.gn = l2_group_width(static_cast<int64_t>(kBN) * K, p.n_tiles);   // one n-tile's weight bytes
  p.bias_dt = bias_dtype;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return launch_persistent(out_dtype == LLMC_BF16 ? fp8_block_gemm_kernel<true>
                                                  : fp8_block_gemm_kernel<false>,
                           p.num_tiles, kThreads, kSmemBytes, st, tmA, tmB, p);
}
