// gemm_w8a8.cu — the forward of the exported W8A8 linears (VllmRealQuantLinear and its aliases) on
// Hopper INT8 and FP8 tensor cores: both operands stay 8-bit, one scale per row of X and one per
// row of W (a per-tensor scale is a vector of stride 0).
//
//   acc[m, n] = sum_k qx[m, k] * qw[n, k]
//   Y[m, n]   = rT(fmul(fmul(fp32(acc), s_w[n]), s_x[m]) (+ bias[n]))   fp32 ops, one rounding
//
//   INT8  wgmma m64n128k32 s32.s8.s8: the int32 sum is exact (K <= 131056 bounds it by 2^31 for
//         any int8 codes), fp32(acc) is cvt.rn.
//   FP8   wgmma m64n128k32 f32.e4m3.e4m3 with a fresh dot per 128-deep K block, promoted into an
//         fp32 register sum in ascending K order (acc = fadd(acc, dot)) as gemm_fp8.cu does: only
//         the hardware's reduced-precision accumulation inside a 128-deep dot differs from an fp32
//         sum of exact products.
//
// The structure is gemm_fp8.cu's: one persistent, warp-specialised kernel (1 CTA per SM, 3
// warpgroups), a TMA producer filling a ring of 128-byte-swizzled stages (one stage = a 128-deep K
// block of a 128 x 128 tile, 16 KB of X + 16 KB of W, both K-major) in the L2-grouped tile order,
// and two consumer warpgroups of 64 rows each.  The INT8 consumer keeps one wgmma group in flight
// across stages (its accumulator needs no promotion); the FP8 one waits for each K block's dot and
// promotes it.  Rows and columns past M / N and the K tail past K are zero-filled by TMA: every
// output element's arithmetic is independent of M, N, the tile schedule and the grid size.
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

template <bool kFp8, int DT>
__global__ void __launch_bounds__(kThreads, 1)
w8a8_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const W8A8Params p) {
  extern __shared__ uint8_t smem_raw[];
  // the ring is reached only through TMA and wgmma descriptors (as in gemm_fp8.cu)
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
  PipeState<kStages> ps;
  for (int u = blockIdx.x; u < p.num_tiles; u += gridDim.x) {
    int m_blk, n_blk;
    grouped_tile(u, p.m_tiles, p.n_tiles, p.gn, m_blk, n_blk);
    float acc[64];
    if constexpr (kFp8) {
      float d[64];                               // the dot of one K block
#pragma unroll
      for (int i = 0; i < 64; ++i) { acc[i] = 0.f; d[i] = 0.f; }
      for (int kb = 0; kb < p.kb_total; ++kb) {
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
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = fadd_rn(acc[i], d[i]);
      }
    } else {
      int32_t iacc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) iacc[i] = 0;
      int prev = -1;
      for (int kb = 0; kb < p.kb_total; ++kb) {
        mbar_wait(&full_bar[ps.stage], ps.phase);
        wgmma_fence();
        const uint32_t a_addr = smem_u32(smem + ps.stage * kStageBytes);
        const uint32_t b_addr = a_addr + kTileBytes;
#pragma unroll
        for (int k = 0; k < kBK / 32; ++k) {
          const uint64_t adesc = make_smem_desc(a_addr + c * 64 * 128 + k * 32, 16, 1024);
          const uint64_t bdesc = make_smem_desc(b_addr + k * 32, 16, 1024);
          wgmma_m64n128k32_s8(iacc, adesc, bdesc, (kb > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();                         // the group that read stage `prev` has retired
        if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);
        prev = ps.stage;
        ps.advance();
      }
      wgmma_wait<0>();
      fence_acc(iacc);
      if (tid == 0) mbar_arrive(&empty_bar[prev]);   // kb_total >= 1
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = __int2float_rn(iacc[i]);
    }
    const int64_t row0 = static_cast<int64_t>(m_blk) * kBM + c * 64;
    store_w8a8_m64n128<DT>(acc, row0, static_cast<int64_t>(n_blk) * kBN, p);
  }
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
  CUtensorMap tmA, tmB;
  if (int rc = encode_tmap_2d(&tmA, x, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, M, K, K, kBM, kBK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  if (int rc = encode_tmap_2d(&tmB, w, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, N, K, K, kBN, kBK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  W8A8Params p{};
  p.s_x = s_x; p.s_w = s_w; p.s_x_stride = s_x_stride; p.s_w_stride = s_w_stride;
  p.bias = bias; p.out = y;
  p.M = M; p.N = N;
  p.kb_total = static_cast<int>((K + kBK - 1) / kBK);
  p.m_tiles = static_cast<int>(m_tiles);
  p.n_tiles = static_cast<int>(n_tiles);
  p.num_tiles = static_cast<int>(m_tiles * n_tiles);
  p.gn = l2_group_width(static_cast<int64_t>(kBN) * K, p.n_tiles);   // one n-tile's weight bytes
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return launch_persistent(dtype == LLMC_BF16 ? w8a8_gemm_kernel<kFp8, LLMC_BF16>
                                              : w8a8_gemm_kernel<kFp8, LLMC_F16>,
                           p.num_tiles, kThreads, kSmemBytes, st, tmA, tmB, p);
}

}  // namespace
}  // namespace llmc

using namespace llmc;

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
