// tf32.cu — fp32-accurate rank-K updates on tensor cores ("3xTF32").
//
//   C[M,N]  <-  C - A * B      (mode 0)      or      C <- A * B      (mode 1)
//
// with fp32 A, B given as pre-split pairs (hi = tf32(x), lo = tf32(x - hi)) and the product
// evaluated as  A_hi*B_hi + A_lo*B_hi + A_hi*B_lo  (three tf32 MMAs accumulating into the same
// fp32 accumulators; the dropped A_lo*B_lo term is ~2^-22 relative).  This is the workhorse for
// every fp32 GEMM-shaped step of GPTQ that the reference runs as cuBLAS SGEMM / cuSOLVER:
//   * W[:, i2:] -= Err1 @ Hinv[i1:i2, i2:]                        (gptq.py:244)
//   * the trailing updates of the blocked Cholesky and of the triangular inverse that replace
//     torch.linalg.cholesky / cholesky_inverse / cholesky(upper) (gptq.py:172-174).
// K is small (128 per call), so these are read-modify-write sweeps over C.
//
// Both operands are K-major: element (i, k) at base[i*ld + k] (i indexes M or N, K contiguous),
// the only layout Hopper's tf32 wgmma reads.  The sweep keeps the split of Err1 and of Hinv^T and
// the Cholesky inverse keeps L^-T, so every operand is already held that way.
// Structure: one TMA producer thread fills a 3-stage tc::Ring of 128B-swizzled tiles (mbarrier
// transaction counts); two consumer warpgroups compute a 128 x 128 tile on wgmma with fp32
// register accumulators and write it back through store_result.
#include "tc.cuh"

namespace llmc {

using namespace tc;

namespace t3 {

constexpr int BM = 128, BN = 128, BK = 32;     // BK tf32 elements = 128 bytes
constexpr int kStages = 3;
constexpr int kABytes = BM * BK * 4;             // 16 KB (per hi / lo)
constexpr int kBBytes = BN * BK * 4;             // 16 KB
constexpr int kStageBytes = 2 * (kABytes + kBBytes);   // 64 KB
constexpr int kSmemBytes = ring_smem_bytes(kStages * kStageBytes);
struct Params {
  int64_t M, N;
  int K;
  float* C;
  int64_t ldc;
  float* Chi;            // optional: tf32 split of the result (same ld)
  float* Clo;
  int mode;              // 0: C -= A*B ; 1: C = A*B
  int tri;               // 0 all tiles; 1 only tiles touching the lower triangle (col <= row)
  int n_tiles_n, n_tiles_m;
  int num_units;
  int64_t row_off, col_off;   // global (row, col) of C[0][0] for the triangle test
  int64_t split_rows, split_cols;   // Chi/Clo are written where row < split_rows or col < split_cols
};

__device__ __forceinline__ void decode(const Params& p, int u, int& m_blk, int& n_blk) {
  if (!p.tri) {
    n_blk = u % p.n_tiles_n;
    m_blk = u / p.n_tiles_n;
    return;
  }
  // lower-triangle tiles of row-block mi: n_blk in [0, cnt(mi)) with
  // cnt = number of BN-wide column tiles whose first column <= last row of the block
  int mi = 0;
  for (;; ++mi) {
    const int64_t last_row = p.row_off + static_cast<int64_t>(mi) * BM + BM - 1;
    int64_t cnt = (last_row - p.col_off) / BN + 1;
    if (last_row < p.col_off) cnt = 0;
    if (cnt > p.n_tiles_n) cnt = p.n_tiles_n;
    if (u < cnt) break;
    u -= static_cast<int>(cnt);
  }
  m_blk = mi;
  n_blk = u;
}

__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// Stores the result pair (v0, v1) of C[row][col], C[row][col + 1] (the second only if col + 1 < N),
// and its tf32 split where asked.  mode 0 and not `folded`: v0, v1 are the products and are
// subtracted from C here; otherwise they are the final values.
__device__ __forceinline__ void store_result(const Params& p, int64_t row, int64_t col, float v0,
                                             float v1, bool folded) {
  const bool pair = col + 1 < p.N;
  float* cp = p.C + row * p.ldc + col;
  const bool vec = pair && (reinterpret_cast<uintptr_t>(cp) & 7) == 0;
  if (p.mode == 0 && !folded) {
    if (vec) {
      const float2 o = *reinterpret_cast<const float2*>(cp);
      v0 = o.x - v0;
      v1 = o.y - v1;
    } else {
      v0 = cp[0] - v0;
      if (pair) v1 = cp[1] - v1;
    }
  }
  if (vec) *reinterpret_cast<float2*>(cp) = make_float2(v0, v1);
  else {
    cp[0] = v0;
    if (pair) cp[1] = v1;
  }
  if (p.Chi != nullptr && (row < p.split_rows || col < p.split_cols)) {
    float* hp = p.Chi + row * p.ldc + col;
    float* lp = p.Clo + row * p.ldc + col;
    const float2 s0 = tf32_split(v0), s1 = tf32_split(v1);
    if (vec && ((reinterpret_cast<uintptr_t>(hp) | reinterpret_cast<uintptr_t>(lp)) & 7) == 0) {
      *reinterpret_cast<float2*>(hp) = make_float2(s0.x, s1.x);
      *reinterpret_cast<float2*>(lp) = make_float2(s0.y, s1.y);
    } else {
      hp[0] = s0.x;
      lp[0] = s0.y;
      if (pair) {
        hp[1] = s1.x;
        lp[1] = s1.y;
      }
    }
  }
}

// Warpgroup 0 is the TMA producer (one thread), warpgroups 1 and 2 each own 64 rows x 128 columns
// of the 128 x 128 tile and issue wgmma m64n128k8 straight from the swizzled ring: a 32-float
// row is one 128-byte swizzle span, so k8 step s is +32 bytes in the descriptor.  Per k8 step
// three wgmmas into one zeroed accumulator, hi*hi, lo*hi, hi*lo (kSwap: hi*hi, hi*lo, lo*hi, see
// Tf32x3Update::transpose), k ascending; the epilogue then rounds C - acc once.  A consumer keeps
// one wgmma group in flight and frees a stage once the group that read it has retired.
constexpr int kWgThreads = 384;

template <bool kSwap>
__global__ void __launch_bounds__(kWgThreads, 1)
tf32x3_wgmma_kernel(const __grid_constant__ CUtensorMap tmAhi, const __grid_constant__ CUtensorMap tmAlo,
                    const __grid_constant__ CUtensorMap tmBhi, const __grid_constant__ CUtensorMap tmBlo,
                    const Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = ring_base(smem_raw);
  const Ring<kStages> ring(smem + kStages * kStageBytes);
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int kb_total = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmAhi); prefetch_tmap(&tmAlo); prefetch_tmap(&tmBhi); prefetch_tmap(&tmBlo);
    ring.init(1, 2);                  // empty: one arrive per consumer warpgroup
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (tid == 0) {
      PipeState<kStages> ps;
      for (int u = blockIdx.x; u < p.num_units; u += gridDim.x) {
        int m_blk, n_blk;
        decode(p, u, m_blk, n_blk);
        for (int kb = 0; kb < kb_total; ++kb) {
          ring.wait_empty(ps);
          uint8_t* ahi = smem + ps.stage * kStageBytes;
          uint64_t* bar = &ring.full[ps.stage];
          ring.expect_tx(ps, kStageBytes);
          tma_load_2d(ahi, &tmAhi, bar, kb * BK, m_blk * BM);
          tma_load_2d(ahi + kABytes, &tmAlo, bar, kb * BK, m_blk * BM);
          tma_load_2d(ahi + 2 * kABytes, &tmBhi, bar, kb * BK, n_blk * BN);
          tma_load_2d(ahi + 2 * kABytes + kBBytes, &tmBlo, bar, kb * BK, n_blk * BN);
          ps.advance();
        }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup c owns rows 64 c .. 64 c + 63 =====================
  const int c = wg - 1;
  const int lane = tid & 31, g = lane >> 2, t = lane & 3;
  PipeState<kStages> ps;
  for (int u = blockIdx.x; u < p.num_units; u += gridDim.x) {
    int m_blk, n_blk;
    decode(p, u, m_blk, n_blk);
    const int64_t row0 = static_cast<int64_t>(m_blk) * BM + c * 64;
    const int64_t col0 = static_cast<int64_t>(n_blk) * BN;
    if (p.mode == 0) {
      // pull this warpgroup's 64 x 128 block of C into L2 while the MMAs run: per row four
      // 32-column segments, the first and last column of each (a segment spans at most two lines)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int q = 2 * tid + r;                // (row, segment) = (q / 4, q % 4)
        const int64_t row = row0 + (q >> 2), c0 = col0 + 32 * (q & 3);
        if (row < p.M && c0 < p.N) {
          const int64_t last = (c0 + 31 < p.N ? c0 + 31 : p.N - 1);
          prefetch_l2(p.C + row * p.ldc + c0);
          prefetch_l2(p.C + row * p.ldc + last);
        }
      }
    }
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < kb_total; ++kb) {
      ring.wait_full(ps);
      wgmma_fence();
      const uint32_t ahi = smem_u32(smem + ps.stage * kStageBytes) + c * 64 * 128, alo = ahi + kABytes;
      const uint32_t bhi = smem_u32(smem + ps.stage * kStageBytes) + 2 * kABytes, blo = bhi + kBBytes;
#pragma unroll
      for (int s = 0; s < BK / 8; ++s) {
        const uint64_t dah = make_smem_desc(ahi + s * 32, 16, 1024), dal = make_smem_desc(alo + s * 32, 16, 1024);
        const uint64_t dbh = make_smem_desc(bhi + s * 32, 16, 1024), dbl = make_smem_desc(blo + s * 32, 16, 1024);
        wgmma_m64n128k8_tf32(acc, dah, dbh);
        if constexpr (!kSwap) {
          wgmma_m64n128k8_tf32(acc, dal, dbh);
          wgmma_m64n128k8_tf32(acc, dah, dbl);
        } else {
          wgmma_m64n128k8_tf32(acc, dah, dbl);
          wgmma_m64n128k8_tf32(acc, dal, dbh);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                           // the group that read stage `prev` has retired
      if (prev >= 0 && tid == 0) ring.release(prev);
      prev = ps.stage;
      ps.advance();
    }
    wgmma_wait<0>();
    fence_acc(acc);
    if (prev >= 0 && tid == 0) ring.release(prev);

    // ---- epilogue: acc[4 j + 2 i + e] = C[row 16 w + g + 8 i][col 8 j + 2 t + e] ----
    // A block inside C with 8-byte aligned pairs is read whole before the first store and folded
    // into the accumulators (C - acc, one rounding); the stores could alias the reads, so
    // interleaved the compiler would wait out one memory round trip per element pair.  Ragged or
    // misaligned blocks read each pair right before its store.
    const int64_t rw = row0 + 16 * (tid >> 5) + g;
    const bool folded = p.mode == 0 && row0 + 64 <= p.M && col0 + BN <= p.N && (p.ldc & 1) == 0 &&
                        (reinterpret_cast<uintptr_t>(p.C) & 7) == 0;
    if (folded) {
      float2 old[16][2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float* cp = p.C + (rw + 8 * i) * p.ldc + col0 + 2 * t;
#pragma unroll
        for (int j = 0; j < 16; ++j) old[j][i] = *reinterpret_cast<const float2*>(cp + 8 * j);
      }
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          acc[4 * j + 2 * i] = old[j][i].x - acc[4 * j + 2 * i];
          acc[4 * j + 2 * i + 1] = old[j][i].y - acc[4 * j + 2 * i + 1];
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int64_t row = rw + 8 * i;
      if (row >= p.M) continue;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int64_t col = col0 + 8 * j + 2 * t;
        if (col >= p.N) continue;
        store_result(p, row, col, acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1], folded);
      }
    }
  }
}

__global__ void __launch_bounds__(256)
split_tf32_kernel(const float* __restrict__ x, int64_t rows, int64_t cols, int64_t ld,
                  float* __restrict__ hi, float* __restrict__ lo, int64_t ld_out) {
  const int64_t total = rows * cols;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols, c = i - r * cols;
    const float2 s = tf32_split(x[r * ld + c]);
    hi[r * ld_out + c] = s.x;
    lo[r * ld_out + c] = s.y;
  }
}

// hi/lo[c * ld_out + r] = tf32_split(x[r * ld + c]): 32 x 32 tiles through shared memory, so
// both the reads and the writes are row segments
__global__ void __launch_bounds__(256)
split_tf32_t_kernel(const float* __restrict__ x, int64_t rows, int64_t cols, int64_t ld,
                    float* __restrict__ hi, float* __restrict__ lo, int64_t ld_out) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t r0 = static_cast<int64_t>(blockIdx.y) * 32, c0 = static_cast<int64_t>(blockIdx.x) * 32;
  for (int i = ty; i < 32; i += 8)
    if (r0 + i < rows && c0 + tx < cols) tile[i][tx] = x[(r0 + i) * ld + c0 + tx];
  __syncthreads();
  for (int i = ty; i < 32; i += 8)
    if (c0 + i < cols && r0 + tx < rows) {
      const float2 s = tf32_split(tile[tx][i]);
      hi[(c0 + i) * ld_out + r0 + tx] = s.x;
      lo[(c0 + i) * ld_out + r0 + tx] = s.y;
    }
}

}  // namespace t3

// One 3xTF32 update (Tf32x3Update, tc.cuh).  The split of the result can be narrowed to C's first
// rows or columns (multiples of 32): the blocked Cholesky uses this to get the split of the *next*
// panel for free from the trailing update.
// one_tile_per_cta: grid = number of tiles, every CTA computes one tile and exits.  Bulk
// updates launched on a LOW-priority stream this way give their SMs back at tile granularity
// (one 128 x 128 tile), so the short kernels of a latency-bound chain on a high-priority stream (blocked
// Cholesky look-ahead, chol.cu) never wait behind a persistent grid that fills every SM.
int tf32x3_update(const Tf32x3Update& u, cudaStream_t st) {
  using namespace t3;
  if (u.M <= 0 || u.N <= 0 || u.K <= 0) return LLMC_OK;
  if ((u.a.ld % 4) || (u.b.ld % 4) || !aligned16(u.a.hi) || !aligned16(u.a.lo) ||
      !aligned16(u.b.hi) || !aligned16(u.b.lo)) {
    set_last_error("tf32x3_update: operands need 16-byte aligned bases and ld %% 4 == 0");
    return LLMC_EALIGN;
  }
  if (u.c_split.hi != nullptr && u.c_split.ld != u.ldc) {
    set_last_error("tf32x3_update: the split of the result must have the result's ld");
    return LLMC_EINVAL;
  }
  // both halves of an operand with `rows` M or N indices, in box_rows x BK boxes (BK fp32 = one
  // 128-byte swizzle span)
  auto encode = [&](CUtensorMap (&tm)[2], const SplitOperand& x, int64_t rows, uint32_t box_rows) -> int {
    for (int h = 0; h < 2; ++h) {
      const int rc = encode_tmap_2d(&tm[h], h ? x.lo : x.hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, rows,
                                    u.K, x.ld, box_rows, BK, CU_TENSOR_MAP_SWIZZLE_128B);
      if (rc) return rc;
    }
    return LLMC_OK;
  };
  CUtensorMap ta[2], tb[2];
  if (int rc = encode(ta, u.a, u.M, BM)) return rc;
  if (int rc = encode(tb, u.b, u.N, BN)) return rc;
  Params p{};
  p.M = u.M; p.N = u.N; p.K = static_cast<int>(u.K); p.C = u.c; p.ldc = u.ldc;
  p.Chi = u.c_split.hi; p.Clo = u.c_split.lo;
  p.mode = u.assign ? 1 : 0; p.tri = u.lower ? 1 : 0; p.row_off = u.row_off; p.col_off = u.col_off;
  p.split_rows = u.split_rows; p.split_cols = u.split_cols;
  p.n_tiles_m = static_cast<int>((u.M + BM - 1) / BM);
  p.n_tiles_n = static_cast<int>((u.N + BN - 1) / BN);
  if (!u.lower) {
    p.num_units = p.n_tiles_m * p.n_tiles_n;
  } else {
    long units = 0;
    for (int mi = 0; mi < p.n_tiles_m; ++mi) {
      const int64_t last_row = u.row_off + static_cast<int64_t>(mi) * BM + BM - 1;
      int64_t cnt = last_row < u.col_off ? 0 : (last_row - u.col_off) / BN + 1;
      if (cnt > p.n_tiles_n) cnt = p.n_tiles_n;
      units += cnt;
    }
    p.num_units = static_cast<int>(units);
  }
  if (p.num_units == 0) return LLMC_OK;
  const Units units{p.num_units, u.one_tile_per_cta};
  return launch_persistent(u.transposed ? tf32x3_wgmma_kernel<true> : tf32x3_wgmma_kernel<false>, units,
                           kWgThreads, kSmemBytes, st, ta[0], ta[1], tb[0], tb[1], p);
}

int split_tf32(const float* x, int64_t rows, int64_t cols, int64_t ld, float* hi, float* lo,
               int64_t ld_out, cudaStream_t st) {
  if (rows <= 0 || cols <= 0) return LLMC_OK;
  int64_t blocks = (rows * cols + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  t3::split_tf32_kernel<<<(int)blocks, 256, 0, st>>>(x, rows, cols, ld, hi, lo, ld_out);
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

int split_tf32_transposed(const float* x, int64_t rows, int64_t cols, int64_t ld, float* hi, float* lo,
                          int64_t ld_out, cudaStream_t st) {
  if (rows <= 0 || cols <= 0) return LLMC_OK;
  const dim3 grid(static_cast<unsigned>((cols + 31) / 32), static_cast<unsigned>((rows + 31) / 32));
  t3::split_tf32_t_kernel<<<grid, 256, 0, st>>>(x, rows, cols, ld, hi, lo, ld_out);
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

}  // namespace llmc

using namespace llmc;

// Exported for unit tests and as a general fp32-accurate tensor-core GEMM building block.
extern "C" int llmc_split_tf32(const float* x, int64_t rows, int64_t cols, int64_t ld, float* hi,
                               float* lo, void* stream) {
  LLMC_CHECK_ARG(x && hi && lo && rows >= 0 && cols >= 0 && ld >= cols, "split_tf32: bad argument");
  return split_tf32(x, rows, cols, ld, hi, lo, ld, static_cast<cudaStream_t>(stream));
}

extern "C" int llmc_gemm_f32x3(const float* a_hi, const float* a_lo, int64_t lda, const float* b_hi,
                               const float* b_lo, int64_t ldb, float* c, int64_t ldc, int64_t M,
                               int64_t N, int64_t K, int mode, int lower_only, void* stream) {
  LLMC_CHECK_ARG(a_hi && a_lo && b_hi && b_lo && c, "gemm_f32x3: null pointer");
  LLMC_CHECK_ARG(M >= 0 && N >= 0 && K > 0 && K % 8 == 0 && K <= (1 << 20), "gemm_f32x3: bad shape (K %% 8 == 0)");
  LLMC_CHECK_ARG(mode == 0 || mode == 1, "gemm_f32x3: mode must be 0 (C -= AB) or 1 (C = AB)");
  Tf32x3Update u{{a_hi, a_lo, lda}, {b_hi, b_lo, ldb}, c, ldc, M, N, K};
  if (mode == 1) u.overwrite();
  if (lower_only) u.lower_tiles(0, 0);
  return tf32x3_update(u, static_cast<cudaStream_t>(stream));
}
