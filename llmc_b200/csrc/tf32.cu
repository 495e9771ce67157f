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
// Operand layouts (per operand flag):
//   K-major : element (i, k) at base[i*ld + k]   (rows = M or N index, K contiguous)
//   MN-major: element (i, k) at base[k*ld + i]   (rows = K index, M or N contiguous)
// The GPTQ weight update has BOTH operands MN-major, which Hopper's wgmma cannot read for tf32
// (tf32 wgmma operands must be K-major), so the MMAs are warp-level mma.sync m16n8k8 whose
// fragments are gathered from shared memory in either layout.
// Structure: one TMA producer warp fills a 3-stage ring of 128B-swizzled tiles (mbarrier
// transaction counts); eight MMA warps (2 x 4, 64 x 32 each) compute a 128 x 128 tile with fp32
// register accumulators and write it back with the fused epilogue.
#include "tc.cuh"

namespace llmc {

using namespace tc;

namespace t3 {

constexpr int BM = 128, BN = 128, BK = 32;     // BK tf32 elements = 128 bytes
constexpr int kStages = 3;
constexpr int kABytes = BM * BK * 4;             // 16 KB (per hi / lo)
constexpr int kBBytes = BN * BK * 4;             // 16 KB
constexpr int kStageBytes = 2 * (kABytes + kBBytes);   // 64 KB
constexpr int kBoxBytes = 32 * BK * 4;           // MN-major box: 32 MN x 32 K rows = 4 KB
constexpr int kSmemBytes = kStages * kStageBytes + 1024 + 256;
constexpr int kMmaWarps = 8;
constexpr int kThreads = (kMmaWarps + 1) * 32;   // + the TMA warp
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

__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// byte offset of element (i, k) inside an operand tile as TMA wrote it (SWIZZLE_128B: 16-byte
// chunk c of a 128-byte row r sits at chunk c ^ (r & 7))
template <bool kMn>
__device__ __forceinline__ uint32_t tile_off(int i, int k) {
  if constexpr (!kMn)   // rows = i, 32 k per 128-byte row
    return i * 128 + ((((k >> 2) ^ (i & 7)) << 4) | ((k & 3) << 2));
  else                  // boxes of 32 i; rows = k
    return (i >> 5) * kBoxBytes + k * 128 + (((((i & 31) >> 2) ^ (k & 7)) << 4) | ((i & 3) << 2));
}

__device__ __forceinline__ uint32_t lds_u32(const uint8_t* base, uint32_t off) {
  return *reinterpret_cast<const uint32_t*>(base + off);
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, "
      "{%8, %9}, {%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <bool kAmn, bool kBmn>
__global__ void __launch_bounds__(kThreads, 1)
tf32x3_kernel(const __grid_constant__ CUtensorMap tmAhi, const __grid_constant__ CUtensorMap tmAlo,
              const __grid_constant__ CUtensorMap tmBhi, const __grid_constant__ CUtensorMap tmBlo,
              const Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty_bar = full_bar + kStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kb_total = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmAhi); prefetch_tmap(&tmAlo); prefetch_tmap(&tmBhi); prefetch_tmap(&tmBlo);
    for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kMmaWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kMmaWarps) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int u = blockIdx.x; u < p.num_units; u += gridDim.x) {
        int m_blk, n_blk;
        decode(p, u, m_blk, n_blk);
        for (int kb = 0; kb < kb_total; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* ahi = smem + stage * kStageBytes;
          uint8_t* alo = ahi + kABytes;
          uint8_t* bhi = alo + kABytes;
          uint8_t* blo = bhi + kBBytes;
          mbar_expect_tx(&full_bar[stage], kStageBytes);
          if constexpr (!kAmn) {
            tma_load_2d(ahi, &tmAhi, &full_bar[stage], kb * BK, m_blk * BM);
            tma_load_2d(alo, &tmAlo, &full_bar[stage], kb * BK, m_blk * BM);
          } else {
#pragma unroll
            for (int i = 0; i < BM / 32; ++i) {
              tma_load_2d(ahi + i * kBoxBytes, &tmAhi, &full_bar[stage], m_blk * BM + i * 32, kb * BK);
              tma_load_2d(alo + i * kBoxBytes, &tmAlo, &full_bar[stage], m_blk * BM + i * 32, kb * BK);
            }
          }
          if constexpr (!kBmn) {
            tma_load_2d(bhi, &tmBhi, &full_bar[stage], kb * BK, n_blk * BN);
            tma_load_2d(blo, &tmBlo, &full_bar[stage], kb * BK, n_blk * BN);
          } else {
#pragma unroll
            for (int i = 0; i < BN / 32; ++i) {
              tma_load_2d(bhi + i * kBoxBytes, &tmBhi, &full_bar[stage], n_blk * BN + i * 32, kb * BK);
              tma_load_2d(blo + i * kBoxBytes, &tmBlo, &full_bar[stage], n_blk * BN + i * 32, kb * BK);
            }
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== MMA warps: warp (wm, wn) owns rows 64 wm .. +63, cols 32 wn .. +31 =====
  const int wm = warp >> 2, wn = warp & 3;
  const int g = lane >> 2, t = lane & 3;
  int stage = 0;
  uint32_t phase = 0;
  for (int u = blockIdx.x; u < p.num_units; u += gridDim.x) {
    int m_blk, n_blk;
    decode(p, u, m_blk, n_blk);
    float acc[4][4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;
    for (int kb = 0; kb < kb_total; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint8_t* ahi = smem + stage * kStageBytes;
      const uint8_t* alo = ahi + kABytes;
      const uint8_t* bhi = alo + kABytes;
      const uint8_t* blo = bhi + kBBytes;
#pragma unroll 1
      for (int kk = 0; kk < BK; kk += 8) {
        uint32_t fbh[4][2], fbl[4][2];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int j = wn * 32 + nt * 8 + g;
          const uint32_t o0 = tile_off<kBmn>(j, kk + t), o1 = tile_off<kBmn>(j, kk + t + 4);
          fbh[nt][0] = lds_u32(bhi, o0); fbh[nt][1] = lds_u32(bhi, o1);
          fbl[nt][0] = lds_u32(blo, o0); fbl[nt][1] = lds_u32(blo, o1);
        }
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {
          const int i0 = wm * 64 + mt * 16 + g;
          const uint32_t o0 = tile_off<kAmn>(i0, kk + t), o1 = tile_off<kAmn>(i0 + 8, kk + t);
          const uint32_t o2 = tile_off<kAmn>(i0, kk + t + 4), o3 = tile_off<kAmn>(i0 + 8, kk + t + 4);
          const uint32_t fah[4] = {lds_u32(ahi, o0), lds_u32(ahi, o1), lds_u32(ahi, o2), lds_u32(ahi, o3)};
          const uint32_t fal[4] = {lds_u32(alo, o0), lds_u32(alo, o1), lds_u32(alo, o2), lds_u32(alo, o3)};
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            mma_tf32(acc[mt][nt], fah, fbh[nt]);
            mma_tf32(acc[mt][nt], fal, fbh[nt]);
            mma_tf32(acc[mt][nt], fah, fbl[nt]);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }

    // ---- epilogue: fragment element (mt, nt, 2 i + c) = C[row g + 8 i][col 2 t + c] ----
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int64_t row = static_cast<int64_t>(m_blk) * BM + wm * 64 + mt * 16 + g + 8 * i;
        if (row >= p.M) continue;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int64_t col = static_cast<int64_t>(n_blk) * BN + wn * 32 + nt * 8 + 2 * t;
          if (col >= p.N) continue;
          const bool pair = col + 1 < p.N;
          float* cp = p.C + row * p.ldc + col;
          const bool vec = pair && (reinterpret_cast<uintptr_t>(cp) & 7) == 0;
          float v0 = acc[mt][nt][2 * i], v1 = acc[mt][nt][2 * i + 1];
          if (p.mode == 0) {
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
            const float h0 = to_tf32(v0), h1 = to_tf32(v1);
            hp[0] = h0;
            lp[0] = to_tf32(v0 - h0);
            if (pair) {
              hp[1] = h1;
              lp[1] = to_tf32(v1 - h1);
            }
          }
        }
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
    const float v = x[r * ld + c];
    const float h = to_tf32(v);
    hi[r * ld_out + c] = h;
    lo[r * ld_out + c] = to_tf32(v - h);
  }
}

}  // namespace t3

// rows x cols fp32 matrix, row stride ld; 128-byte swizzle => box_cols must be 32.
static int encode_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                              uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols) {
  return encode_tmap_2d(out, base, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, rows, cols, ld_elems, box_rows,
                        box_cols, CU_TENSOR_MAP_SWIZZLE_128B);
}

// One 3xTF32 update.  a_mn / b_mn: operand is MN-major (element (i,k) at base[k*ld + i]).
// split_rows / split_cols restrict where the tf32 split of the result (Chi/Clo) is written: rows
// [0, split_rows) and columns [0, split_cols) of C (multiples of 32).  The blocked Cholesky uses
// this to get the split of the *next* panel for free from the trailing update.
int tf32x3_update(const float* Ahi, const float* Alo, int a_mn, int64_t lda, const float* Bhi,
                  const float* Blo, int b_mn, int64_t ldb, float* C, int64_t ldc, int64_t M,
                  int64_t N, int K, int mode, int tri, int64_t row_off, int64_t col_off,
                  float* Chi, float* Clo, cudaStream_t st) {
  return tf32x3_update_ex(Ahi, Alo, a_mn, lda, Bhi, Blo, b_mn, ldb, C, ldc, M, N, K, mode, tri,
                          row_off, col_off, Chi, Clo, INT64_MAX, INT64_MAX, st);
}

int tf32x3_update_ex(const float* Ahi, const float* Alo, int a_mn, int64_t lda, const float* Bhi,
                     const float* Blo, int b_mn, int64_t ldb, float* C, int64_t ldc, int64_t M,
                     int64_t N, int K, int mode, int tri, int64_t row_off, int64_t col_off,
                     float* Chi, float* Clo, int64_t split_rows, int64_t split_cols,
                     cudaStream_t st) {
  return tf32x3_update_grid(Ahi, Alo, a_mn, lda, Bhi, Blo, b_mn, ldb, C, ldc, M, N, K, mode, tri,
                            row_off, col_off, Chi, Clo, split_rows, split_cols, 0, st);
}

// one_tile_per_cta != 0: grid = number of tiles, every CTA computes one tile and exits.  Bulk
// updates launched on a LOW-priority stream this way give their SMs back at tile granularity
// (one 128 x 128 tile), so the short kernels of a latency-bound chain on a high-priority stream (blocked
// Cholesky look-ahead, chol.cu) never wait behind a persistent grid that fills every SM.
int tf32x3_update_grid(const float* Ahi, const float* Alo, int a_mn, int64_t lda, const float* Bhi,
                       const float* Blo, int b_mn, int64_t ldb, float* C, int64_t ldc, int64_t M,
                       int64_t N, int K, int mode, int tri, int64_t row_off, int64_t col_off,
                       float* Chi, float* Clo, int64_t split_rows, int64_t split_cols,
                       int one_tile_per_cta, cudaStream_t st) {
  using namespace t3;
  if (M <= 0 || N <= 0 || K <= 0) return LLMC_OK;
  if ((lda % 4) || (ldb % 4) || !aligned16(Ahi) || !aligned16(Alo) || !aligned16(Bhi) ||
      !aligned16(Blo)) {
    set_last_error("tf32x3_update: operands need 16-byte aligned bases and ld %% 4 == 0");
    return LLMC_EALIGN;
  }
  CUtensorMap tah, tal, tbh, tbl;
  int rc;
  if (!a_mn) {
    if ((rc = encode_tmap_2d_f32(&tah, Ahi, M, K, lda, BM, BK))) return rc;
    if ((rc = encode_tmap_2d_f32(&tal, Alo, M, K, lda, BM, BK))) return rc;
  } else {
    if ((rc = encode_tmap_2d_f32(&tah, Ahi, K, M, lda, BK, 32))) return rc;
    if ((rc = encode_tmap_2d_f32(&tal, Alo, K, M, lda, BK, 32))) return rc;
  }
  if (!b_mn) {
    if ((rc = encode_tmap_2d_f32(&tbh, Bhi, N, K, ldb, BN, BK))) return rc;
    if ((rc = encode_tmap_2d_f32(&tbl, Blo, N, K, ldb, BN, BK))) return rc;
  } else {
    if ((rc = encode_tmap_2d_f32(&tbh, Bhi, K, N, ldb, BK, 32))) return rc;
    if ((rc = encode_tmap_2d_f32(&tbl, Blo, K, N, ldb, BK, 32))) return rc;
  }
  Params p{};
  p.M = M; p.N = N; p.K = K; p.C = C; p.ldc = ldc; p.Chi = Chi; p.Clo = Clo;
  p.mode = mode; p.tri = tri; p.row_off = row_off; p.col_off = col_off;
  p.split_rows = split_rows; p.split_cols = split_cols;
  p.n_tiles_m = static_cast<int>((M + BM - 1) / BM);
  p.n_tiles_n = static_cast<int>((N + BN - 1) / BN);
  if (!tri) {
    p.num_units = p.n_tiles_m * p.n_tiles_n;
  } else {
    long units = 0;
    for (int mi = 0; mi < p.n_tiles_m; ++mi) {
      const int64_t last_row = row_off + static_cast<int64_t>(mi) * BM + BM - 1;
      int64_t cnt = last_row < col_off ? 0 : (last_row - col_off) / BN + 1;
      if (cnt > p.n_tiles_n) cnt = p.n_tiles_n;
      units += cnt;
    }
    p.num_units = static_cast<int>(units);
  }
  if (p.num_units == 0) return LLMC_OK;
  const int grid = (one_tile_per_cta || p.num_units < kNumSMs) ? p.num_units : kNumSMs;
  LLMC_ONCE_PER_DEVICE({
    LLMC_CHECK_CUDA(cudaFuncSetAttribute(tf32x3_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    LLMC_CHECK_CUDA(cudaFuncSetAttribute(tf32x3_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    LLMC_CHECK_CUDA(cudaFuncSetAttribute(tf32x3_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    LLMC_CHECK_CUDA(cudaFuncSetAttribute(tf32x3_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  });
  if (!a_mn && !b_mn) tf32x3_kernel<false, false><<<grid, kThreads, kSmemBytes, st>>>(tah, tal, tbh, tbl, p);
  else if (!a_mn && b_mn) tf32x3_kernel<false, true><<<grid, kThreads, kSmemBytes, st>>>(tah, tal, tbh, tbl, p);
  else if (a_mn && !b_mn) tf32x3_kernel<true, false><<<grid, kThreads, kSmemBytes, st>>>(tah, tal, tbh, tbl, p);
  else tf32x3_kernel<true, true><<<grid, kThreads, kSmemBytes, st>>>(tah, tal, tbh, tbl, p);
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
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

}  // namespace llmc

using namespace llmc;

// Exported for unit tests and as a general fp32-accurate tensor-core GEMM building block.
extern "C" int llmc_split_tf32(const float* x, int64_t rows, int64_t cols, int64_t ld, float* hi,
                               float* lo, void* stream) {
  LLMC_CHECK_ARG(x && hi && lo && rows >= 0 && cols >= 0 && ld >= cols, "split_tf32: bad argument");
  return split_tf32(x, rows, cols, ld, hi, lo, ld, static_cast<cudaStream_t>(stream));
}

extern "C" int llmc_gemm_f32x3(const float* a_hi, const float* a_lo, int a_mn, int64_t lda,
                               const float* b_hi, const float* b_lo, int b_mn, int64_t ldb,
                               float* c, int64_t ldc, int64_t M, int64_t N, int64_t K, int mode,
                               int lower_only, void* stream) {
  LLMC_CHECK_ARG(a_hi && a_lo && b_hi && b_lo && c, "gemm_f32x3: null pointer");
  LLMC_CHECK_ARG(M >= 0 && N >= 0 && K > 0 && K % 8 == 0 && K <= (1 << 20), "gemm_f32x3: bad shape (K %% 8 == 0)");
  LLMC_CHECK_ARG(mode == 0 || mode == 1, "gemm_f32x3: mode must be 0 (C -= AB) or 1 (C = AB)");
  return tf32x3_update(a_hi, a_lo, a_mn, lda, b_hi, b_lo, b_mn, ldb, c, ldc, M, N, (int)K, mode,
                       lower_only, 0, 0, nullptr, nullptr, static_cast<cudaStream_t>(stream));
}
