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
// Hopper's tf32 wgmma reads K-major operands only.  Every caller in the library holds both
// operands K-major (the sweep keeps the split of Err1 and of Hinv^T, the Cholesky inverse keeps
// L^-T), and those calls run on tf32x3_wgmma_kernel.  A call with an MN-major operand (possible
// through llmc_gemm_f32x3 only) runs on tf32x3_kernel, whose warp-level mma.sync m16n8k8 gathers
// its fragments from shared memory in either layout.  Both issue the same three terms per k8
// step in the same order and give the same bits.
// Structure: one TMA producer thread fills a 3-stage tc::Ring of 128B-swizzled tiles (mbarrier
// transaction counts); two consumer warpgroups (wgmma) or eight MMA warps (mma.sync, 2 x 4 of
// 64 x 32) compute a 128 x 128 tile with fp32 register accumulators and write it back with the
// shared epilogue, store_result.
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
constexpr int kSmemBytes = ring_smem_bytes(kStages * kStageBytes);
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

// Operand tiles as TMA wrote them (SWIZZLE_128B: 16-byte chunk c of a 128-byte row r sits at
// chunk c ^ (r & 7)), every tile 1024-byte aligned:
//   K-major : element (i, k) at  i * 128 + (((k / 4) ^ (i % 8)) * 16) + (k % 4) * 4
//   MN-major: element (i, k) at  (i / 32) * kBoxBytes + k * 128 + ((((i % 32) / 4) ^ (k % 8)) * 16) + (i % 4) * 4
// The mma.m16n8k8 tf32 fragments of lane (g = lane / 4, t = lane % 4) are
//   A: a0 = (g, t), a1 = (g + 8, t), a2 = (g, t + 4), a3 = (g + 8, t + 4)     (i, k)
//   B: b0 = (g, t), b1 = (g, t + 4)
// K-major: an 8 x 4 block of tf32 (8 rows of one 16-byte chunk) is, read as b16, exactly one
// ldmatrix 8 x 8 matrix with the (g, t) element in lane 4 g + t, so A is one ldmatrix.x4 and two B
// fragments are another; the 8 row addresses of each matrix hit 8 different chunks (conflict free).
// MN-major: 32-bit loads.  For a k8 step kk (kk % 8 == 0) the swizzle term k % 8 does not depend
// on kk, so each lane's offsets are fixed and a k step only adds kk * 128.
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}

__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// Per-lane byte offsets of this warp's fragments inside an operand tile.
//   A K-major : a[s]  = ldmatrix row address for k8 step s (rows 64 wm + .., mt adds mt * 2048)
//   A MN-major: a[ih] = element (64 wm + g + 8 ih, t); (mt, kh, s) only add constants
//   B K-major : b[s]  = ldmatrix row address for k8 step s (cols 32 wn + .., pair np adds np * 2048)
//   B MN-major: b[nt] = element (32 wn + 8 nt + g, t); kh = 1 is b[nt ^ 2] + 512
template <bool kAmn, bool kBmn>
struct LaneOffsets {
  uint32_t a[4], b[4];
  __device__ __forceinline__ LaneOffsets(int wm, int wn, int lane) {
    const int g = lane >> 2, t = lane & 3, r = lane & 7;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      if constexpr (!kAmn) {
        const int row = wm * 64 + r + 8 * ((lane >> 3) & 1);
        a[s] = row * 128 + (((2 * s + (lane >> 4)) ^ r) << 4);
      } else {
        a[s] = s < 2 ? wm * 2 * kBoxBytes + t * 128 + ((((2 * s + (g >> 2)) ^ t)) << 4) + (g & 3) * 4 : 0;
      }
      if constexpr (!kBmn) {
        const int row = wn * 32 + r + 8 * (lane >> 4);
        b[s] = row * 128 + (((2 * s + ((lane >> 3) & 1)) ^ r) << 4);
      } else {
        b[s] = wn * kBoxBytes + t * 128 + (((2 * s) ^ (g >> 2) ^ t) << 4) + (g & 3) * 4;
      }
    }
  }
};

// A fragment (hi and lo) of k8 step s for the warp's 16-row block mt (both compile-time after
// unrolling)
template <bool kMn>
__device__ __forceinline__ void load_a(uint32_t (&fa)[2][4], uint32_t hi, uint32_t lo,
                                       const uint32_t (&off)[4], int mt, int s) {
  if constexpr (!kMn) {
    ldsm_x4(fa[0], hi + mt * 2048 + off[s]);
    ldsm_x4(fa[1], lo + mt * 2048 + off[s]);
  } else {
#pragma unroll
    for (int q = 0; q < 4; ++q) {   // q = ih + 2 kh
      const int ih = q & 1, kh = q >> 1;
      const uint32_t o = off[ih] + (mt >> 1) * kBoxBytes + kh * 512 + (((mt & 1) ^ kh) << 6) + s * 1024;
      fa[0][q] = lds_u32(hi + o);
      fa[1][q] = lds_u32(lo + o);
    }
  }
}

// B fragments (hi and lo) of k8 step s for the warp's four 8-column blocks
template <bool kMn>
__device__ __forceinline__ void load_b(uint32_t (&fb)[4][2][2], uint32_t hi, uint32_t lo,
                                       const uint32_t (&off)[4], int s) {
  if constexpr (!kMn) {
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t h[4], l[4];
      ldsm_x4(h, hi + np * 2048 + off[s]);
      ldsm_x4(l, lo + np * 2048 + off[s]);
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        fb[2 * np + q][0][0] = h[2 * q]; fb[2 * np + q][0][1] = h[2 * q + 1];
        fb[2 * np + q][1][0] = l[2 * q]; fb[2 * np + q][1][1] = l[2 * q + 1];
      }
    }
  } else {
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const uint32_t o0 = off[nt] + s * 1024, o1 = off[nt ^ 2] + 512 + s * 1024;
      fb[nt][0][0] = lds_u32(hi + o0); fb[nt][0][1] = lds_u32(hi + o1);
      fb[nt][1][0] = lds_u32(lo + o0); fb[nt][1][1] = lds_u32(lo + o1);
    }
  }
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, "
      "{%8, %9}, {%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
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

template <bool kAmn, bool kBmn>
__global__ void __launch_bounds__(kThreads, 1)
tf32x3_kernel(const __grid_constant__ CUtensorMap tmAhi, const __grid_constant__ CUtensorMap tmAlo,
              const __grid_constant__ CUtensorMap tmBhi, const __grid_constant__ CUtensorMap tmBlo,
              const Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = ring_base(smem_raw);
  const Ring<kStages> ring(smem + kStages * kStageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kb_total = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmAhi); prefetch_tmap(&tmAlo); prefetch_tmap(&tmBhi); prefetch_tmap(&tmBlo);
    ring.init(1, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kMmaWarps) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      PipeState<kStages> ps;
      for (int u = blockIdx.x; u < p.num_units; u += gridDim.x) {
        int m_blk, n_blk;
        decode(p, u, m_blk, n_blk);
        for (int kb = 0; kb < kb_total; ++kb) {
          ring.wait_empty(ps);
          uint8_t* ahi = smem + ps.stage * kStageBytes;
          uint8_t* alo = ahi + kABytes;
          uint8_t* bhi = alo + kABytes;
          uint8_t* blo = bhi + kBBytes;
          uint64_t* bar = &ring.full[ps.stage];
          ring.expect_tx(ps, kStageBytes);
          if constexpr (!kAmn) {
            tma_load_2d(ahi, &tmAhi, bar, kb * BK, m_blk * BM);
            tma_load_2d(alo, &tmAlo, bar, kb * BK, m_blk * BM);
          } else {
#pragma unroll
            for (int i = 0; i < BM / 32; ++i) {
              tma_load_2d(ahi + i * kBoxBytes, &tmAhi, bar, m_blk * BM + i * 32, kb * BK);
              tma_load_2d(alo + i * kBoxBytes, &tmAlo, bar, m_blk * BM + i * 32, kb * BK);
            }
          }
          if constexpr (!kBmn) {
            tma_load_2d(bhi, &tmBhi, bar, kb * BK, n_blk * BN);
            tma_load_2d(blo, &tmBlo, bar, kb * BK, n_blk * BN);
          } else {
#pragma unroll
            for (int i = 0; i < BN / 32; ++i) {
              tma_load_2d(bhi + i * kBoxBytes, &tmBhi, bar, n_blk * BN + i * 32, kb * BK);
              tma_load_2d(blo + i * kBoxBytes, &tmBlo, bar, n_blk * BN + i * 32, kb * BK);
            }
          }
          ps.advance();
        }
      }
    }
    return;
  }

  // ===================== MMA warps: warp (wm, wn) owns rows 64 wm .. +63, cols 32 wn .. +31 =====
  const int wm = warp >> 2, wn = warp & 3;
  const int g = lane >> 2, t = lane & 3;
  const LaneOffsets<kAmn, kBmn> off(wm, wn, lane);
  PipeState<kStages> ps;
  for (int u = blockIdx.x; u < p.num_units; u += gridDim.x) {
    int m_blk, n_blk;
    decode(p, u, m_blk, n_blk);
    const int64_t row0 = static_cast<int64_t>(m_blk) * BM + wm * 64;
    const int64_t col0 = static_cast<int64_t>(n_blk) * BN + wn * 32;
    if (p.mode == 0 && col0 < p.N) {
      // pull this warp's 64 x 32 block of C into L2 while the MMAs run: two rows per lane, the
      // first and last column of each (a row segment spans at most two 128-byte lines)
      const int64_t last = (col0 + 31 < p.N ? col0 + 31 : p.N - 1) - col0;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int64_t row = row0 + 2 * lane + r;
        if (row < p.M) {
          prefetch_l2(p.C + row * p.ldc + col0);
          prefetch_l2(p.C + row * p.ldc + col0 + last);
        }
      }
    }
    float acc[4][4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;
    for (int kb = 0; kb < kb_total; ++kb) {
      ring.wait_full(ps);
      // the MMA warps address the ring by 32-bit shared addresses
      const uint32_t ahi = smem_u32(smem + ps.stage * kStageBytes), alo = ahi + kABytes;
      const uint32_t bhi = alo + kABytes, blo = bhi + kBBytes;
      // Fragments are double-buffered: B per k8 step (s), A per (s, 16-row block mt), so the next
      // fragments load while the current ones feed the MMAs.  Every accumulator sees hi*hi,
      // lo*hi, hi*lo per k8 step, k ascending.
      uint32_t fa[2][2][4], fb[2][4][2][2];
      load_b<kBmn>(fb[0], bhi, blo, off.b, 0);
      load_a<kAmn>(fa[0], ahi, alo, off.a, 0, 0);
#pragma unroll
      for (int s = 0; s < BK / 8; ++s) {
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {
          const int q = 4 * s + mt;
          if (mt == 0 && s + 1 < BK / 8) load_b<kBmn>(fb[(s + 1) & 1], bhi, blo, off.b, s + 1);
          if (q + 1 < BK / 2) load_a<kAmn>(fa[(q + 1) & 1], ahi, alo, off.a, (q + 1) & 3, (q + 1) >> 2);
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            mma_tf32(acc[mt][nt], fa[q & 1][0], fb[s & 1][nt][0]);
            mma_tf32(acc[mt][nt], fa[q & 1][1], fb[s & 1][nt][0]);
            mma_tf32(acc[mt][nt], fa[q & 1][0], fb[s & 1][nt][1]);
          }
        }
      }
      // Free the stage only once every MMA thread's reads of it are performed.  ptxas schedules
      // the arrive above MMAs whose fragment loads may still be in flight, and neither the
      // arrive nor a warp sync waits for them; bar.sync does (it orders all prior shared-memory
      // accesses of the participating threads before it).
      asm volatile("bar.sync 1, %0;" ::"n"(kMmaWarps * 32) : "memory");
      if (threadIdx.x == 0) ring.release(ps.stage);
      ps.advance();
    }

    // ---- epilogue: fragment element (mt, nt, 2 i + c) = C[row g + 8 i][col 2 t + c] ----
    // A warp whose 64 x 32 block lies inside C with 8-byte aligned pairs reads all of it before
    // the first store and folds it into the accumulators (C - acc, one rounding as below); the
    // stores could alias the reads, so interleaved the compiler would wait out one memory round
    // trip per element pair.  Ragged or misaligned blocks read each pair right before its store.
    const bool folded = p.mode == 0 && row0 + 64 <= p.M && col0 + 32 <= p.N && (p.ldc & 1) == 0 &&
                        (reinterpret_cast<uintptr_t>(p.C) & 7) == 0;
    if (folded) {
      float2 old[4][2][4];
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float* cp = p.C + (row0 + mt * 16 + g + 8 * i) * p.ldc + col0 + 2 * t;
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) old[mt][i][nt] = *reinterpret_cast<const float2*>(cp + nt * 8);
        }
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            acc[mt][nt][2 * i] = old[mt][i][nt].x - acc[mt][nt][2 * i];
            acc[mt][nt][2 * i + 1] = old[mt][i][nt].y - acc[mt][nt][2 * i + 1];
          }
    }
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int64_t row = row0 + mt * 16 + g + 8 * i;
        if (row >= p.M) continue;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int64_t col = col0 + nt * 8 + 2 * t;
          if (col >= p.N) continue;
          store_result(p, row, col, acc[mt][nt][2 * i], acc[mt][nt][2 * i + 1], folded);
        }
      }
    }
  }
}

// ---- K-major x K-major: wgmma ---------------------------------------------------------------
// Warpgroup 0 is the TMA producer (one thread), warpgroups 1 and 2 each own 64 rows x 128 columns
// of the 128 x 128 tile and issue wgmma m64n128k8 straight from the swizzled ring: a 32-float
// row is one 128-byte swizzle span, so k8 step s is +32 bytes in the descriptor.  Per k8 step
// three wgmmas into one zeroed accumulator, hi*hi, lo*hi, hi*lo (kSwap: hi*hi, hi*lo, lo*hi, see
// Tf32x3Update::transpose), k ascending: the order of tf32x3_kernel's mma.sync.  A consumer keeps
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
    // As in tf32x3_kernel: a block inside C with 8-byte aligned pairs is read whole before the
    // first store and folded into the accumulators; ragged or misaligned blocks read each pair
    // right before its store.
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
  if (u.transposed && (u.a.mn || u.b.mn)) {
    set_last_error("tf32x3_update: a transposed update needs K-major operands");
    return LLMC_EINVAL;
  }
  // both halves of an operand with `rows` M or N indices: K-major boxes are box_rows x BK,
  // MN-major boxes BK x 32 (128-byte swizzle: a box row is 32 fp32)
  auto encode = [&](CUtensorMap (&tm)[2], const SplitOperand& x, int64_t rows, uint32_t box_rows) -> int {
    for (int h = 0; h < 2; ++h) {
      const float* base = h ? x.lo : x.hi;
      const int rc =
          x.mn ? encode_tmap_2d(&tm[h], base, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, u.K, rows, x.ld,
                                BK, 32, CU_TENSOR_MAP_SWIZZLE_128B)
               : encode_tmap_2d(&tm[h], base, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, rows, u.K, x.ld,
                                box_rows, BK, CU_TENSOR_MAP_SWIZZLE_128B);
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
  if (!u.a.mn && !u.b.mn)
    return launch_persistent(u.transposed ? tf32x3_wgmma_kernel<true> : tf32x3_wgmma_kernel<false>, units,
                             kWgThreads, kSmemBytes, st, ta[0], ta[1], tb[0], tb[1], p);
  const auto kern = !u.a.mn ? tf32x3_kernel<false, true>
                            : (!u.b.mn ? tf32x3_kernel<true, false> : tf32x3_kernel<true, true>);
  return launch_persistent(kern, units, kThreads, kSmemBytes, st, ta[0], ta[1], tb[0], tb[1], p);
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

extern "C" int llmc_gemm_f32x3(const float* a_hi, const float* a_lo, int a_mn, int64_t lda,
                               const float* b_hi, const float* b_lo, int b_mn, int64_t ldb,
                               float* c, int64_t ldc, int64_t M, int64_t N, int64_t K, int mode,
                               int lower_only, void* stream) {
  LLMC_CHECK_ARG(a_hi && a_lo && b_hi && b_lo && c, "gemm_f32x3: null pointer");
  LLMC_CHECK_ARG(M >= 0 && N >= 0 && K > 0 && K % 8 == 0 && K <= (1 << 20), "gemm_f32x3: bad shape (K %% 8 == 0)");
  LLMC_CHECK_ARG(mode == 0 || mode == 1, "gemm_f32x3: mode must be 0 (C -= AB) or 1 (C = AB)");
  Tf32x3Update u{{a_hi, a_lo, lda, a_mn != 0}, {b_hi, b_lo, ldb, b_mn != 0}, c, ldc, M, N, K};
  if (mode == 1) u.overwrite();
  if (lower_only) u.lower_tiles(0, 0);
  return tf32x3_update(u, static_cast<cudaStream_t>(stream));
}
