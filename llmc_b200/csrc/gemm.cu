// gemm.cu — K3 (Hessian SYRK) and K6 (fake-quant forward GEMM) on Hopper wgmma tensor cores.
//
// One persistent, warp-specialised kernel template (1 CTA per SM, 3 warpgroups):
//   warpgroup 0     TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring,
//                   mbarrier transaction counts)
//   warpgroups 1-2  consumers: each owns 64 rows of the 128 x 256 tile and issues
//                   wgmma.mma_async m64n128k16 (two per 16-deep K step, one per 128-column half)
//                   with fp32 accumulators in registers, then stores its rows from registers.
// Tile 128(M) x 256(N) x 64(K), 4-stage tc::Ring (48 KB / stage).  A consumer keeps one wgmma
// group in flight and frees a ring stage as soon as the group that read it has retired.
//
//  * GEMM  (llmc_gemm_bf16):  Y[M,N] = X[M,K] . W[N,K]^T (+bias) — both operands K-major.
//      Replaces F.linear in FakeQuantLinear / EffcientFakeQuantLinear.forward
//      (llmc/compression/quantization/module_utils.py:643, 719).
//  * SYRK  (llmc_syrk_accum): H <- H*n/(n+b) + 2/(n+b) * X^T X, X[T,C] row-major so BOTH
//      operands are MN-major views of the same tensor (no transpose pass).  Only tiles touching
//      the upper triangle are computed; split-K partial slabs + a finalize kernel that applies
//      the running-mean scaling and mirrors.  Replaces GPTQ.add_batch (gptq.py:283-290), whose
//      fp32 SGEMM on X.float() has exactly representable bf16/fp16 operands, so an fp32-
//      accumulating tensor-core product differs only by summation order.
//  * grouped GEMM (llmc_moe_gemm_swiglu / llmc_moe_gemm_down): one launch runs every expert of a
//      sparse-MoE layer.  A = the routed rows gathered in expert order, expert e owning rows
//      [offsets[e], offsets[e+1]); B = expert e's weight through its own tensor map (MoeOperands).
//      Same main loop, tile and wgmma as the GEMM; only the unit decode, the B loads and the row
//      bound of the store differ (see decode_moe_unit and tc::moe_load_b).
#include "tc.cuh"

namespace llmc {

using namespace tc;

constexpr int BM = 128, BN = 256, BK = 64;
constexpr int kStages = 4;
constexpr int kABytes = BM * BK * 2;                 // 16 KB
constexpr int kBBytes = BN * BK * 2;                 // 32 KB
constexpr int kStageBytes = kABytes + kBBytes;       // 48 KB
constexpr int kBoxBytes = 64 * 64 * 2;               // SYRK box: 64 tokens x 64 channels
constexpr int kSmemBytes = ring_smem_bytes(kStages * kStageBytes);
constexpr int kThreads = 384;
struct GemmParams {
  int64_t M, N, K;          // GEMM: Y[M,N]; SYRK: M = N = C, K = T
  void* out;                // GEMM: Y (bf16/fp16) ; SYRK: partial slabs fp32 [splits][C][C]
  const void* bias;         // GEMM only, may be null (dtype = out dtype)
  int64_t ld_out;
  int n_tiles_n;            // tiles along N
  int num_units;            // GEMM: tiles ; SYRK: upper tiles * splits
  int num_tiles;            // SYRK: upper tiles
  int splits;               // SYRK split-K factor
  int kb_total;             // k-blocks in K
  int kb_per_split;
  int gn;                   // rasterisation group: n-tiles (GEMM) / m-blocks (SYRK) per group
};

// Operands of the fused GEMM epilogues (see Epilogue).  A kernel argument of its own: grown
// GemmParams fields change the plain GEMM's and the SYRK's register allocation.
struct EpiParams {
  const void* res;          // kEpiResidual: the residual [M, N], may be GemmParams::out
  void* out_k;              // kEpiRopeQkv: k [M, n_k] and v [M, N - n_q - n_k]; q is GemmParams::out
  void* out_v;              // kEpiMlaQkv: k [M, n_q] and the latent [M, n_k]; kEpiMlaKvB: v [M, n_k]
  const void* cosv;         // kEpiRopeQkv: [seq, 128] rotary tables in the output dtype
  const void* sinv;         // kEpiMlaQkv: [seq, 32] fp32
  int64_t n_q, n_k, seq;    // kEpiMlaQkv: n_q = H * 192, n_k = kv_lora; kEpiMlaKvB: H * 192, H * 128
};

// What the GEMM does with a finished tile.  Every fused epilogue first rounds the accumulator to
// the output dtype, as the plain GEMM's store does, so it computes exactly what the plain GEMM
// followed by the block_ops.cu kernel of the same name computes.
enum Epilogue {
  kEpiLinear,     // Y = X W^T (+ bias)
  kEpiRopeQkv,    // W = [Wq; Wk; Wv]: q, k, v to three outputs, rope_kernel applied to q and k
  kEpiSwiGLU,     // W = gate / up interleaved in 128-row blocks: act = silu(gate) * up
  kEpiResidual,   // Y = res + X W^T (add_kernel)
  kEpiMlaQkv,     // W = [Wq; Wkv_a] of MLA: q with each head's pe slice rotated, the latent, and
                  // the rotated k_pe into every head's pe slot of k (store_mla_tile)
  kEpiMlaKvB,     // W = Wkv_b of MLA, one head per n-tile: k_nope into k's nope slots, v apart
};

// The grouped operands: one tensor map per expert weight (AWQ rewrites the expert weights between
// calls, so they cannot be one tensor) and the segment offsets, read from device memory so that the
// host never learns the routing.  A kernel argument of its own, like EpiParams.
struct MoeOperands {
  CUtensorMap tmB[2 * LLMC_MOE_MAX_EXPERTS];   // one per expert linear (tc::moe_load_b)
  MoeSegments seg;
};
// The whole argument list of the grouped kernel fits the 32,764-byte kernel-parameter space of
// CUDA 12.1+ (driver R530+): that is what caps the number of experts.
static_assert(sizeof(CUtensorMap) + sizeof(MoeOperands) + sizeof(GemmParams) <= 32764,
              "LLMC_MOE_MAX_EXPERTS exceeds the kernel-parameter space");

struct Unit {
  int m_blk, n_blk, kb0, kb1, split;
  int e, row0, row_end;     // grouped mode: expert, first A row of the tile, end of its segment
};

template <bool kSyrk>
__device__ __forceinline__ Unit decode_unit(const GemmParams& p, int u) {
  Unit t;
  if constexpr (!kSyrk) {
    grouped_tile(u, p.num_tiles / p.n_tiles_n, p.n_tiles_n, p.gn, t.m_blk, t.n_blk);
    t.kb0 = 0;
    t.kb1 = p.kb_total;
    t.split = 0;
  } else {
    // tile fastest, split slowest: concurrent CTAs stream the same token range (L2 reuse).
    // Tiles are visited in super-rows of `gn` m-blocks, n-major inside a super-row, so the 132
    // tiles of a wave form a compact patch of H and touch ~4.6K channels of X per k-block instead
    // of all C (X is streamed from HBM once per wave).
    int tile = u % p.num_tiles;
    t.split = u / p.num_tiles;
    const int m_tiles = (static_cast<int>(p.M) + BM - 1) / BM;
    int m0 = 0;
    for (;; m0 += p.gn) {
      const int m1 = min(m0 + p.gn, m_tiles);
      int cnt = 0;
      for (int mi = m0; mi < m1; ++mi) cnt += p.n_tiles_n - (mi >> 1);
      if (tile < cnt) break;
      tile -= cnt;
    }
    const int m1 = min(m0 + p.gn, m_tiles);
    int n = m0 >> 1;
    for (;; ++n) {
      const int cnt = min(m1, 2 * n + 2) - m0;     // m-blocks of the group with m/2 <= n
      if (tile < cnt) break;
      tile -= cnt;
    }
    t.m_blk = m0 + tile;
    t.n_blk = n;
    t.kb0 = t.split * p.kb_per_split;
    t.kb1 = min(t.kb0 + p.kb_per_split, p.kb_total);
  }
  return t;
}

// Grouped mode: the tile of unit u (tc::moe_segment_tile); false past the last expert's tiles.
__device__ __forceinline__ bool decode_moe_unit(const GemmParams& p, const MoeOperands& g, int u,
                                                Unit& t) {
  t.kb0 = 0;
  t.kb1 = p.kb_total;
  t.split = 0;
  return moe_segment_tile<BM>(g.seg, u, p.n_tiles_n, p.gn, t.e, t.m_blk, t.n_blk, t.row0, t.row_end);
}

// ---- fused epilogues: this thread's part of the 64-row half tile (fragment layout at
// tc::wgmma_m64n128k16_bf16) whose row 0 is row0 -----------------------------------------------
__device__ __forceinline__ int64_t frag_row(int64_t row0, int i) {
  const int tid = threadIdx.x & 127, lane = threadIdx.x & 31;
  return row0 + (tid >> 5) * 16 + (lane >> 2) + 8 * i;
}

// rope_kernel on one head (head_dim 128) of q or k: acc holds the head's 128 columns, which go to
// out[row][col0 + d] (ld even).  Columns d and d + 64 of a row are fragments j and j + 8 of the same
// thread.  The position of a row is row % seq: chunks hold whole samples.
template <int DT>
__device__ __forceinline__ void store_rope_m64n128(const float (&acc)[64], int64_t row0, int64_t col0,
                                                   int64_t M, const EpiParams& e, int64_t ld,
                                                   void* out) {
  using T = DType<DT>;
  const int lane = threadIdx.x & 31;
  const uint32_t* cosv = static_cast<const uint32_t*>(e.cosv);
  const uint32_t* sinv = static_cast<const uint32_t*>(e.sinv);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int64_t row = frag_row(row0, i);
    if (row >= M) continue;
    const int64_t tab = (row % e.seq) * 64 + (lane & 3);          // 32-bit pairs of [seq, 128]
    uint16_t* o = static_cast<uint16_t*>(out) + row * ld + col0 + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t c1 = __ldg(cosv + tab + 4 * j), s1 = __ldg(sinv + tab + 4 * j);
      const uint32_t c2 = __ldg(cosv + tab + 32 + 4 * j), s2 = __ldg(sinv + tab + 32 + 4 * j);
      float oa[2], ob[2];
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float a = T::rT(acc[4 * j + 2 * i + c]), b = T::rT(acc[4 * (j + 8) + 2 * i + c]);
        const float cs1 = c ? pair_hi<DT>(c1) : pair_lo<DT>(c1);
        const float sn1 = c ? pair_hi<DT>(s1) : pair_lo<DT>(s1);
        const float cs2 = c ? pair_hi<DT>(c2) : pair_lo<DT>(c2);
        const float sn2 = c ? pair_hi<DT>(s2) : pair_lo<DT>(s2);
        oa[c] = fadd_rn(T::rT(fmul_rn(a, cs1)), T::rT(fmul_rn(-b, sn1)));
        ob[c] = fadd_rn(T::rT(fmul_rn(b, cs2)), T::rT(fmul_rn(a, sn2)));
      }
      *reinterpret_cast<uint32_t*>(o + 8 * j) = pack_pair<DT>(oa[0], oa[1]);
      *reinterpret_cast<uint32_t*>(o + 8 * j + 64) = pack_pair<DT>(ob[0], ob[1]);
    }
  }
}

// One 64 x 256 half tile of kEpiRopeQkv: the n-tile's columns lie in one of q, k, v (n_q and n_k
// are multiples of 256); q and k tiles are two heads each.
template <int DT>
__device__ __forceinline__ void store_qkv_tile(const float (&acc0)[64], const float (&acc1)[64],
                                               int64_t row0, int64_t col0, const GemmParams& p,
                                               const EpiParams& e) {
  if (col0 < e.n_q) {
    store_rope_m64n128<DT>(acc0, row0, col0, p.M, e, e.n_q, p.out);
    store_rope_m64n128<DT>(acc1, row0, col0 + 128, p.M, e, e.n_q, p.out);
  } else if (col0 < e.n_q + e.n_k) {
    store_rope_m64n128<DT>(acc0, row0, col0 - e.n_q, p.M, e, e.n_k, e.out_k);
    store_rope_m64n128<DT>(acc1, row0, col0 - e.n_q + 128, p.M, e, e.n_k, e.out_k);
  } else {
    const int64_t nv = p.N - e.n_q - e.n_k, c = col0 - e.n_q - e.n_k;
    store_linear_m64n128<DT>(acc0, row0, c, p.M, nv, nv, nullptr, e.out_v);
    store_linear_m64n128<DT>(acc1, row0, c + 128, p.M, nv, nv, nullptr, e.out_v);
  }
}

// silu_mul_kernel on one 64 x 256 half tile of kEpiSwiGLU: gate in acc0, up in acc1, both for the
// 128 act columns from col0 of act[M, ld].
template <int DT>
__device__ __forceinline__ void store_swiglu_m64n128(const float (&gate)[64], const float (&up)[64],
                                                     int64_t row0, int64_t col0, int64_t M,
                                                     int64_t ld, void* out) {
  using T = DType<DT>;
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int64_t row = frag_row(row0, i);
    if (row >= M) continue;
    uint16_t* o = static_cast<uint16_t*>(out) + row * ld + col0 + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      float v[2];
#pragma unroll
      for (int c = 0; c < 2; ++c)
        v[c] = silu_mul_f32<DT, true>(gate[4 * j + 2 * i + c], up[4 * j + 2 * i + c]);
      *reinterpret_cast<uint32_t*>(o + 8 * j) = pack_pair<DT>(v[0], v[1]);
    }
  }
}

// add_kernel(res, Y) on one half tile of kEpiResidual (N even).  Each element of res is read by the
// thread that then writes it, so res may be the output.
template <int DT>
__device__ __forceinline__ void store_residual_m64n128(const float (&acc)[64], int64_t row0,
                                                       int64_t col0, const GemmParams& p,
                                                       const void* res) {
  using T = DType<DT>;
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int64_t col = col0 + 8 * j + 2 * (lane & 3);
    if (col >= p.N) continue;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int64_t row = frag_row(row0, i);
      if (row >= p.M) continue;
      const int64_t off = row * p.ld_out + col;
      const uint32_t r = *(static_cast<const uint32_t*>(res) + off / 2);
      const float v0 = fadd_rn(pair_lo<DT>(r), T::rT(acc[4 * j + 2 * i]));
      const float v1 = fadd_rn(pair_hi<DT>(r), T::rT(acc[4 * j + 2 * i + 1]));
      *(static_cast<uint32_t*>(p.out) + off / 2) = pack_pair<DT>(v0, v1);
    }
  }
}

// One 64-column chunk of a half tile, fragments jb .. jb + 7 of acc, to out[row][col0 + d] (ld
// even), rounded once as the plain GEMM's store rounds.  kRope: MLA's apply_rotary_emb on the chunk
// (rope dim 64): interleaved pairs (2p, 2p + 1) are (a, b) = rT(acc), and the stored pair is
// (a c - b s, a s + b c) in fp32, one rounding per operation as torch's complex64 product takes it,
// with (c, s) = (cos, sin)[row % seq][p] of the fp32 [seq, 32] tables.  A pair is fragments
// 4j + 2i and 4j + 2i + 1 of one thread.  n_out > 1 writes the same values at col0 + h * ld_h for
// h < n_out (k_pe, which every head shares).
template <int DT, bool kRope>
__device__ __forceinline__ void store_mla_chunk(const float (&acc)[64], int jb, int64_t row0, int64_t col0,
                                                int64_t M, const EpiParams& e, int64_t ld, void* out,
                                                int64_t n_out, int64_t ld_h) {
  using T = DType<DT>;
  const int lane = threadIdx.x & 31;
  const float* cosv = static_cast<const float*>(e.cosv);
  const float* sinv = static_cast<const float*>(e.sinv);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int64_t row = frag_row(row0, i);
    if (row >= M) continue;
    const int64_t tab = (row % e.seq) * 32 + (lane & 3);
    uint32_t v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float a = acc[4 * (jb + j) + 2 * i], b = acc[4 * (jb + j) + 2 * i + 1];
      if constexpr (kRope) {
        const float ra = T::rT(a), rb = T::rT(b);
        const float cs = __ldg(cosv + tab + 4 * j), sn = __ldg(sinv + tab + 4 * j);
        v[j] = pack_pair<DT>(fadd_rn(fmul_rn(ra, cs), -fmul_rn(rb, sn)),
                             fadd_rn(fmul_rn(ra, sn), fmul_rn(rb, cs)));
      } else {
        v[j] = pack_pair<DT>(a, b);
      }
    }
    for (int64_t h = 0; h < n_out; ++h) {
      uint16_t* o = static_cast<uint16_t*>(out) + row * ld + col0 + h * ld_h + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t*>(o + 8 * j) = v[j];
    }
  }
}

// One 64-column chunk of kEpiMlaQkv starting at column gc of [q | latent | k_pe]: q's chunks are
// nope, nope, pe per 192-wide head; the latent is n_k columns; k_pe goes to the pe slot (columns
// 128 .. 191) of each of the n_q / 192 heads of k.  Chunks past N (the tile's tail) are skipped.
template <int DT>
__device__ __forceinline__ void store_mla_qkv_chunk(const float (&acc)[64], int jb, int64_t row0, int64_t gc,
                                                    const GemmParams& p, const EpiParams& e) {
  if (gc < e.n_q) {
    if ((gc >> 6) % 3 == 2)
      store_mla_chunk<DT, true>(acc, jb, row0, gc, p.M, e, e.n_q, p.out, 1, 0);
    else
      store_mla_chunk<DT, false>(acc, jb, row0, gc, p.M, e, e.n_q, p.out, 1, 0);
  } else if (gc - e.n_q < e.n_k) {
    store_mla_chunk<DT, false>(acc, jb, row0, gc - e.n_q, p.M, e, e.n_k, e.out_v, 1, 0);
  } else if (gc - e.n_q == e.n_k) {
    store_mla_chunk<DT, true>(acc, jb, row0, 128, p.M, e, e.n_q, e.out_k, e.n_q / 192, 192);
  }
}

template <int DT>
__device__ __forceinline__ void store_mla_tile(const float (&acc0)[64], const float (&acc1)[64], int64_t row0,
                                               int64_t col0, const GemmParams& p, const EpiParams& e) {
  store_mla_qkv_chunk<DT>(acc0, 0, row0, col0, p, e);
  store_mla_qkv_chunk<DT>(acc0, 8, row0, col0 + 64, p, e);
  store_mla_qkv_chunk<DT>(acc1, 0, row0, col0 + 128, p, e);
  store_mla_qkv_chunk<DT>(acc1, 8, row0, col0 + 192, p, e);
}

// The kernel body.  Plain mode (wgmma_gemm_kernel, kMoe == kMoeOff): B is tmB, the epilogue kEpi.
// Grouped mode (wgmma_moe_kernel): tiles come from decode_moe_unit and B from g's maps of the
// tile's expert; for kMoeSwiGLU the 256-row B stage is two 128-row boxes, w1 rows then w3 rows of
// the same n-block, which the 128-byte swizzle lays out exactly as one box of interleave_gate_up's
// weight, so the epilogue is kEpiSwiGLU's.
template <bool kSyrk, bool kBf16, int kEpi, int kMoe>
__device__ __forceinline__ void gemm_body(const CUtensorMap* tmA, const CUtensorMap* tmB,
                                          const GemmParams& p, const EpiParams& e,
                                          const MoeOperands* g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = ring_base(smem_raw);
  const Ring<kStages> ring(smem + kStages * kStageBytes);

  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;

  if (threadIdx.x == 0) {
    prefetch_tmap(tmA);
    if constexpr (kMoe != kMoeOff) {
      prefetch_moe_tmaps<kMoe>(g->tmB, g->seg);
    } else {
      prefetch_tmap(tmB);
    }
    ring.init(1, 2);                  // empty: one arrive per consumer warpgroup
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (tid == 0) {
      PipeState<kStages> ps;
      for (int u = blockIdx.x; u < p.num_units; u += gridDim.x) {
        Unit t;
        if constexpr (kMoe != kMoeOff) {
          if (!decode_moe_unit(p, *g, u, t)) break;
        } else {
          t = decode_unit<kSyrk>(p, u);
        }
        for (int kb = t.kb0; kb < t.kb1; ++kb) {
          ring.wait_empty(ps);
          uint8_t* a_dst = smem + ps.stage * kStageBytes;
          uint8_t* b_dst = a_dst + kABytes;
          uint64_t* bar = &ring.full[ps.stage];
          ring.expect_tx(ps, kStageBytes);
          if constexpr (kMoe != kMoeOff) {
            tma_load_2d(a_dst, tmA, bar, kb * BK, t.row0);
            moe_load_b<kMoe>(b_dst, g->tmB, bar, t.e, kb * BK, t.n_blk, BN, kBBytes / 2);
          } else if constexpr (!kSyrk) {
            tma_load_2d(a_dst, tmA, bar, kb * BK, t.m_blk * BM);
            tma_load_2d(b_dst, tmB, bar, kb * BK, t.n_blk * BN);
          } else {
            // X[T, C]: coordinate 0 = channel, coordinate 1 = token; box = 64 ch x 64 tok
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)
              tma_load_2d(a_dst + i * kBoxBytes, tmA, bar, t.m_blk * BM + i * 64, kb * BK);
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)
              tma_load_2d(b_dst + i * kBoxBytes, tmA, bar, t.n_blk * BN + i * 64, kb * BK);
          }
          ps.advance();
        }
      }
    }
    return;
  }

  // ===================== consumers (warpgroups 1, 2): rows 64 * c .. 64 * c + 63 =====================
  const int c = wg - 1;
  PipeState<kStages> ps;
  for (int u = blockIdx.x; u < p.num_units; u += gridDim.x) {
    Unit t;
    if constexpr (kMoe != kMoeOff) {
      if (!decode_moe_unit(p, *g, u, t)) break;
    } else {
      t = decode_unit<kSyrk>(p, u);
    }
    float acc0[64], acc1[64];                    // columns [0, 128) and [128, 256) of the tile
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    int prev = -1;
    for (int kb = t.kb0; kb < t.kb1; ++kb) {
      ring.wait_full(ps);
      wgmma_fence();
      const uint32_t a_addr = smem_u32(smem + ps.stage * kStageBytes);
      const uint32_t b_addr = a_addr + kABytes;
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        uint64_t adesc, bdesc0, bdesc1;
        if constexpr (!kSyrk) {
          adesc = make_smem_desc(a_addr + c * 64 * 128 + k * 32, 16, 1024);
          bdesc0 = make_smem_desc(b_addr + k * 32, 16, 1024);
          bdesc1 = make_smem_desc(b_addr + 128 * 128 + k * 32, 16, 1024);
        } else {
          adesc = make_smem_desc(a_addr + c * kBoxBytes + k * 2048, kBoxBytes, 1024);
          bdesc0 = make_smem_desc(b_addr + k * 2048, kBoxBytes, 1024);
          bdesc1 = make_smem_desc(b_addr + 2 * kBoxBytes + k * 2048, kBoxBytes, 1024);
        }
        const uint32_t accum = (kb > t.kb0 || k > 0) ? 1u : 0u;
        wgmma_m64n128k16<kBf16, kSyrk ? 1 : 0, kSyrk ? 1 : 0>(acc0, adesc, bdesc0, accum);
        wgmma_m64n128k16<kBf16, kSyrk ? 1 : 0, kSyrk ? 1 : 0>(acc1, adesc, bdesc1, accum);
      }
      wgmma_commit();
      wgmma_wait<1>();                           // the group that read stage `prev` has retired
      if (prev >= 0 && tid == 0) ring.release(prev);
      prev = ps.stage;
      ps.advance();
    }
    wgmma_wait<0>();
    fence_acc(acc0);
    fence_acc(acc1);
    if (prev >= 0 && tid == 0) ring.release(prev);

    // ---- epilogue straight from the accumulator registers ----
    int64_t row0 = static_cast<int64_t>(t.m_blk) * BM + c * 64;
    if constexpr (kMoe != kMoeOff) row0 = t.row0 + c * 64;
    const int64_t col0 = static_cast<int64_t>(t.n_blk) * BN;
    if constexpr (kMoe != kMoeOff) {
      constexpr int DT = kBf16 ? LLMC_BF16 : LLMC_F16;
      if constexpr (kMoe == kMoeSwiGLU) {
        store_swiglu_m64n128<DT>(acc0, acc1, row0, col0 / 2, t.row_end, p.ld_out, p.out);
      } else {
        store_routed_m64n128<DT>(acc0, row0, col0, t.row_end, p.N, p.ld_out, p.out, g->seg.w_route);
        store_routed_m64n128<DT>(acc1, row0, col0 + 128, t.row_end, p.N, p.ld_out, p.out, g->seg.w_route);
      }
    } else if constexpr (!kSyrk) {
      constexpr int DT = kBf16 ? LLMC_BF16 : LLMC_F16;
      if constexpr (kEpi == kEpiLinear) {
        store_linear_m64n128<DT>(acc0, row0, col0, p.M, p.N, p.ld_out, p.bias, p.out);
        store_linear_m64n128<DT>(acc1, row0, col0 + 128, p.M, p.N, p.ld_out, p.bias, p.out);
      } else if constexpr (kEpi == kEpiRopeQkv) {
        store_qkv_tile<DT>(acc0, acc1, row0, col0, p, e);
      } else if constexpr (kEpi == kEpiSwiGLU) {
        store_swiglu_m64n128<DT>(acc0, acc1, row0, col0 / 2, p.M, p.ld_out, p.out);
      } else if constexpr (kEpi == kEpiMlaQkv) {
        store_mla_tile<DT>(acc0, acc1, row0, col0, p, e);
      } else if constexpr (kEpi == kEpiMlaKvB) {
        // n-tile h is head h: its k_nope (128) and v (128) columns
        store_linear_m64n128<DT>(acc0, row0, t.n_blk * 192, p.M, e.n_q, e.n_q, nullptr, p.out);
        store_linear_m64n128<DT>(acc1, row0, t.n_blk * 128, p.M, e.n_k, e.n_k, nullptr, e.out_v);
      } else {
        store_residual_m64n128<DT>(acc0, row0, col0, p, e.res);
        store_residual_m64n128<DT>(acc1, row0, col0 + 128, p, e.res);
      }
    } else {
      // fp32 partial slab `t.split` of the split-K sum
      float* slab = static_cast<float*>(p.out) + static_cast<int64_t>(t.split) * p.M * p.ld_out;
      __builtin_assume((p.ld_out & 1) == 0);   // ld_out = C, a multiple of 8: all pairs are float2
      store_f32_m64n128(acc0, row0, col0, p.M, p.N, p.ld_out, slab);
      store_f32_m64n128(acc1, row0, col0 + 128, p.M, p.N, p.ld_out, slab);
    }
  }
}

template <bool kSyrk, bool kBf16, int kEpi = kEpiLinear>
__global__ void __launch_bounds__(kThreads, 1)
wgmma_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const GemmParams p, const EpiParams e) {
  gemm_body<kSyrk, kBf16, kEpi, kMoeOff>(&tmA, &tmB, p, e, nullptr);
}

template <bool kBf16, int kMoe>
__global__ void __launch_bounds__(kThreads, 1)
wgmma_moe_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ MoeOperands g,
                 const GemmParams p) {
  gemm_body<false, kBf16, kEpiLinear, kMoe>(&tmA, nullptr, p, EpiParams{}, &g);
}

// ---- SYRK finalize: H = a*H + b*sum_s P_s on the upper triangle, mirrored -----------------------
__global__ void __launch_bounds__(256)
syrk_finalize_kernel(float* __restrict__ H, const float* __restrict__ P, int64_t C, int splits,
                     float a, float b) {
  // 32x32 tiles; block (bx, by) with bx >= by handles tile rows by, cols bx and its mirror.
  __shared__ float tile[32][33];
  const int bx = blockIdx.x, by = blockIdx.y;
  if (bx < by) return;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int64_t r = static_cast<int64_t>(by) * 32 + i, c = static_cast<int64_t>(bx) * 32 + tx;
    float v = 0.f;
    if (r < C && c < C) {
      float acc = 0.f;
      for (int s = 0; s < splits; ++s) acc += P[(static_cast<int64_t>(s) * C + r) * C + c];
      // for diagonal tiles take the upper-triangle value for both (r,c) and (c,r)
      if (bx == by && c < r) {
        acc = 0.f;
        for (int s = 0; s < splits; ++s) acc += P[(static_cast<int64_t>(s) * C + c) * C + r];
        v = a * H[c * C + r] + b * acc;
      } else {
        v = a * H[r * C + c] + b * acc;
      }
    }
    tile[i][tx] = v;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int64_t r = static_cast<int64_t>(by) * 32 + i, c = static_cast<int64_t>(bx) * 32 + tx;
    if (r < C && c < C) H[r * C + c] = tile[i][tx];
    if (bx != by) {
      const int64_t r2 = static_cast<int64_t>(bx) * 32 + i, c2 = static_cast<int64_t>(by) * 32 + tx;
      if (r2 < C && c2 < C) H[r2 * C + c2] = tile[tx][i];
    }
  }
}

// ---- host side -------------------------------------------------------------------------------------
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                        const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                        const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion,
                                        CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode_fn() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) {
    set_last_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s",
                   cudaGetErrorString(e));
    return nullptr;
  }
  fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
  return fn;
}

int encode_tmap_2d(CUtensorMap* out, const void* base, CUtensorMapDataType dtype, uint32_t elem_bytes,
                   uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows,
                   uint32_t box_cols, CUtensorMapSwizzle swizzle) {
  PFN_tmapEncodeTiled fn = get_encode_fn();
  if (!fn) return LLMC_ECUDA;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld_elems * elem_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, dtype, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult %d (dtype %d rows %llu cols %llu ld %llu)",
                   (int)r, (int)dtype, (unsigned long long)rows, (unsigned long long)cols,
                   (unsigned long long)ld_elems);
    return LLMC_ECUDA;
  }
  return LLMC_OK;
}

struct SyrkPlan {
  int n_tiles_n, num_tiles, splits, kb_total, kb_per_split;
};

static SyrkPlan plan_syrk(int64_t T, int64_t C) {
  SyrkPlan s;
  const int mt = static_cast<int>((C + BM - 1) / BM);
  s.n_tiles_n = static_cast<int>((C + BN - 1) / BN);
  int tiles = 0;
  for (int mi = 0; mi < mt; ++mi) {
    int cnt = s.n_tiles_n - (mi >> 1);
    if (cnt > 0) tiles += cnt;
  }
  s.num_tiles = tiles;
  s.kb_total = static_cast<int>((T + BK - 1) / BK);
  // choose the split-K factor that best fills whole waves of kNumSMs CTAs
  int best = 1;
  double best_eff = 0.0;
  for (int sp = 1; sp <= 16; ++sp) {
    if (sp > 1 && s.kb_total / sp < 16) break;
    const long units = static_cast<long>(tiles) * sp;
    const long waves = (units + kNumSMs - 1) / kNumSMs;
    const double eff = static_cast<double>(units) / (waves * kNumSMs) - 0.004 * (sp - 1);
    if (eff > best_eff + 1e-9) { best_eff = eff; best = sp; }
  }
  s.splits = best;
  s.kb_per_split = (s.kb_total + best - 1) / best;
  s.splits = (s.kb_total + s.kb_per_split - 1) / s.kb_per_split;
  return s;
}

// Checks and launches the forward GEMM Y[M, N] = X[M, K] W[N, K]^T with epilogue kEpi into p.out
// (and e's outputs; the caller checks e's pointers).  p's other fields are filled in here.
template <int kEpi>
static int launch_gemm(const void* x, const void* w, int64_t M, int64_t N, int64_t K, int dtype,
                       GemmParams p, const EpiParams& e, void* stream) {
  LLMC_CHECK_ARG(M >= 0 && N >= 0 && K > 0, "gemm: bad shape");
  if (M == 0 || N == 0) return LLMC_OK;
  LLMC_CHECK_ARG(x && w && p.out, "gemm: null pointer");
  LLMC_CHECK_ARG(dtype == LLMC_BF16 || dtype == LLMC_F16, "gemm: dtype must be bf16 or fp16");
  if (K % 8 != 0 || !aligned16(x) || !aligned16(w) || !aligned16(p.out)) {
    set_last_error("gemm: K=%lld must be a multiple of 8 and pointers 16-byte aligned", (long long)K);
    return LLMC_EALIGN;
  }
  CUtensorMap tmA, tmB;
  if (int rc = encode_tmap_2d(&tmA, x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, M, K, K, BM, BK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  if (int rc = encode_tmap_2d(&tmB, w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, N, K, K, BN, BK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  p.M = M; p.N = N; p.K = K;
  p.n_tiles_n = static_cast<int>((N + BN - 1) / BN);
  const int64_t mt = (M + BM - 1) / BM;
  LLMC_CHECK_ARG(mt * p.n_tiles_n < (1ll << 31), "gemm: too many tiles");
  p.num_units = static_cast<int>(mt * p.n_tiles_n);
  p.num_tiles = p.num_units;
  p.splits = 1;
  p.kb_total = static_cast<int>((K + BK - 1) / BK);
  p.kb_per_split = p.kb_total;
  p.gn = l2_group_width(static_cast<int64_t>(BN) * K * 2, p.n_tiles_n);   // K > 0: one n-tile's bytes
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return launch_persistent(dtype == LLMC_BF16 ? wgmma_gemm_kernel<false, true, kEpi>
                                              : wgmma_gemm_kernel<false, false, kEpi>,
                           p.num_units, kThreads, kSmemBytes, st, tmA, tmB, p, e);
}

// Checks and launches the grouped GEMM over m.rows gathered rows: n-tiles of BN output columns per
// expert, each expert's B one tensor map (kMoeSwiGLU: BN / 2 rows of w1, then of w3).
template <int kMoe>
static int launch_moe(const MoeLaunch<kMoe>& m, void* stream) {
  int n_tiles, units;
  if (int rc = m.check_values(BM, BN)) return rc;
  if (m.K % 8 != 0) {
    set_last_error("%s: K=%lld must be a multiple of 8", m.what, (long long)m.K);
    return LLMC_EALIGN;
  }
  if (int rc = m.plan(BM, BN, n_tiles, units)) return rc;
  if (m.rows == 0) return LLMC_OK;
  if (int rc = m.check_pointers()) return rc;
  CUtensorMap tmA;
  if (int rc = encode_tmap_2d(&tmA, m.a, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, m.rows, m.K, m.K, BM, BK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  MoeOperands g{};
  if (int rc = m.encode_tmaps(g.tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, m.K, BN, BK, CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  g.seg = m.segments();
  GemmParams p{};
  p.out = m.out; p.ld_out = m.N;
  p.M = m.rows; p.N = kMoe == kMoeSwiGLU ? 2 * m.N : m.N; p.K = m.K;   // gate/up: w1 and w3 columns
  p.n_tiles_n = n_tiles;
  p.num_units = units;
  p.num_tiles = p.num_units;
  p.splits = 1;
  p.kb_total = static_cast<int>((m.K + BK - 1) / BK);
  p.kb_per_split = p.kb_total;
  p.gn = l2_group_width(static_cast<int64_t>(BN) * m.K * 2, p.n_tiles_n);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return launch_persistent(m.dtype == LLMC_BF16 ? wgmma_moe_kernel<true, kMoe> : wgmma_moe_kernel<false, kMoe>,
                           p.num_units, kThreads, kSmemBytes, st, tmA, g, p);
}

// out[t] = rT(...rT(rT(0 + y[rows[t, 0]]) + y[rows[t, 1]]) + ...): the k expert outputs of token t
// added in the order given (ascending expert), as `zeros` + one index_add_ per expert does.
// kCombineGated (Qwen2-MoE's gated shared expert): then out[t] = rT(out[t] + rT(rT(sigmoid(g[t])) * s[t])),
// the roundings of F.sigmoid(gate(x)) * shared_expert(x) and the add that follows.
// kCombineWeighted (DeepSeek-V2's fp32 routing weights and ungated shared experts): each term is
// rT(y[r] * w[r]) with w fp32 [rows] in y's row order (g), then out[t] = rT(out[t] + s[t]).
enum CombineMode { kCombinePlain, kCombineGated, kCombineWeighted };

template <int DT, int kMode>
__global__ void __launch_bounds__(256)
moe_combine_kernel(const void* __restrict__ y, const int64_t* __restrict__ rows,
                   const void* __restrict__ g, const void* __restrict__ sh,
                   void* __restrict__ out, int64_t T, int64_t k, int64_t N) {
  using D = DType<DT>;
  const int64_t chunks = N >> 3;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < T * chunks;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t t = i / chunks, ch = i - t * chunks;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int64_t s = 0; s < k; ++s) {
      float v[8];
      const int64_t r = __ldg(rows + t * k + s);
      load8<DT>(y, r * N + ch * 8, v);
      if constexpr (kMode == kCombineWeighted) {
        const float w = __ldg(static_cast<const float*>(g) + r);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = D::rT(fadd_rn(acc[j], D::rT(fmul_rn(v[j], w))));
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = D::rT(fadd_rn(acc[j], v[j]));
      }
    }
    if constexpr (kMode == kCombineGated) {
      const float sg = D::rT(sigmoid_f32(D::load(g, t)));
      float v[8];
      load8<DT>(sh, i << 3, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = D::rT(fadd_rn(acc[j], D::rT(fmul_rn(sg, v[j]))));
    } else if constexpr (kMode == kCombineWeighted) {
      float v[8];
      load8<DT>(sh, i << 3, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = D::rT(fadd_rn(acc[j], v[j]));
    }
    store8<DT>(out, i << 3, acc);
  }
}

// The launch behind the llmc_moe_combine* entry points (g, sh unused by llmc_moe_combine), on
// arguments its caller has checked: T > 0, N a multiple of 8.
template <int kMode>
static int launch_moe_combine(const void* y, const int64_t* rows, const void* g, const void* sh, void* out,
                              int64_t T, int64_t top_k, int64_t N, int dtype, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t blocks = (T * (N >> 3) + 255) / 256;
  if (blocks > kNumSMs * 32) blocks = kNumSMs * 32;
#define CALL(DT) moe_combine_kernel<DT, kMode><<<(int)blocks, 256, 0, st>>>(y, rows, g, sh, out, T, top_k, N); \
  LLMC_CHECK_LAUNCH()
  if (dtype == LLMC_BF16) { CALL(LLMC_BF16); } else { CALL(LLMC_F16); }
#undef CALL
  return LLMC_OK;
}

}  // namespace llmc

using namespace llmc;

extern "C" int llmc_moe_gemm_swiglu(const void* xp, const void* const* w1, const void* const* w3,
                                    const int32_t* offsets, void* act, int64_t rows, int64_t inter,
                                    int64_t K, int64_t n_experts, int dtype, void* stream) {
  return launch_moe<kMoeSwiGLU>({"moe_gemm_swiglu", xp, act, w1, w3, offsets, nullptr, rows, inter, K, n_experts,
                                 dtype, "weight"}, stream);
}

extern "C" int llmc_moe_gemm_down(const void* act, const void* const* w2, const int32_t* offsets,
                                  const void* w_route, void* y, int64_t rows, int64_t N,
                                  int64_t inter, int64_t n_experts, int dtype, void* stream) {
  return launch_moe<kMoeDown>({"moe_gemm_down", act, y, w2, nullptr, offsets, w_route, rows, N, inter, n_experts,
                               dtype, "weight"}, stream);
}

extern "C" int llmc_moe_combine(const void* y, const int64_t* rows, void* out, int64_t T,
                                int64_t top_k, int64_t N, int dtype, void* stream) {
  LLMC_CHECK_ARG(T >= 0 && top_k > 0 && N > 0, "moe_combine: bad shape");
  if (T == 0) return LLMC_OK;
  LLMC_CHECK_ARG(y && rows && out, "moe_combine: null pointer");
  LLMC_CHECK_ARG(dtype == LLMC_BF16 || dtype == LLMC_F16, "moe_combine: dtype must be bf16 or fp16");
  if (N % 8 != 0 || !aligned16(y) || !aligned16(out)) {
    set_last_error("moe_combine: N=%lld must be a multiple of 8 and pointers 16-byte aligned",
                   (long long)N);
    return LLMC_EALIGN;
  }
  return launch_moe_combine<kCombinePlain>(y, rows, nullptr, nullptr, out, T, top_k, N, dtype, stream);
}

extern "C" int llmc_moe_combine_shared(const void* y, const int64_t* rows, const void* gate_logit,
                                       const void* shared, void* out, int64_t T, int64_t top_k, int64_t N,
                                       int dtype, void* stream) {
  LLMC_CHECK_ARG(T >= 0 && top_k > 0 && N > 0, "moe_combine_shared: bad shape T=%lld top_k=%lld N=%lld",
                 (long long)T, (long long)top_k, (long long)N);
  LLMC_CHECK_ARG(dtype == LLMC_BF16 || dtype == LLMC_F16, "moe_combine_shared: dtype must be bf16 or fp16");
  if (N % 8 != 0) {
    set_last_error("moe_combine_shared: N=%lld must be a multiple of 8", (long long)N);
    return LLMC_EALIGN;
  }
  if (T == 0) return LLMC_OK;
  LLMC_CHECK_ARG(y && rows && gate_logit && shared && out, "moe_combine_shared: null pointer");
  if (!aligned16(y) || !aligned16(shared) || !aligned16(out)) {
    set_last_error("moe_combine_shared: y, shared and out must be 16-byte aligned");
    return LLMC_EALIGN;
  }
  return launch_moe_combine<kCombineGated>(y, rows, gate_logit, shared, out, T, top_k, N, dtype, stream);
}

extern "C" int llmc_moe_combine_weighted(const void* y, const int64_t* rows, const float* w, const void* shared,
                                         void* out, int64_t T, int64_t top_k, int64_t N, int dtype,
                                         void* stream) {
  LLMC_CHECK_ARG(T >= 0 && top_k > 0 && N > 0, "moe_combine_weighted: bad shape T=%lld top_k=%lld N=%lld",
                 (long long)T, (long long)top_k, (long long)N);
  LLMC_CHECK_ARG(dtype == LLMC_BF16 || dtype == LLMC_F16, "moe_combine_weighted: dtype must be bf16 or fp16");
  if (N % 8 != 0) {
    set_last_error("moe_combine_weighted: N=%lld must be a multiple of 8", (long long)N);
    return LLMC_EALIGN;
  }
  if (T == 0) return LLMC_OK;
  LLMC_CHECK_ARG(y && rows && w && shared && out, "moe_combine_weighted: null pointer");
  if (!aligned16(y) || !aligned16(shared) || !aligned16(out)) {
    set_last_error("moe_combine_weighted: y, shared and out must be 16-byte aligned");
    return LLMC_EALIGN;
  }
  return launch_moe_combine<kCombineWeighted>(y, rows, w, shared, out, T, top_k, N, dtype, stream);
}

extern "C" int llmc_gemm_bf16(const void* x, const void* w, const void* bias, void* y, int64_t M,
                              int64_t N, int64_t K, int dtype, void* stream) {
  GemmParams p{};
  p.out = y; p.bias = bias; p.ld_out = N;
  return launch_gemm<kEpiLinear>(x, w, M, N, K, dtype, p, EpiParams{}, stream);
}

extern "C" int llmc_gemm_rope_qkv(const void* x, const void* w_qkv, void* q, void* k, void* v,
                                  const void* cosv, const void* sinv, int64_t M, int64_t n_q,
                                  int64_t n_k, int64_t n_v, int64_t K, int64_t seq, int dtype,
                                  void* stream) {
  LLMC_CHECK_ARG(n_q > 0 && n_k > 0 && n_v > 0 && seq > 0 && M % seq == 0,
                 "gemm_rope_qkv: need n_q, n_k, n_v, seq > 0 and M a multiple of seq");
  LLMC_CHECK_ARG(n_q % BN == 0 && n_k % BN == 0 && n_v % 8 == 0,
                 "gemm_rope_qkv: n_q=%lld and n_k=%lld must be multiples of %d, n_v=%lld of 8",
                 (long long)n_q, (long long)n_k, BN, (long long)n_v);
  LLMC_CHECK_ARG(k && v && cosv && sinv, "gemm_rope_qkv: null pointer");
  if (!aligned16(k) || !aligned16(v) || !aligned16(cosv) || !aligned16(sinv)) {
    set_last_error("gemm_rope_qkv: pointers must be 16-byte aligned");
    return LLMC_EALIGN;
  }
  GemmParams p{};
  p.out = q;
  EpiParams e{};
  e.out_k = k; e.out_v = v; e.cosv = cosv; e.sinv = sinv;
  e.n_q = n_q; e.n_k = n_k; e.seq = seq;
  return launch_gemm<kEpiRopeQkv>(x, w_qkv, M, n_q + n_k + n_v, K, dtype, p, e, stream);
}

extern "C" int llmc_gemm_swiglu(const void* x, const void* w_gate_up, void* act, int64_t M,
                                int64_t inter, int64_t K, int dtype, void* stream) {
  LLMC_CHECK_ARG(inter > 0 && inter % 128 == 0,
                 "gemm_swiglu: inter=%lld must be a positive multiple of 128", (long long)inter);
  GemmParams p{};
  p.out = act; p.ld_out = inter;
  return launch_gemm<kEpiSwiGLU>(x, w_gate_up, M, 2 * inter, K, dtype, p, EpiParams{}, stream);
}

extern "C" int llmc_gemm_residual(const void* x, const void* w, const void* res, void* y, int64_t M,
                                  int64_t N, int64_t K, int dtype, void* stream) {
  LLMC_CHECK_ARG(N % 8 == 0, "gemm_residual: N=%lld must be a multiple of 8", (long long)N);
  LLMC_CHECK_ARG(res != nullptr, "gemm_residual: null pointer");
  if (!aligned16(res)) {
    set_last_error("gemm_residual: pointers must be 16-byte aligned");
    return LLMC_EALIGN;
  }
  GemmParams p{};
  p.out = y; p.ld_out = N;
  EpiParams e{};
  e.res = res;
  return launch_gemm<kEpiResidual>(x, w, M, N, K, dtype, p, e, stream);
}

extern "C" int llmc_gemm_mla_qkv(const void* x, const void* w_qkva, void* q, void* k, void* latent,
                                 const float* cosv, const float* sinv, int64_t M, int64_t heads,
                                 int64_t kv_lora, int64_t K, int64_t seq, int dtype, void* stream) {
  LLMC_CHECK_ARG(heads > 0 && heads % 4 == 0, "gemm_mla_qkv: heads=%lld must be a positive multiple of 4",
                 (long long)heads);
  LLMC_CHECK_ARG(kv_lora > 0 && kv_lora % 64 == 0, "gemm_mla_qkv: kv_lora=%lld must be a positive multiple of 64",
                 (long long)kv_lora);
  LLMC_CHECK_ARG(seq > 0 && M % seq == 0, "gemm_mla_qkv: need seq > 0 and M a multiple of seq");
  LLMC_CHECK_ARG(k && latent && cosv && sinv, "gemm_mla_qkv: null pointer");
  if (!aligned16(k) || !aligned16(latent) || !aligned16(cosv) || !aligned16(sinv)) {
    set_last_error("gemm_mla_qkv: pointers must be 16-byte aligned");
    return LLMC_EALIGN;
  }
  GemmParams p{};
  p.out = q;
  EpiParams e{};
  e.out_k = k; e.out_v = latent; e.cosv = cosv; e.sinv = sinv;
  e.n_q = heads * 192; e.n_k = kv_lora; e.seq = seq;
  return launch_gemm<kEpiMlaQkv>(x, w_qkva, M, e.n_q + kv_lora + 64, K, dtype, p, e, stream);
}

extern "C" int llmc_gemm_mla_kv_b(const void* x, const void* w_kv_b, void* k, void* v, int64_t M,
                                  int64_t heads, int64_t K, int dtype, void* stream) {
  LLMC_CHECK_ARG(heads > 0, "gemm_mla_kv_b: heads=%lld must be positive", (long long)heads);
  LLMC_CHECK_ARG(v != nullptr, "gemm_mla_kv_b: null pointer");
  if (!aligned16(v)) {
    set_last_error("gemm_mla_kv_b: pointers must be 16-byte aligned");
    return LLMC_EALIGN;
  }
  GemmParams p{};
  p.out = k;
  EpiParams e{};
  e.out_v = v; e.n_q = heads * 192; e.n_k = heads * 128;
  return launch_gemm<kEpiMlaKvB>(x, w_kv_b, M, heads * 256, K, dtype, p, e, stream);
}

extern "C" int64_t llmc_syrk_workspace_bytes(int64_t T, int64_t C) {
  if (T <= 0 || C <= 0) return 0;
  const SyrkPlan s = plan_syrk(T, C);
  return static_cast<int64_t>(s.splits) * C * C * 4;
}

extern "C" int llmc_syrk_accum(const void* x, int64_t T, int64_t C, int dtype, float* H, double n,
                               double b, void* workspace, int64_t workspace_bytes, void* stream) {
  LLMC_CHECK_ARG(T > 0 && C > 0 && x && H && workspace, "syrk: bad argument");
  LLMC_CHECK_ARG(dtype == LLMC_BF16 || dtype == LLMC_F16, "syrk: X must be bf16 or fp16");
  LLMC_CHECK_ARG(n >= 0 && b > 0, "syrk: need n >= 0 and b > 0");
  if (C % 8 != 0 || !aligned16(x) || !aligned16(H) || !aligned16(workspace)) {
    set_last_error("syrk: C=%lld must be a multiple of 8 and pointers 16-byte aligned", (long long)C);
    return LLMC_EALIGN;
  }
  const SyrkPlan s = plan_syrk(T, C);
  LLMC_CHECK_ARG(workspace_bytes >= static_cast<int64_t>(s.splits) * C * C * 4,
                 "syrk: workspace too small (%lld < %lld)", (long long)workspace_bytes,
                 (long long)(static_cast<int64_t>(s.splits) * C * C * 4));
  CUtensorMap tmX;
  if (int rc = encode_tmap_2d(&tmX, x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, T, C, C, 64, 64,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  GemmParams p{};
  p.M = C; p.N = C; p.K = T;
  p.out = workspace; p.bias = nullptr; p.ld_out = C;
  p.n_tiles_n = s.n_tiles_n;
  p.num_tiles = s.num_tiles;
  p.splits = s.splits;
  p.num_units = s.num_tiles * s.splits;
  p.kb_total = s.kb_total;
  p.kb_per_split = s.kb_per_split;
  p.gn = 12;                      // 12 m-blocks (1536 rows) x ~11 n-tiles ~ one wave of 132 tiles
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = launch_persistent(dtype == LLMC_BF16 ? wgmma_gemm_kernel<true, true>
                                                : wgmma_gemm_kernel<true, false>,
                             p.num_units, kThreads, kSmemBytes, st, tmX, tmX, p, EpiParams{});
  if (rc) return rc;
  // gptq.py:283-290: H *= n/(n+b); H += (sqrt(2/(n+b)) X)^T (sqrt(2/(n+b)) X)
  const float fa = static_cast<float>(n / (n + b));
  const float fb = static_cast<float>(2.0 / (n + b));
  const unsigned nb = static_cast<unsigned>((C + 31) / 32);
  syrk_finalize_kernel<<<dim3(nb, nb), 256, 0, st>>>(H, reinterpret_cast<const float*>(workspace),
                                                     C, s.splits, fa, fb);
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}
