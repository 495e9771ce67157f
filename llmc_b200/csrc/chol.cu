// chol.cu — K4: U = cholesky(cholesky_inverse(cholesky(H)), upper)  (gptq.py:172-174) as ONE
// reverse-ordered blocked factorisation + ONE blocked triangular inverse.
//
// Identity used (DESIGN.md §K4): let J be the index reversal and G = J H J = L L^T (lower
// Cholesky).  Then H = (J L J)(J L J)^T with R = J L J upper triangular, so H^-1 = R^-T R^-1 and
// the unique upper factor with positive diagonal is U = R^-1 = J L^-1 J, i.e.
//        U[i][j] = (L^-1)[n-1-i][n-1-j].
// Work: C^3/3 (factor) + C^3/3 (inverse) flops instead of the reference's potrf + potri + potrf
// (4/3 C^3), and every O(C^3) part is a 128-deep rank update executed by the 3xTF32 tensor-core
// kernel of tf32.cu (fp32-accurate); only the 128x128 diagonal blocks run on CUDA cores.
#include "tc.cuh"

namespace llmc {
namespace ch {

constexpr int NB = 128;
constexpr int LDS = NB + 1;

// G[i][j] = H[n-1-i][n-1-j]
__global__ void __launch_bounds__(256)
reverse_kernel(const float* __restrict__ H, float* __restrict__ G, int64_t n) {
  const int64_t total = n * n;
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    G[idx] = H[total - 1 - idx];
  }
}

// U[i][j] = j >= i ? Y[n-1-i][n-1-j] = Z[n-1-j][n-1-i] : 0, for Z = Y^T; 32 x 32 tiles through
// shared memory, so both the reads of Z and the writes of U are row segments
__global__ void __launch_bounds__(256)
reverse_upper_kernel(const float* __restrict__ Z, float* __restrict__ U, int64_t n) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t i0 = static_cast<int64_t>(blockIdx.y) * 32, j0 = static_cast<int64_t>(blockIdx.x) * 32;
  for (int jj = ty; jj < 32; jj += 8) {
    const int64_t i = i0 + tx, j = j0 + jj;
    tile[jj][tx] = (i < n && j < n && j >= i) ? Z[(n - 1 - j) * n + (n - 1 - i)] : 0.f;
  }
  __syncthreads();
  for (int ii = ty; ii < 32; ii += 8) {
    const int64_t i = i0 + ii, j = j0 + tx;
    if (i < n && j < n) U[i * n + j] = tile[tx][ii];
  }
}

// One CTA: factor the nb x nb diagonal block at G[k0][k0] (lower) and invert the factor, blocked by
// 32: 32x32 diagonal sub-blocks are factored in registers (warp shuffles), the sub-panel is solved
// with one thread per row in registers, the trailing update uses 4x4 register tiles, and L^-1 is
// built from 32x32 block products (X_ij = -X_ii * sum_k L_ik X_kj).  Rows/cols >= nb are padded
// with the identity so every loop runs at the full 128.  G block <- L_kk; Lhi / Llo block <- the
// tf32 split of L_kk^-1; Z / Zhi / Zlo block <- L_kk^-T and its split (ld n).  info[0] = k0 + j + 1
// on a non-positive pivot.
constexpr int SBK = 32;

__global__ void __launch_bounds__(256, 1)
diag_kernel(float* __restrict__ G, int64_t n, int64_t k0, int nb, float* __restrict__ Z,
            float* __restrict__ Zhi, float* __restrict__ Zlo, float* __restrict__ Lhi,
            float* __restrict__ Llo, int* __restrict__ info) {
  extern __shared__ float sm[];
  float* S = sm;                 // [NB][LDS]
  float* X = sm + NB * LDS;      // [NB][LDS]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  __shared__ __align__(16) float colbuf[SBK];
  __shared__ float rinv[NB];
  {
    // 64 elements per thread, 16 independent loads in flight at a time (the block was just
    // written by the trailing update: L2 latency, not bandwidth, is what this costs)
    const int j = tid & 127;
#pragma unroll 1
    for (int t0 = 0; t0 < NB / 2; t0 += 16) {
      float v[16];
#pragma unroll
      for (int t = 0; t < 16; ++t) {
        const int i = (tid >> 7) + 2 * (t0 + t);
        v[t] = (i == j) ? 1.f : 0.f;
        if (i < nb && j < nb) v[t] = (j <= i) ? __ldcg(G + (k0 + i) * n + k0 + j) : 0.f;
      }
#pragma unroll
      for (int t = 0; t < 16; ++t) {
        const int i = (tid >> 7) + 2 * (t0 + t);
        S[i * LDS + j] = v[t];
        X[i * LDS + j] = 0.f;
      }
    }
  }
  __syncthreads();

  // ---------------- phase A: L = chol(S), panels of 32 columns ----------------
  for (int b0 = 0; b0 < NB; b0 += SBK) {
    if (warp == 0) {                      // A1: 32x32 diagonal block, lane i = row i, in registers
      float a[SBK];
#pragma unroll
      for (int k = 0; k < SBK; ++k) a[k] = (k <= lane) ? S[(b0 + lane) * LDS + b0 + k] : 0.f;
      // Per column j the dependent chain is: broadcast a[j][j] -> rsqrt (+ one Newton step) ->
      // scale -> broadcast L[j+1][j] -> update a[j+1].  The updates of columns >= j+2 go through
      // shared memory (8 broadcast LDS.128 instead of 30 shuffles) and are consumed one
      // iteration later, so their latency is off the chain.
      float4 pend[SBK / 4];
      float lprev = 0.f;
#pragma unroll
      for (int j = 0; j < SBK; ++j) {
        const float ajj = __shfl_sync(0xffffffffu, a[j], j);
        if (!(ajj > 0.f) && lane == j && (b0 + j) < nb && info[0] == 0)
          info[0] = static_cast<int>(k0) + b0 + j + 1;
        const float ac = fmaxf(ajj, 1e-30f);
        float r = rsqrtf(ac);
        r = r * fmaf(-0.5f * ac * r, r, 1.5f);            // 1/sqrt(a), ~1 ulp
        float d = ac * r;
        d = fmaf(fmaf(-d, d, ac), 0.5f * r, d);           // sqrt(a), ~1 ulp
        const float lij = (lane > j) ? a[j] * r : ((lane == j) ? d : 0.f);
        a[j] = lij;
        if (lane == j) rinv[b0 + j] = r;                  // 1 / L[j][j] for A2 and B1
        if (j + 1 < SBK) {
          const float lnext = __shfl_sync(0xffffffffu, lij, j + 1);
          a[j + 1] = fmaf(-lij, lnext, a[j + 1]);
        }
        if (j > 0) {                                       // deferred updates of column j-1: k >= j+1
#pragma unroll
          for (int k4 = (j + 1) & ~3; k4 < SBK; k4 += 4) {
            const float4 l4 = pend[k4 / 4];
            if (k4 + 0 > j) a[k4 + 0] = fmaf(-lprev, l4.x, a[k4 + 0]);
            if (k4 + 1 > j) a[k4 + 1] = fmaf(-lprev, l4.y, a[k4 + 1]);
            if (k4 + 2 > j) a[k4 + 2] = fmaf(-lprev, l4.z, a[k4 + 2]);
            if (k4 + 3 > j) a[k4 + 3] = fmaf(-lprev, l4.w, a[k4 + 3]);
          }
        }
        if (j + 2 < SBK) {                                 // publish column j, fetch it for k >= j+2
          __syncwarp();
          colbuf[lane] = lij;
          __syncwarp();
#pragma unroll
          for (int k4 = (j + 2) & ~3; k4 < SBK; k4 += 4)
            pend[k4 / 4] = *reinterpret_cast<const float4*>(colbuf + k4);
          lprev = lij;
        }
      }
#pragma unroll
      for (int k = 0; k < SBK; ++k)
        if (k <= lane) S[(b0 + lane) * LDS + b0 + k] = a[k];
    }
    __syncthreads();
    const int nrem = NB - b0 - SBK;       // rows below the diagonal sub-block
    if (tid < nrem) {                     // A2: P = A_panel * L_kk^-T by forward substitution
      const int i = b0 + SBK + tid;
      float p[SBK];
#pragma unroll
      for (int j = 0; j < SBK; ++j) p[j] = S[i * LDS + b0 + j];
#pragma unroll
      for (int j = 0; j < SBK; ++j) {
        float acc = p[j];
#pragma unroll
        for (int k = 0; k < j; ++k) acc = fmaf(-p[k], S[(b0 + j) * LDS + b0 + k], acc);
        p[j] = acc * rinv[b0 + j];
      }
#pragma unroll
      for (int j = 0; j < SBK; ++j) S[i * LDS + b0 + j] = p[j];
    } else if (warp == 7) {
      // B1, overlapped with A2 (which occupies warps 0-2 at most): the inverse of this panel's
      // 32x32 diagonal block, lane c = column c, forward substitution in registers
      float x[SBK];
#pragma unroll
      for (int i = 0; i < SBK; ++i) {
        float acc = (i == lane) ? 1.f : 0.f;
#pragma unroll
        for (int k = 0; k < i; ++k) acc = fmaf(-S[(b0 + i) * LDS + b0 + k], x[k], acc);
        x[i] = acc * rinv[b0 + i];                        // zero for i < c (acc stays 0)
      }
#pragma unroll
      for (int i = 0; i < SBK; ++i) X[(b0 + i) * LDS + b0 + lane] = x[i];
    }
    __syncthreads();
    if (nrem > 0) {                       // A3: trailing S[i][j] -= sum_k P[i][k] P[j][k], j <= i
      const int nt = nrem >> 2;           // 4x4 tiles per side
      const int ntiles = nt * (nt + 1) / 2;
      for (int t = tid; t < ntiles; t += 256) {
        // unrank the lower-triangular tile index t -> (ti >= tj)
        int ti = static_cast<int>((sqrtf(8.f * t + 1.f) - 1.f) * 0.5f);
        while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
        while (ti * (ti + 1) / 2 > t) --ti;
        const int tj = t - ti * (ti + 1) / 2;
        const int r0 = b0 + SBK + ti * 4, c0 = b0 + SBK + tj * 4;
        float acc[4][4];
#pragma unroll
        for (int x = 0; x < 4; ++x)
#pragma unroll
          for (int y = 0; y < 4; ++y) acc[x][y] = 0.f;
#pragma unroll 8
        for (int k = 0; k < SBK; ++k) {
          float pr[4], pc[4];
#pragma unroll
          for (int x = 0; x < 4; ++x) { pr[x] = S[(r0 + x) * LDS + b0 + k]; pc[x] = S[(c0 + x) * LDS + b0 + k]; }
#pragma unroll
          for (int x = 0; x < 4; ++x)
#pragma unroll
            for (int y = 0; y < 4; ++y) acc[x][y] = fmaf(pr[x], pc[y], acc[x][y]);
        }
#pragma unroll
        for (int x = 0; x < 4; ++x)
#pragma unroll
          for (int y = 0; y < 4; ++y)
            if (c0 + y <= r0 + x) S[(r0 + x) * LDS + c0 + y] -= acc[x][y];
      }
    }
    __syncthreads();
  }

  // ---------------- phase B: X = L^-1 (the diagonal 32x32 inverses were built in phase A) ------
  // B2: off-diagonal blocks by distance d = i - j; thread (ty, tx) of a 16x16 grid owns a 2x2 patch
  {
    const int tx = tid & 15, ty = tid >> 4;
    for (int d = 1; d < NB / SBK; ++d) {
      for (int bi = d; bi < NB / SBK; ++bi) {
        const int bj = bi - d;
        const int ri = bi * SBK, cj = bj * SBK;
        // T = sum_{k=bj}^{bi-1} L[bi][k] X[k][bj]   (X[k][bj] for k > bj was produced at smaller d)
        float t00 = 0.f, t01 = 0.f, t10 = 0.f, t11 = 0.f;
        for (int kk = cj; kk < ri; ++kk) {
          const float l0 = S[(ri + 2 * ty) * LDS + kk], l1 = S[(ri + 2 * ty + 1) * LDS + kk];
          const float x0 = X[kk * LDS + cj + 2 * tx], x1 = X[kk * LDS + cj + 2 * tx + 1];
          t00 = fmaf(l0, x0, t00); t01 = fmaf(l0, x1, t01);
          t10 = fmaf(l1, x0, t10); t11 = fmaf(l1, x1, t11);
        }
        // stash T in the (still unused) X[bi][bj] block
        X[(ri + 2 * ty) * LDS + cj + 2 * tx] = t00;
        X[(ri + 2 * ty) * LDS + cj + 2 * tx + 1] = t01;
        X[(ri + 2 * ty + 1) * LDS + cj + 2 * tx] = t10;
        X[(ri + 2 * ty + 1) * LDS + cj + 2 * tx + 1] = t11;
        __syncthreads();
        // X[bi][bj] = -X[bi][bi] * T
        float o00 = 0.f, o01 = 0.f, o10 = 0.f, o11 = 0.f;
        for (int m = 0; m < SBK; ++m) {
          const float a0 = X[(ri + 2 * ty) * LDS + ri + m], a1 = X[(ri + 2 * ty + 1) * LDS + ri + m];
          const float b0v = X[(ri + m) * LDS + cj + 2 * tx], b1v = X[(ri + m) * LDS + cj + 2 * tx + 1];
          o00 = fmaf(a0, b0v, o00); o01 = fmaf(a0, b1v, o01);
          o10 = fmaf(a1, b0v, o10); o11 = fmaf(a1, b1v, o11);
        }
        __syncthreads();
        X[(ri + 2 * ty) * LDS + cj + 2 * tx] = -o00;
        X[(ri + 2 * ty) * LDS + cj + 2 * tx + 1] = -o01;
        X[(ri + 2 * ty + 1) * LDS + cj + 2 * tx] = -o10;
        X[(ri + 2 * ty + 1) * LDS + cj + 2 * tx + 1] = -o11;
        __syncthreads();
      }
    }
  }
  for (int idx = tid; idx < NB * NB; idx += 256) {
    const int i = idx >> 7, j = idx & 127;
    if (i < nb && j < nb) {
      // L_kk and the tf32 split of X = L_kk^-1 in the diagonal block of Lhi/Llo, where the GEMMs
      // that multiply by X read it (K-major, ld n), zero above the diagonal; and the diagonal
      // block of Z = Y^T = L^-T with its tf32 split, (i, j) = X[j][i] for j >= i (the part below
      // the diagonal is zero from the memsets at the start of llmc_chol_inv_upper).
      const int64_t o = (k0 + i) * n + k0 + j;
      if (j <= i) G[o] = S[i * LDS + j];
      const float2 s = tf32_split(j <= i ? X[i * LDS + j] : 0.f);
      Lhi[o] = s.x;
      Llo[o] = s.y;
      if (j >= i) {
        const float z = X[j * LDS + i];
        const float2 t = tf32_split(z);
        Z[o] = z;
        Zhi[o] = t.x;
        Zlo[o] = t.y;
      }
    }
  }
}

}  // namespace ch
}  // namespace llmc

using namespace llmc;

extern "C" int64_t llmc_chol_workspace_bytes(int64_t C) {
  if (C <= 0) return 0;
  // G, Lhi, Llo, Z, Zhi, Zlo (C^2 each)
  return 6 * C * C * 4 + 256;
}

extern "C" int llmc_chol_inv_upper(float* A, int64_t C, void* workspace, int64_t workspace_bytes,
                                   int* info, void* stream) {
  using namespace ch;
  LLMC_CHECK_ARG(A && workspace && info && C > 0, "chol_inv_upper: bad argument");
  LLMC_CHECK_ARG(C % 8 == 0, "chol_inv_upper: C=%lld must be a multiple of 8", (long long)C);
  LLMC_CHECK_ARG(workspace_bytes >= llmc_chol_workspace_bytes(C), "chol_inv_upper: workspace too small");
  LLMC_CHECK_ARG(aligned16(A) && aligned16(workspace), "chol_inv_upper: 16-byte alignment required");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t n = C, nn = C * C;
  const int64_t nbk = (n + NB - 1) / NB;
  float* G = reinterpret_cast<float*>(workspace);
  float* Lhi = G + nn;
  float* Llo = Lhi + nn;
  float* Z = Llo + nn;
  float* Zhi = Z + nn;
  float* Zlo = Zhi + nn;
  // tf32 split of L's sub-diagonal panels, and of L_kk^-1 in the diagonal blocks
  const SplitMatrix L{Lhi, Llo, n};
  // tf32 split of Z = Y^T = L^-T.  The inverse is kept transposed so that every update of it reads
  // both operands K-major: Y[r0:, 0:r0] -= L[r0:, k] Y[k, 0:r0] is Z[0:r0, r0:] -= Z[0:r0, k] L[r0:, k]^T.
  const SplitMatrix Zs{Zhi, Zlo, n};
  const int diag_smem = 2 * NB * LDS * 4;
  if (int rc = opt_in_smem(diag_kernel, diag_smem)) return rc;
  // Side streams + events (common.cuh); the call stays asynchronous with respect to the host and
  // ordered on `stream` through the final join.
  SideStreams* side = nullptr;
  if (int rc = side_streams(nbk + 1, &side)) return rc;
  cudaEvent_t* ev = side->ev[0].data();   // L panel kb and L_kk^-1 final
  // super-panel width of the lazy trailing updates: 4 blocks
  constexpr int64_t spw = 4 * NB;
  LLMC_CHECK_CUDA(cudaMemsetAsync(info, 0, sizeof(int), st));
  LLMC_CHECK_CUDA(cudaMemsetAsync(Z, 0, nn * sizeof(float), st));
  // the inverse updates read Zhi/Zlo over whole super-panel columns: the part below the diagonal
  // (blocks) inside each super-panel square is never written, so it must be zero
  for (int64_t s0 = 0; s0 < n; s0 += spw) {
    const int64_t w = (s0 + spw < n) ? spw : n - s0;
    LLMC_CHECK_CUDA(cudaMemset2DAsync(Zhi + s0 * n + s0, n * sizeof(float), 0, w * sizeof(float), w, st));
    LLMC_CHECK_CUDA(cudaMemset2DAsync(Zlo + s0 * n + s0, n * sizeof(float), 0, w * sizeof(float), w, st));
  }
  int64_t blocks = (nn + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  reverse_kernel<<<(int)blocks, 256, 0, st>>>(A, G, n);
  LLMC_CHECK_LAUNCH();
  const dim3 tiles32(static_cast<unsigned>((n + 31) / 32), static_cast<unsigned>((n + 31) / 32));

  auto width = [n](int64_t k0) { return static_cast<int>((n - k0) < NB ? (n - k0) : NB); };
  // Step kb of the factorisation on stream s, once column block kb is up to date: factor and invert
  // the diagonal block, then the panel below it.  ev[kb] marks L panel kb and L_kk^-1 final.
  auto factor_block = [&](int64_t kb, cudaStream_t s) -> int {
    const int64_t k0 = kb * NB;
    const int nb = width(k0);
    const int64_t r0 = k0 + nb;
    const int64_t m = n - r0;
    diag_kernel<<<1, 256, diag_smem, s>>>(G, n, k0, nb, Z, Zhi, Zlo, Lhi, Llo, info);
    LLMC_CHECK_LAUNCH();
    if (m > 0) {
      float* P = G + r0 * n + k0;          // panel [m x nb], ld n
      // the split of panel 0 is made here; later panels get theirs from the trailing updates
      if (kb == 0)
        if (int rc = split_tf32(P, m, nb, n, Lhi + r0 * n + k0, Llo + r0 * n + k0, n, s)) return rc;
      // P <- P * L_kk^-T : out[i][j] = sum_k P[i][k] * X[j][k]  (both K-major; X = L_kk^-1 is the
      // diagonal block of Lhi/Llo), + split
      if (int rc = tf32x3_update(
              Tf32x3Update{L.at(r0, k0), L.at(k0, k0), P, n, m, nb, nb}.overwrite().split_into(L, r0, k0), s))
        return rc;
    }
    LLMC_CHECK_CUDA(cudaEventRecord(ev[kb], s));
    return LLMC_OK;
  };
  // Row step kb of the inverse on stream s, after ev[kb]: Y[k rows, 0:k0] = Y_kk T'[k rows, 0:k0],
  // kept transposed: Z[0:k0, k cols] = T'^T Y_kk^T (T'^T = Z[0:k0, k cols], Y_kk = the diagonal
  // block of Lhi/Llo, both K-major); the split of T'^T was emitted by step kb-1.
  auto inverse_row = [&](int64_t kb, cudaStream_t s) -> int {
    LLMC_CHECK_CUDA(cudaStreamWaitEvent(s, ev[kb], 0));
    if (kb == 0) return LLMC_OK;
    const int64_t k0 = kb * NB;
    const int nb = width(k0);
    return tf32x3_update(
        Tf32x3Update{Zs.at(0, k0), L.at(k0, k0), Z + k0, n, k0, nb, nb}.overwrite().split_into(Zs, 0, k0).transpose(), s);
  };

  // More than one super-panel: the look-ahead schedule; otherwise the serial schedule below.
  if (n > spw) {
    // ================= look-ahead schedule ====================================================
    // The factorisation's dependent chain is  diag(k) -> panel solve(k) -> update of column block
    // k+1  (1..112 CTAs wide); everything else — 90 % of the flops — is
    // off that chain.  Side streams:
    //   hi    highest priority : the chain.  Inside a super-panel of 4 blocks it is LEFT-looking
    //                            (column block j receives the rank-128*(j-j0) update of its
    //                            super-panel's earlier panels right before it is factored); at a
    //                            super-panel boundary it applies the rank-512 update to the next
    //                            column block only.
    //   bulk  lowest priority  : the rest of each rank-512 trailing update, first the part the
    //                            chain needs next (A': the following 512 columns, event evA), then
    //                            everything beyond (B).  One tile per CTA, so SMs return to the
    //                            chain within a tile time.
    //   si    middle priority  : the inverse chain (needs panel k of L only), with its own bulk
    //                            stream s3 for the rows beyond the next super-panel.
    // Every column block receives its updates in a fixed order (events), so the result does not
    // depend on timing.
    cudaStream_t hi = side->stream[kChain], bulk = side->stream[kBulk];
    cudaStream_t si = side->stream[kInverse], s3 = side->stream[kInverseBulk];
    cudaEvent_t* evA = side->ev[1].data();    // A' of super-panel s done (bulk)
    cudaEvent_t* evI = side->ev[2].data();    // inverse chain reached the end of super-panel s
    cudaEvent_t* evIB = side->ev[3].data();   // inverse bulk of super-panel s done (s3)
    if (int rc = side->fork(st, {kChain})) return rc;
    for (int64_t kb = 0; kb < nbk; ++kb) {
      const int64_t k0 = kb * NB;
      const int nb = width(k0);
      const int64_t sidx = k0 / spw;
      const int64_t sp0 = sidx * spw;
      const int64_t sp1 = (sp0 + spw < n) ? sp0 + spw : n;
      const int64_t r0 = k0 + nb;
      const int64_t m = n - r0;
      // ---- chain (hi): bring column block kb up to date ----
      if (k0 > sp0) {
        if (sidx > 0 && k0 == sp0 + NB)      // columns sp0+128.. of this super-panel come from A' of the previous one
          LLMC_CHECK_CUDA(cudaStreamWaitEvent(hi, evA[sidx - 1], 0));
        // G[k0:, k0:k0+nb] -= L[k0:, sp0:k0] L[k0:k0+nb, sp0:k0]^T ; emits the split of the block
        if (int rc = tf32x3_update(Tf32x3Update{L.at(k0, sp0), L.at(k0, sp0), G + k0 * n + k0, n, n - k0, nb,
                                                k0 - sp0}.split_into(L, k0, k0), hi))
          return rc;
      }
      if (int rc = factor_block(kb, hi)) return rc;
      if (m > 0 && r0 == sp1) {
        // ---- super-panel boundary: rank-(sp1-sp0) update of G[sp1:, sp1:] in three pieces ----
        const int64_t kk = sp1 - sp0;
        const SplitOperand Lsp = L.at(sp1, sp0);   // L[sp1:, sp0:sp1]
        const int64_t w1 = (n - sp1) < NB ? (n - sp1) : NB;
        // chain: the next column block (also waits for what earlier bulk pieces wrote there)
        if (sidx > 0) LLMC_CHECK_CUDA(cudaStreamWaitEvent(hi, evA[sidx - 1], 0));
        if (int rc = tf32x3_update(
                Tf32x3Update{Lsp, Lsp, G + sp1 * n + sp1, n, n - sp1, w1, kk}.split_into(L, sp1, sp1), hi))
          return rc;
        // bulk: A' = columns [sp1+128, sp1+128+spw), then B = the rest; lower tiles only
        LLMC_CHECK_CUDA(cudaStreamWaitEvent(bulk, ev[kb], 0));
        const int64_t ca = sp1 + NB;
        const int64_t cb = (ca + spw < n) ? ca + spw : n;
        if (ca < n) {
          if (int rc = tf32x3_update(Tf32x3Update{Lsp, L.at(ca, sp0), G + sp1 * n + ca, n, n - sp1, cb - ca, kk}
                                         .lower_tiles(sp1, ca).tile_per_cta(), bulk))
            return rc;
        }
        LLMC_CHECK_CUDA(cudaEventRecord(evA[sidx], bulk));
        if (cb < n) {
          if (int rc = tf32x3_update(Tf32x3Update{Lsp, L.at(cb, sp0), G + sp1 * n + cb, n, n - sp1, n - cb, kk}
                                         .lower_tiles(sp1, cb).tile_per_cta(), bulk))
            return rc;
        }
      }
      // ---- inverse chain (si): Y = L^-1 as Z = Y^T, one block column per panel ----
      if (int rc = inverse_row(kb, si)) return rc;
      if (m > 0 && r0 < sp1) {
        if (int rc = tf32x3_update(Tf32x3Update{Zs.at(0, k0), L.at(r0, k0), Z + r0, n, r0, sp1 - r0, nb}
                                       .split_into(Zs, 0, r0).split_first_cols(NB).transpose(), si))
          return rc;
      } else if (m > 0) {
        // T'[sp1:, 0:sp1] -= L[sp1:, sp0:sp1] Y[sp0:sp1, 0:sp1], as its transpose: the next
        // super-panel's columns on the chain, the columns beyond on s3 (they are next touched by
        // the following boundary's pieces, which wait for evIB)
        const int64_t kk = sp1 - sp0;
        const int64_t ra = (sp1 + spw < n) ? sp1 + spw : n;
        if (sidx > 0) LLMC_CHECK_CUDA(cudaStreamWaitEvent(si, evIB[sidx - 1], 0));
        if (int rc = tf32x3_update(Tf32x3Update{Zs.at(0, sp0), L.at(sp1, sp0), Z + sp1, n, sp1, ra - sp1, kk}
                                       .split_into(Zs, 0, sp1).split_first_cols(NB).transpose(), si))
          return rc;
        LLMC_CHECK_CUDA(cudaEventRecord(evI[sidx], si));
        LLMC_CHECK_CUDA(cudaStreamWaitEvent(s3, evI[sidx], 0));
        if (ra < n) {
          if (int rc = tf32x3_update(Tf32x3Update{Zs.at(0, sp0), L.at(ra, sp0), Z + ra, n, sp1, n - ra, kk}
                                         .tile_per_cta().transpose(), s3))
            return rc;
        }
        LLMC_CHECK_CUDA(cudaEventRecord(evIB[sidx], s3));
      }
    }
    if (int rc = side->join(st, {kChain, kBulk, kInverse, kInverseBulk})) return rc;
    reverse_upper_kernel<<<tiles32, 256, 0, st>>>(Z, A, n);
    LLMC_CHECK_LAUNCH();
    return LLMC_OK;
  }

  // ================= serial schedule (n <= spw: one super-panel) ==============================
  // The factorisation runs on `stream`, the inverse steps on the least-priority side stream.
  cudaStream_t inv = side->stream[kBulk];
  // ---- factor: G = L L^T (lower, in place), Lhi/Llo = split of the sub-diagonal panels ----
  for (int64_t kb = 0; kb < nbk; ++kb) {
    const int64_t k0 = kb * NB;
    const int nb = width(k0);
    const int64_t r0 = k0 + nb;
    const int64_t m = n - r0;
    if (int rc = factor_block(kb, st)) return rc;
    if (m > 0) {
      // G[r0:, r0:] -= P P^T  (lower tiles only); emits the tf32 split of the next panel
      if (int rc = tf32x3_update(Tf32x3Update{L.at(r0, k0), L.at(r0, k0), G + r0 * n + r0, n, m, m, nb}
                                     .lower_tiles(0, 0).split_into(L, r0, r0).split_first_cols(NB), st))
        return rc;
    }

    // ---- inverse step kb on the side stream: Y = L^-1 (lower), kept as Z = Y^T.  T' (stored in
    //      Y below the diagonal blocks, in Z above them) accumulates -sum_{k<i} L_ik Y_k ;
    //      Y_i = Y_ii T'_i.  It needs panel kb of L only, so it overlaps the factorisation's
    //      trailing update and later steps. ----
    if (int rc = inverse_row(kb, inv)) return rc;
    if (m > 0) {
      // T'[r0:, 0:r0] -= L[r0:, kblock] * Y[k rows, 0:r0] as Z[0:r0, r0:] -= Z[0:r0, k cols] *
      // L[r0:, kblock]^T; emits the split of the next T' rows (Z columns)
      if (int rc = tf32x3_update(Tf32x3Update{Zs.at(0, k0), L.at(r0, k0), Z + r0, n, r0, m, nb}
                                     .split_into(Zs, 0, r0).split_first_cols(NB).transpose(), inv))
        return rc;
    }
  }
  if (int rc = side->join(st, {kBulk})) return rc;
  reverse_upper_kernel<<<tiles32, 256, 0, st>>>(Z, A, n);
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}
