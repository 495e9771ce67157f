// gptq.cu — K5: GPTQ column-block update, plus the gathers around it.
//
// Replaces GPTQ.process_hessian_and_weights (dead columns, act-order gather, damping;
// llmc/compression/quantization/gptq.py:128-171) and GPTQ.weight_transform (:198-244) with
// search_column_qparams (:358-366).  The reference spends ~15 tiny launches per COLUMN; here a
// 128-column block is one launch of `gptq_inblock_kernel` (rows are independent: eight lanes
// share one weight row, 32 rows per CTA, the row tile and the 128x128 Hinv block live in shared
// memory) followed by the trailing update W[:, i2:] -= Err1 @ Hinv[i1:i2, i2:] (:244) as a 3xTF32
// GEMM (tf32.cu), or the fp32 `trailing_update_kernel` where the operands do not allow TMA.
//
// Numerics: fp32 throughout like the reference (gptq.py:135).  Inside a block every op is
// rounded exactly like torch (separate multiply and subtract for the rank-1 updates, :240;
// correctly rounded divides), so single-block problems are bit-exact; across blocks only the
// summation order of the 128-deep trailing dot products differs from the CPU BLAS.
#include "tc.cuh"
#include "quant_math.cuh"
#include "spqr_row.cuh"

namespace llmc {

constexpr int GB = 128;          // gptq blocksize (gptq_w_only.yml: blocksize 128)
// Trailing updates are applied lazily per super-panel of 4 blocks: inside the super-panel each
// block updates only the super-panel's remaining columns (rank 128), and the columns beyond it get
// ONE rank-512 update.  Same terms as gptq.py:244 block by block, grouped differently (fp32
// summation order only), and a quarter of the read-modify-write traffic over W.
constexpr int kSuperPanel = 4 * GB;

// ---- prepare -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
diag_mean_kernel(const float* __restrict__ H, int64_t C, float percdamp, float* __restrict__ out) {
  // out[0] = percdamp * mean(diag(H) with zeros replaced by 1)   (gptq.py:139-140, 169)
  __shared__ float red[8];
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < C; i += blockDim.x) {
    const float d = H[i * C + i];
    acc += (d == 0.f) ? 1.f : d;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) out[0] = percdamp * (v / static_cast<float>(C));
  }
}

__global__ void __launch_bounds__(256)
gather_h_kernel(const float* __restrict__ H, int64_t C, const int64_t* __restrict__ perm,
                const float* __restrict__ damp, float* __restrict__ Hp) {
  extern __shared__ float row[];
  const int64_t i = blockIdx.x;
  const int64_t pi = perm ? perm[i] : i;
  for (int64_t j = threadIdx.x; j < C; j += blockDim.x) row[j] = H[pi * C + j];
  __syncthreads();
  const float dmp = damp[0];
  for (int64_t j = threadIdx.x; j < C; j += blockDim.x) {
    const int64_t pj = perm ? perm[j] : j;
    float v = row[pj];
    if (i == j) v = ((v == 0.f) ? 1.f : v) + dmp;
    Hp[i * C + j] = v;
  }
}

template <int WT>
__global__ void __launch_bounds__(256)
gather_w_kernel(const void* __restrict__ W, int64_t R, int64_t C, const float* __restrict__ H,
                const int64_t* __restrict__ perm, float* __restrict__ Wp) {
  extern __shared__ float row[];
  const int64_t r = blockIdx.x;
  for (int64_t j = threadIdx.x; j < C; j += blockDim.x) row[j] = DType<WT>::load(W, r * C + j);
  __syncthreads();
  for (int64_t j = threadIdx.x; j < C; j += blockDim.x) {
    const int64_t pj = perm ? perm[j] : j;
    const bool dead = H[pj * C + pj] == 0.f;
    Wp[r * C + j] = dead ? 0.f : row[pj];
  }
}

// ---- in-block column loop ------------------------------------------------------------------------------
struct InblockArgs {
  float* W;              // [R, C] fp32 working copy (permuted)
  const float* Hinv;     // [C, C] upper factor
  int64_t R, C;
  int i1, count;         // block start, columns in this block (<= 128)
  int64_t group;         // elements per group (C for per_channel)
  int64_t ng;
  int sym;
  float qmin, qmax;
  int static_groups;     // qparams are inputs
  const int32_t* gmap;   // static: column -> group index (perm[idx]/g), may be null
  void* scales;          // dynamic: fp32 out [R, ng]; static: q_dtype in
  void* zeros;
  int q_dtype;
  float* tmp;            // [R, C] out
  const int64_t* out_perm;  // optional: scatter tmp columns back to the original order
  float* losses;         // [R] accumulated
  float* err;            // [128, Rpad] out (Err1 transposed)
  float* err_hi;         // tf32 split of err
  float* err_lo;
  int64_t Rpad;          // R rounded up to 128
};

// A row is spread over 8 lanes (lane l owns columns l, l+8, ...), 32 rows per CTA, 256 threads,
// two CTAs per SM (one thread per row would give R = 4096 only 32 CTAs, one warp per scheduler):
//   * per 8-column sub-block each lane keeps ITS column in a register; the eight sequential
//     quantise -> err -> rank-1 steps exchange `err` with one width-8 shuffle each;
//   * the other columns of the row stay in shared memory and receive the sub-block's eight
//     updates lazily, in the reference's order (same op sequence per element as gptq.py:240);
//   * x / s with s fixed is evaluated as a reciprocal multiply plus two FMA corrections
//     (MarksteinDiv, quant_math.cuh), which is the correctly rounded quotient, at a third of
//     div.rn's cost.
constexpr int IR = 32;            // rows per CTA
constexpr int IL = 8;             // lanes per row
constexpr int WP = GB + 8;        // pitch of the row-major W tile: 4 rows x 8 lanes hit 32 banks
constexpr int EP = IR + 1;        // pitch of the transposed err tile
constexpr int HP = GB + 4;        // pitch of the row-major Hinv block
constexpr int kInblockSmem = (IR * WP + GB * EP + GB * HP + 2 * GB) * 4;

__device__ __forceinline__ float group8_min(float v) {
  v = fminf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  v = fminf(v, __shfl_xor_sync(0xffffffffu, v, 2));
  return fminf(v, __shfl_xor_sync(0xffffffffu, v, 4));
}
__device__ __forceinline__ float group8_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
}

__global__ void __launch_bounds__(IR * IL, 2)
gptq_inblock_kernel(InblockArgs a) {
  extern __shared__ float sm[];
  float* Wr = sm;                        // [32 rows][136]   current (lazily updated) weights
  float* Et = Wr + IR * WP;              // [128 cols][33]   err (Err1 transposed)
  float* Hs = Et + GB * EP;              // [128 j][132]     Hs[j][k] = Hinv1[j][k]
  float* dd = Hs + GB * HP;              // [128] Hinv1[c][c]
  float* rd = dd + GB;                   // [128] RN(1 / Hinv1[c][c])
  const int tid = threadIdx.x, rg = tid >> 3, l = tid & 7;
  const int warp = tid >> 5, lane = tid & 31;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * IR;
  const int64_t row = r0 + rg;
  const bool live = row < a.R;
  const int cnt = a.count;

  {
    const bool vec = (cnt == GB) && ((a.C & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.W) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(a.Hinv) & 15) == 0);
    if (vec) {
      float4 v[8];
#pragma unroll
      for (int b = 0; b < 4; ++b) {        // W tile: 32 rows x 32 float4
        const int item = b * (IR * IL) + tid;
        const int rr = item >> 5, c4 = item & 31;
        const int64_t r = r0 + rr;
        v[b] = (r < a.R) ? *reinterpret_cast<const float4*>(&a.W[r * a.C + a.i1 + c4 * 4])
                         : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int item = b * (IR * IL) + tid;
        const int rr = item >> 5, c4 = item & 31;
        *reinterpret_cast<float4*>(&Wr[rr * WP + c4 * 4]) = v[b];
      }
#pragma unroll 1
      for (int base = 0; base < GB * 32; base += 8 * IR * IL) {   // Hinv block: 128 rows x 32 float4
#pragma unroll
        for (int b = 0; b < 8; ++b) {
          const int item = base + b * (IR * IL) + tid;
          const int i = item >> 5, j4 = item & 31;
          v[b] = *reinterpret_cast<const float4*>(
              &a.Hinv[(static_cast<int64_t>(a.i1) + i) * a.C + a.i1 + j4 * 4]);
        }
#pragma unroll
        for (int b = 0; b < 8; ++b) {
          const int item = base + b * (IR * IL) + tid;
          const int i = item >> 5, j4 = item & 31;
          *reinterpret_cast<float4*>(&Hs[i * HP + j4 * 4]) = v[b];
        }
      }
    } else {
      for (int idx = tid; idx < IR * GB; idx += IR * IL) {
        const int rr = idx >> 7, c = idx & 127;
        const int64_t r = r0 + rr;
        Wr[rr * WP + c] = (r < a.R && c < cnt) ? a.W[r * a.C + a.i1 + c] : 0.f;
      }
      for (int idx = tid; idx < GB * GB; idx += IR * IL) {
        const int i = idx >> 7, j = idx & 127;
        Hs[i * HP + j] = (i < cnt && j < cnt) ? a.Hinv[(static_cast<int64_t>(a.i1) + i) * a.C + a.i1 + j]
                                               : 0.f;
      }
    }
  }
  __syncthreads();
  if (tid < GB) {
    const float d = (tid < cnt) ? Hs[tid * HP + tid] : 1.f;
    dd[tid] = d;
    rd[tid] = __frcp_rn(d);
  }

  // ---- qparams of the groups that start inside this block (gptq.py:215-223), searched on W as
  //      it stands at block entry (the reference indexes the global W, not the in-block clone)
  float s_cur = 1.f, z_cur = 0.f;
  const bool dynamic = !a.static_groups;
  const int gsz = static_cast<int>(a.group < GB ? a.group : GB);
  float s_small[8], z_small[8];
#pragma unroll
  for (int g = 0; g < 8; ++g) { s_small[g] = 1.f; z_small[g] = 0.f; }
  if (dynamic) {
    if (a.group >= GB) {
      const int64_t gi = a.i1 / a.group;
      if ((a.i1 % a.group) == 0) {
        float mn = INFINITY, mx = -INFINITY;
        const int64_t gend = min(static_cast<int64_t>(a.i1) + a.group, a.C);
        if (gend - a.i1 <= cnt) {
          for (int c = l; c < cnt; c += IL) { const float v = Wr[rg * WP + c]; mn = fminf(mn, v); mx = fmaxf(mx, v); }
        } else if (live) {
          for (int64_t c = a.i1 + l; c < gend; c += IL) { const float v = a.W[row * a.C + c]; mn = fminf(mn, v); mx = fmaxf(mx, v); }
        } else {
          mn = 0.f; mx = 0.f;
        }
        mn = group8_min(mn); mx = group8_max(mx);
        qparams<F32Round>(mn, mx, a.sym, 1, a.qmin, a.qmax, s_cur, z_cur);
        if (live && l == 0) {
          reinterpret_cast<float*>(a.scales)[row * a.ng + gi] = s_cur;
          if (!a.sym) reinterpret_cast<float*>(a.zeros)[row * a.ng + gi] = z_cur;
        }
      } else if (live) {                   // group opened by an earlier block
        s_cur = reinterpret_cast<const float*>(a.scales)[row * a.ng + gi];
        z_cur = a.sym ? 0.f : reinterpret_cast<const float*>(a.zeros)[row * a.ng + gi];
      }
    } else {
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        if (g * gsz < cnt) {               // uniform across the CTA
          float mn = INFINITY, mx = -INFINITY;
          const int cend = min((g + 1) * gsz, cnt);
          for (int c = g * gsz + l; c < cend; c += IL) { const float v = Wr[rg * WP + c]; mn = fminf(mn, v); mx = fmaxf(mx, v); }
          mn = group8_min(mn); mx = group8_max(mx);
          qparams<F32Round>(mn, mx, a.sym, 1, a.qmin, a.qmax, s_small[g], z_small[g]);
          if (live && l == 0) {
            const int64_t gi = (a.i1 + g * gsz) / a.group;
            reinterpret_cast<float*>(a.scales)[row * a.ng + gi] = s_small[g];
            if (!a.sym) reinterpret_cast<float*>(a.zeros)[row * a.ng + gi] = z_small[g];
          }
        }
      }
    }
  } else if (live && a.group >= a.C) {
    s_cur = load_as(a.q_dtype, a.scales, row);                 // per_channel
    z_cur = a.zeros ? load_as(a.q_dtype, a.zeros, row) : 0.f;
  }
  __syncthreads();                         // dd / rd

  float loss = 0.f;
  const int nsb = (cnt + IL - 1) / IL;
#pragma unroll 1
  for (int m = 0; m < nsb; ++m) {
    const int cb = m * IL, c_own = cb + l;
    const bool col_live = c_own < cnt;
    float s = s_cur, z = z_cur;
    if (dynamic && a.group < GB) {
      const int g = cb / gsz;              // a sub-block of 8 never straddles a group (group >= 16)
#pragma unroll
      for (int t = 0; t < 8; ++t) { if (g == t) { s = s_small[t]; z = z_small[t]; } }
    } else if (!dynamic && a.group < a.C && live && col_live) {
      const int64_t idx = static_cast<int64_t>(a.i1) + c_own;
      const int64_t gi = a.gmap ? a.gmap[idx] : idx / a.group;     // gptq.py:225-227
      s = load_as(a.q_dtype, a.scales, row * a.ng + gi);
      z = a.zeros ? load_as(a.q_dtype, a.zeros, row * a.ng + gi) : 0.f;
    }
    const MarksteinDiv div_s(s);
    float wc = Wr[rg * WP + c_own];
    float hd[IL];
#pragma unroll
    for (int jj = 0; jj < IL; ++jj) hd[jj] = Hs[(cb + jj) * HP + c_own];
    const float d = dd[c_own];
    const MarksteinDiv div_d(d, rd[c_own]);
    float ev[IL];
    float my_err = 0.f, my_diff = 0.f;
    // the eight sequential columns of the sub-block: lane jj's column is final at step jj
#pragma unroll
    for (int jj = 0; jj < IL; ++jj) {
      const float q = dequant<F32Round>(quant_code<F32Round>(wc, div_s, z, a.qmin, a.qmax), s, z);
      const float diff = fsub_rn(wc, q);
      float err = div_d(diff);                                                      // :239
      if (!col_live) err = 0.f;
      const float e = __shfl_sync(0xffffffffu, err, jj, IL);
      ev[jj] = e;
      if (l == jj) { my_err = err; my_diff = diff; }
      if (l > jj) wc = fsub_rn(wc, fmul_rn(e, hd[jj]));                       // :240
    }
    if (col_live) loss += fdiv_rn(fmul_rn(my_diff, my_diff), fmul_rn(2.f, fmul_rn(d, d)));   // :238
    Wr[rg * WP + c_own] = wc;              // tmp: the compensated, not yet rounded weight (:237)
    Et[c_own * EP + rg] = my_err;          // Err1 (:241)
    // lazy propagation of the sub-block's eight errors to the later columns this lane owns
    int mp = m + 1;
    for (; mp + 3 < nsb; mp += 4) {
      float w0 = Wr[rg * WP + (mp + 0) * IL + l], w1 = Wr[rg * WP + (mp + 1) * IL + l];
      float w2 = Wr[rg * WP + (mp + 2) * IL + l], w3 = Wr[rg * WP + (mp + 3) * IL + l];
      const float* hp = Hs + cb * HP + mp * IL + l;
#pragma unroll
      for (int jj = 0; jj < IL; ++jj) {
        w0 = fsub_rn(w0, fmul_rn(ev[jj], hp[jj * HP]));
        w1 = fsub_rn(w1, fmul_rn(ev[jj], hp[jj * HP + IL]));
        w2 = fsub_rn(w2, fmul_rn(ev[jj], hp[jj * HP + 2 * IL]));
        w3 = fsub_rn(w3, fmul_rn(ev[jj], hp[jj * HP + 3 * IL]));
      }
      Wr[rg * WP + (mp + 0) * IL + l] = w0; Wr[rg * WP + (mp + 1) * IL + l] = w1;
      Wr[rg * WP + (mp + 2) * IL + l] = w2; Wr[rg * WP + (mp + 3) * IL + l] = w3;
    }
    for (; mp < nsb; ++mp) {
      float w0 = Wr[rg * WP + mp * IL + l];
      const float* hp = Hs + cb * HP + mp * IL + l;
#pragma unroll
      for (int jj = 0; jj < IL; ++jj) w0 = fsub_rn(w0, fmul_rn(ev[jj], hp[jj * HP]));
      Wr[rg * WP + mp * IL + l] = w0;
    }
  }
  loss += __shfl_xor_sync(0xffffffffu, loss, 4);
  loss += __shfl_xor_sync(0xffffffffu, loss, 2);
  loss += __shfl_xor_sync(0xffffffffu, loss, 1);
  if (live && l == 0) a.losses[row] += loss;
  __syncthreads();
  // write-back: tmp[:, invperm] (gptq.py:186-188) fused as a scatter — permuted column i1+c goes
  // back to original column perm[i1+c] — and Err1 transposed ([k][row], so the trailing GEMM
  // reads its A operand with unit stride) with its tf32 split
  for (int rr = warp; rr < IR; rr += (IR * IL) / 32) {
    const int64_t r = r0 + rr;
    if (r >= a.R) break;
    for (int c = lane; c < cnt; c += 32) {
      const int64_t oc = a.out_perm ? a.out_perm[a.i1 + c] : static_cast<int64_t>(a.i1) + c;
      a.tmp[r * a.C + oc] = Wr[rr * WP + c];
    }
  }
  if (r0 + lane < a.Rpad) {
    for (int c = warp; c < GB; c += (IR * IL) / 32) {
      const float evv = (c < cnt) ? Et[c * EP + lane] : 0.f;
      const int64_t o = static_cast<int64_t>(c) * a.Rpad + r0 + lane;
      a.err[o] = evv;
      uint32_t hb, lb;                                   // tf32 split for the 3xTF32 trailing GEMM
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(evv));
      const float h = __uint_as_float(hb);
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(evv - h));
      a.err_hi[o] = h;
      a.err_lo[o] = __uint_as_float(lb);
    }
  }
}


// ---- SpQR in-block kernel (spqr.py:215-268) ------------------------------------------------------------------
// Same role as gptq_inblock_kernel for the SpQR sweep (rows are independent): the row tile / Hinv
// block / Err1 / outlier mask live in shared memory.  Per group of `gs` columns: leave-one-out
// outlier search (gs * (gs - 1) quantise-dequantise evaluations per row), bilevel (scale / zero)
// quantisation; per column: quantise, unstructured outlier mask, rank-1 update of the block's
// remaining columns.
struct SpqrArgs {
  float* W;
  const float* Hinv;
  int64_t R, C, Rpad;
  int i1, count;
  int64_t ng;
  spqr::Cfg cfg;             // thr / has_thr / outliers are filled in by the kernel from `thr`
  const float* thr;          // device scalar: relative_threshold * outlier_scale (may be +inf)
  int simplified;
  float* scales;             // [R, ng] out
  float* zeros;              // [R, ng] out
  float* tmp;                // [R, C] out
  uint8_t* mask;             // [R, C] out
  const int64_t* out_perm;
  float* losses;
  float* err; float* err_hi; float* err_lo;
};

// A row is spread over 16 lanes (16 rows per CTA, 256 threads, two CTAs per SM; one thread per row
// would give R = 4096 only 32 CTAs, one warp per scheduler): lane j evaluates the leave-one-out
// cases j, j + 16, ... of a group, every lane recomputes the cheap group statistics, and after the
// (redundant) quantise -> err step of a column each lane applies the rank-1 update to the later
// columns it owns.  The three phases are spqr::lanes_* of spqr_row.cuh, which the CPU tests run on
// the host in lock step against the oracle.  Lanes talk through the row's shared-memory storage,
// with __syncwarp() between phases.
constexpr int SL = 16;            // lanes per row
constexpr int SR = 16;            // rows per CTA
constexpr int SWP = GB + 16;      // pitch of a W row: the two rows of a warp sit 16 banks apart
constexpr int SHP = GB + 4;       // pitch of the row-major Hinv block
constexpr int SEP = SR + 1;       // pitch of the transposed err tile
constexpr int kSpqrSmem = (SR * SWP + GB * SHP + GB * SEP) * 4 + 2 * SR * GB;

__global__ void __launch_bounds__(SR * SL, 2)
spqr_inblock_kernel(SpqrArgs a) {
  extern __shared__ float sm[];
  float* Ws = sm;                        // [row][col]   current (in place updated) weights
  float* Hs = Ws + SR * SWP;             // [i][j]       Hinv1, upper triangle
  float* Et = Hs + GB * SHP;             // [col][row]   Err1 transposed
  uint8_t* Ms = reinterpret_cast<uint8_t*>(Et + GB * SEP);   // [row][col] outlier mask
  uint8_t* Fl = Ms + SR * GB;                                // [row][k]   leave-one-out flags of the group
  const int tid = threadIdx.x, rr = tid / SL, lane = tid % SL;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * SR;
  const int64_t row = r0 + rr;
  const int cnt = a.count;
  for (int idx = tid; idx < SR * GB; idx += SR * SL) {
    const int r = idx >> 7, c = idx & 127;
    float v = 0.f;
    if (r0 + r < a.R && c < cnt) v = a.W[(r0 + r) * a.C + a.i1 + c];
    Ws[r * SWP + c] = v;
    Ms[idx] = 0;
    Fl[idx] = 0;
  }
  for (int idx = tid; idx < GB * GB; idx += SR * SL) {
    const int i = idx >> 7, j = idx & 127;
    float v = (i == j) ? 1.f : 0.f;
    if (i < cnt && j < cnt && j >= i) v = a.Hinv[(static_cast<int64_t>(a.i1) + i) * a.C + a.i1 + j];
    Hs[i * SHP + j] = v;
  }
  for (int idx = tid; idx < GB * SEP; idx += SR * SL) Et[idx] = 0.f;
  __syncthreads();
  const bool live = row < a.R;
  spqr::Cfg cfg = a.cfg;
  cfg.thr = a.thr[0];
  cfg.has_thr = !isinf(cfg.thr);
  cfg.outliers = (!a.simplified && cfg.has_thr) ? 1 : 0;
  float* w = Ws + rr * SWP;
  uint8_t* fl = Fl + rr * GB;
  float loss = 0.f, s = 1.f, z = 0.f;
  for (int col = 0; col < cnt; ++col) {
    if (col % cfg.gs == 0) {
      if (live) spqr::lanes_group_flags(w + col, 1, Hs + col * SHP + col, SHP + 1, cfg, lane, SL, fl);
      __syncwarp();
      if (live) {
        spqr::lanes_group_qparams(w + col, 1, fl, cfg, s, z);
        if (lane == 0) {
          const int64_t gi = (static_cast<int64_t>(a.i1) + col) / cfg.gs;
          a.scales[row * a.ng + gi] = s;
          a.zeros[row * a.ng + gi] = z;
        }
      }
      __syncwarp();
    }
    float err = 0.f;
    uint8_t m = 0;
    if (live) err = spqr::lanes_column(w, 1, Hs, SHP, 1, cnt, col, s, z, cfg, lane, SL, m);
    if (live && lane == 0) {
      Et[col * SEP + rr] = err;
      Ms[rr * GB + col] = m;
      loss = add(loss, mul(err, err));
    }
    __syncwarp();
  }
  if (live && lane == 0) a.losses[row] += loss;
  __syncthreads();
  for (int idx = tid; idx < SR * GB; idx += SR * SL) {
    const int r = idx >> 7, c = idx & 127;
    if (r0 + r < a.R && c < cnt) {
      const int64_t oc = a.out_perm ? a.out_perm[a.i1 + c] : static_cast<int64_t>(a.i1) + c;
      a.tmp[(r0 + r) * a.C + oc] = Ws[r * SWP + c];
      a.mask[(r0 + r) * a.C + oc] = Ms[idx];
    }
  }
  for (int idx = tid; idx < GB * SR; idx += SR * SL) {
    const int c = idx / SR, r = idx % SR;
    const float ev = (c < cnt) ? Et[c * SEP + r] : 0.f;
    const int64_t o = static_cast<int64_t>(c) * a.Rpad + r0 + r;
    a.err[o] = ev;
    uint32_t hb, lb;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(ev));
    const float h = __uint_as_float(hb);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(ev - h));
    a.err_hi[o] = h;
    a.err_lo[o] = __uint_as_float(lb);
  }
}

// ---- trailing update: W[:, n0:] -= Err[R,128] @ Hinv[i1:i1+128, n0:] ---------------------------------------
// fp32 SIMT GEMM, 128x128 tile, 8x8 per thread, K = 128 resident in shared memory.
constexpr int TT = 128;
constexpr int kTrailingSmem = 2 * TT * TT * 4;   // 131,072 B
__global__ void __launch_bounds__(256, 1)
trailing_update_kernel(float* __restrict__ W, int64_t R, int64_t Rpad, int64_t C, const float* __restrict__ Err,
                       const float* __restrict__ Hinv, int i1, int kcount, int64_t n0) {
  extern __shared__ float sm[];
  float* As = sm;               // [k][m]  (Err transposed), 128 x 128
  float* Bs = sm + TT * TT;     // [k][n]
  const int tid = threadIdx.x;
  const int64_t m0 = static_cast<int64_t>(blockIdx.y) * TT;
  const int64_t nb0 = n0 + static_cast<int64_t>(blockIdx.x) * TT;
  // load A: ErrT[k][Rpad] (k-major) -> As[k][m], unit stride both sides (Rpad % 128 == 0)
  for (int idx = tid; idx < TT * TT / 4; idx += 256) {
    const int k = idx >> 5;            // 32 float4 per k row
    const int m4 = (idx & 31) << 2;
    *reinterpret_cast<float4*>(&As[k * TT + m4]) =
        *reinterpret_cast<const float4*>(&Err[static_cast<int64_t>(k) * Rpad + m0 + m4]);
  }
  // load B: Hinv rows i1..i1+kcount-1, cols nb0..nb0+127
  for (int idx = tid; idx < TT * TT; idx += 256) {
    const int k = idx >> 7, n = idx & 127;
    float v = 0.f;
    if (k < kcount && nb0 + n < C) v = Hinv[(static_cast<int64_t>(i1) + k) * C + nb0 + n];
    Bs[k * TT + n] = v;
  }
  __syncthreads();
  const int tx = tid & 15, ty = tid >> 4;       // 16 x 16 threads; thread tile 8 x 8
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
#pragma unroll 4
  for (int k = 0; k < TT; ++k) {
    const float4 a0 = *reinterpret_cast<const float4*>(&As[k * TT + ty * 4]);
    const float4 a1 = *reinterpret_cast<const float4*>(&As[k * TT + 64 + ty * 4]);
    const float4 b0 = *reinterpret_cast<const float4*>(&Bs[k * TT + tx * 4]);
    const float4 b1 = *reinterpret_cast<const float4*>(&Bs[k * TT + 64 + tx * 4]);
    const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= R) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int64_t n = nb0 + jh * 64 + tx * 4;
      float* wp = &W[m * C + n];
      if (n + 3 < C && ((reinterpret_cast<uintptr_t>(wp) & 15) == 0)) {
        float4 v = *reinterpret_cast<float4*>(wp);
        v.x -= acc[i][jh * 4 + 0]; v.y -= acc[i][jh * 4 + 1];
        v.z -= acc[i][jh * 4 + 2]; v.w -= acc[i][jh * 4 + 3];
        *reinterpret_cast<float4*>(wp) = v;
      } else {
        for (int j = 0; j < 4; ++j)
          if (n + j < C) wp[j] -= acc[i][jh * 4 + j];
      }
    }
  }
}

}  // namespace llmc

using namespace llmc;

extern "C" int llmc_gptq_prepare(const float* H, int64_t C, const int64_t* perm, float percdamp,
                                 float* Hp, const void* W, int64_t R, int w_dtype, float* Wp,
                                 float* diag_scratch, void* stream) {
  // Hp == NULL skips the Hessian gather, W == NULL the weight gather (linears that share one
  // Hessian need Hp once and one Wp each)
  LLMC_CHECK_ARG(H && (Hp || W) && (!W || (Wp && R > 0)) && diag_scratch && C > 0, "gptq_prepare: bad argument");
  LLMC_CHECK_ARG(C * 4 <= 200 * 1024, "gptq_prepare: C=%lld exceeds the shared-memory row buffer",
                 (long long)C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int smem = static_cast<int>(C * 4);
  LLMC_ONCE_PER_DEVICE({
    LLMC_CHECK_CUDA(cudaFuncSetAttribute(gather_h_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    LLMC_CHECK_CUDA(cudaFuncSetAttribute(gather_w_kernel<LLMC_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    LLMC_CHECK_CUDA(cudaFuncSetAttribute(gather_w_kernel<LLMC_F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    LLMC_CHECK_CUDA(cudaFuncSetAttribute(gather_w_kernel<LLMC_BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  });
  diag_mean_kernel<<<1, 256, 0, st>>>(H, C, percdamp, diag_scratch);
  LLMC_CHECK_LAUNCH();
  // W first: it reads the ORIGINAL diagonal of H (dead test), Hp may alias neither H nor W
  if (W != nullptr) {
#define CALL(DT) gather_w_kernel<DT><<<(unsigned)R, 256, smem, st>>>(W, R, C, H, perm, Wp)
    LLMC_DISPATCH_DT("gptq_prepare", w_dtype, CALL);
#undef CALL
    LLMC_CHECK_LAUNCH();
  }
  if (Hp != nullptr) {
    gather_h_kernel<<<(unsigned)C, 256, smem, st>>>(H, C, perm, diag_scratch, Hp);
    LLMC_CHECK_LAUNCH();
  }
  return LLMC_OK;
}

// The schedule shared by the GPTQ and SpQR sweeps: in-block kernel per 128 columns (launched by
// `launch_inblock(i1, count, err, err_hi, err_lo, stream)`), lazy trailing updates per super-panel
// and the look-ahead split of the bulk update.  `wide_dynamic_group`: the in-block kernel reads
// columns beyond its super-panel (a dynamic group wider than 512), which the look-ahead cannot
// order.
template <class F>
static int sweep_schedule(float* W, const float* Hinv, int64_t R, int64_t C, int64_t group,
                          bool wide_dynamic_group, void* workspace, cudaStream_t st, F&& launch_inblock) {
  LLMC_ONCE_PER_DEVICE({
    LLMC_CHECK_CUDA(cudaFuncSetAttribute(trailing_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTrailingSmem));
  });
  const int64_t Rpad = ((R + GB - 1) / GB) * GB;
  // [512][Rpad] x {err, hi, lo}, two sets selected by the parity of the super-panel
  float* const err_set[2] = {reinterpret_cast<float*>(workspace),
                             reinterpret_cast<float*>(workspace) + 3 * kSuperPanel * Rpad};
  float* Hh = err_set[1] + 3 * kSuperPanel * Rpad;
  float* Hl = Hh + C * C;
  const SplitMatrix Hs{Hh, Hl, C};    // tf32 split of Hinv
  // trailing updates on tensor cores (3xTF32) when the shapes allow TMA; fp32 SIMT otherwise.
  // LLMC_B200_SIMT_TRAILING=1 forces the fp32 CUDA-core kernel everywhere: a second summation
  // order for scripts/check_spqr_summation_order.py, whose measurements PARITY.md records.
  static const bool force_simt = getenv("LLMC_B200_SIMT_TRAILING") != nullptr;
  const bool tensor_trailing = !force_simt && (C % 8 == 0) && aligned16(W) && aligned16(Hinv) &&
                               aligned16(workspace);
  if (tensor_trailing && C > GB) {
    if (int rc = split_tf32(Hinv, C, C, C, Hh, Hl, C, st)) return rc;
  }
  // super-panel width: 512 on the tensor path, one block (the reference's schedule) otherwise
  // (a dynamic group is searched on W[:, start : start+group] at its first column, so a group
  // must never reach past the super-panel it starts in unless it starts with it)
  const bool groups_fit = group <= GB || kSuperPanel % group == 0 || group % kSuperPanel == 0;
  const int64_t sp_width = (tensor_trailing && groups_fit) ? kSuperPanel : GB;
  // ---- look-ahead schedule ------------------------------------------------------------------
  // The sweep's dependent chain is  in-block kernel -> in-panel update -> next in-block kernel;
  // the rank-512 update of everything beyond a super-panel is a large share of the sweep's work
  // at R >= 4096 and is NOT on that chain beyond the next 512 columns.  So at a
  // super-panel boundary the chain (high-priority stream) updates the next super-panel's columns
  // only, and the rest goes to a low-priority stream, one tile per CTA, overlapping the next
  // panel's chain.  Every column receives its panel updates in the same order as before (events),
  // and a 3xTF32 tile's value does not depend on how the N range is cut, so results are
  // bit-identical to the serial schedule (LLMC_B200_SWEEP_LOOKAHEAD=0 selects it).
  const char* la_env = getenv("LLMC_B200_SWEEP_LOOKAHEAD");      // read per call: tests toggle it
  const bool la_off = la_env != nullptr && la_env[0] == '0';
  // (a dynamic group wider than a super-panel is searched on columns a bulk piece may still be
  //  updating: those sweeps keep the serial schedule)
  const bool lookahead = !la_off && tensor_trailing && sp_width == kSuperPanel && C > 2 * kSuperPanel &&
                         !wide_dynamic_group;
  cudaStream_t chain = st, bulk = st;
  SideStreams* side = nullptr;
  cudaEvent_t* panel_done = nullptr;   // per parity: the panel's errors are complete (chain)
  cudaEvent_t* bulk_done = nullptr;    // per parity: the panel's bulk update is done (bulk)
  if (lookahead) {
    if (int rc = side_streams(2, &side)) return rc;
    chain = side->stream[kChain];
    bulk = side->stream[kBulk];
    panel_done = side->ev[0].data();
    bulk_done = side->ev[1].data();
    if (int rc = side->fork(st, {kChain})) return rc;
  }
  bool bulk_pending[2] = {false, false};        // a bulk update of that parity has been enqueued
  for (int64_t i1 = 0; i1 < C; i1 += GB) {
    const int64_t i2 = (i1 + GB < C) ? i1 + GB : C;
    const int64_t sp0 = (i1 / sp_width) * sp_width;
    const int64_t sp1 = (sp0 + sp_width < C) ? sp0 + sp_width : C;
    const int par = static_cast<int>((i1 / sp_width) & 1);
    float* err_base = err_set[par];
    // the tf32 split of the super-panel's errors, row j - sp0 for column j
    const SplitMatrix E{err_base + kSuperPanel * Rpad, err_base + 2 * kSuperPanel * Rpad, Rpad};
    const int b_i1 = static_cast<int>(i1);
    const int b_count = static_cast<int>(i2 - i1);
    float* const b_err = err_base + (i1 - sp0) * Rpad;
    if (int rc = launch_inblock(b_i1, b_count, b_err, E.hi + (i1 - sp0) * Rpad, E.lo + (i1 - sp0) * Rpad, chain))
      return rc;
    // W[:, n0:n1] -= Err1[:, k0:k1] @ Hinv[k0:k1, n0:n1]   (gptq.py:244) for columns k0..k1 of this
    // super-panel: A = Err1^T (MN-major, ld Rpad), B = Hinv rows (MN-major, ld C)
    auto trailing = [&](int64_t k0, int64_t k1, int64_t n0, int64_t n1) {
      return Tf32x3Update{E.at_mn(k0 - sp0, 0), Hs.at_mn(k0, n0), W + n0, C, R, n1 - n0, k1 - k0};
    };
    if (i2 < C && tensor_trailing) {
      // Inside the super-panel: this block's errors onto the super-panel's remaining columns; at its
      // end: all of its errors onto everything beyond.
      if (i2 < sp1) {
        if (int rc = tf32x3_update(trailing(i1, i2, i2, sp1), chain)) return rc;
      } else if (!lookahead) {
        if (int rc = tf32x3_update(trailing(sp0, sp1, sp1, C), chain)) return rc;
      } else {
        const int64_t nx1 = (sp1 + sp_width < C) ? sp1 + sp_width : C;
        // the errors of this panel are complete: the bulk piece may start (after the previous one)
        LLMC_CHECK_CUDA(cudaEventRecord(panel_done[par], chain));
        // chain: the next super-panel's columns, last written by the previous panel's bulk piece
        if (bulk_pending[par ^ 1]) LLMC_CHECK_CUDA(cudaStreamWaitEvent(chain, bulk_done[par ^ 1], 0));
        if (int rc = tf32x3_update(trailing(sp0, sp1, sp1, nx1), chain)) return rc;
        // bulk: everything beyond.  After this wait the chain goes on to write the OTHER error set,
        // which the previous bulk piece (just waited for) was the last reader of.
        if (nx1 < C) {
          LLMC_CHECK_CUDA(cudaStreamWaitEvent(bulk, panel_done[par], 0));
          if (int rc = tf32x3_update(trailing(sp0, sp1, nx1, C).tile_per_cta(), bulk)) return rc;
          LLMC_CHECK_CUDA(cudaEventRecord(bulk_done[par], bulk));
          bulk_pending[par] = true;
        }
      }
    } else if (i2 < C) {
      dim3 grid(static_cast<unsigned>((C - i2 + TT - 1) / TT), static_cast<unsigned>((R + TT - 1) / TT));
      trailing_update_kernel<<<grid, 256, kTrailingSmem, chain>>>(W, R, Rpad, C, b_err, Hinv, b_i1, b_count, i2);
      LLMC_CHECK_LAUNCH();
    }
  }
  if (lookahead) {
    if (int rc = side->join(st, {kChain, kBulk})) return rc;
  }
  return LLMC_OK;
}

extern "C" int64_t llmc_gptq_workspace_bytes(int64_t R, int64_t C) {
  // Err1^T + its tf32 split for TWO super-panels ([512, Rpad] x 3 each: the bulk trailing update
  // of panel p reads its errors while the chain of panel p+1 writes the other set) and the tf32
  // split of Hinv ([C, C] x 2)
  const int64_t rpad = ((R + GB - 1) / GB) * GB;
  return (6 * kSuperPanel * rpad + 2 * C * C) * 4;
}

extern "C" int llmc_gptq_colblock(float* W, const float* Hinv, int64_t R, int64_t C, int64_t group,
                                  int bit, int sym, int static_groups, const int32_t* gmap,
                                  void* scales, void* zeros, int q_dtype, float* tmp,
                                  const int64_t* out_perm, float* losses, void* workspace,
                                  int64_t workspace_bytes, void* stream) {
  LLMC_CHECK_ARG(W && Hinv && tmp && losses && workspace && R > 0 && C > 0, "gptq_colblock: bad argument");
  LLMC_CHECK_ARG(bit >= 2 && bit <= 8, "gptq_colblock: bit %d outside 2..8", bit);
  LLMC_CHECK_ARG(group > 0 && group <= C && C % group == 0, "gptq_colblock: C=%lld %% group=%lld != 0",
                 (long long)C, (long long)group);
  LLMC_CHECK_ARG((group >= C) || (group >= GB ? group % GB == 0 : (GB % group == 0 && GB / group <= 8)),
                 "gptq_colblock: group %lld must divide or be a multiple of the block size 128 "
                 "(and be >= 16)", (long long)group);
  LLMC_CHECK_ARG(scales, "gptq_colblock: scales is NULL");
  LLMC_CHECK_ARG(sym || zeros, "gptq_colblock: zeros is NULL for asymmetric quantisation");
  LLMC_CHECK_ARG(static_groups || q_dtype == LLMC_F32, "gptq_colblock: dynamic groups write fp32 qparams");
  LLMC_CHECK_ARG(workspace_bytes >= llmc_gptq_workspace_bytes(R, C), "gptq_colblock: workspace too small");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LLMC_ONCE_PER_DEVICE({
    LLMC_CHECK_CUDA(cudaFuncSetAttribute(gptq_inblock_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kInblockSmem));
  });
  LLMC_CHECK_CUDA(cudaMemsetAsync(losses, 0, R * sizeof(float), st));
  InblockArgs a{};
  a.W = W; a.Hinv = Hinv; a.R = R; a.C = C;
  a.group = group; a.ng = C / group; a.sym = sym;
  int_range(bit, sym, a.qmin, a.qmax);
  a.static_groups = static_groups; a.gmap = gmap;
  a.scales = scales; a.zeros = sym ? nullptr : zeros; a.q_dtype = q_dtype;
  a.tmp = tmp; a.out_perm = out_perm; a.losses = losses;
  a.Rpad = ((R + GB - 1) / GB) * GB;
  const bool wide = !static_groups && group > kSuperPanel;
  return sweep_schedule(W, Hinv, R, C, group, wide, workspace, st,
                        [&](int i1, int count, float* err, float* err_hi, float* err_lo, cudaStream_t cs) -> int {
    a.i1 = i1; a.count = count; a.err = err; a.err_hi = err_hi; a.err_lo = err_lo;
    gptq_inblock_kernel<<<static_cast<unsigned>(a.Rpad / IR), IR * IL, kInblockSmem, cs>>>(a);
    LLMC_CHECK_LAUNCH();
    return LLMC_OK;
  });
}

static spqr::QCfg spqr_qcfg(int bit, int sym, int round_zp) {
  spqr::QCfg q{};
  int_range(bit, sym, q.qmin, q.qmax);
  q.sym = sym; q.round_zp = round_zp;
  return q;
}

extern "C" int llmc_spqr_colblock(float* W, const float* Hinv, int64_t R, int64_t C, int64_t group,
                                  int bit, int sym, int round_zp, int s_bit, int s_sym, int s_round_zp,
                                  int z_bit, int z_sym, int z_round_zp, const float* threshold,
                                  int simplified_outliers, float* scales, float* zeros, float* tmp,
                                  uint8_t* mask, const int64_t* out_perm, float* losses, void* workspace,
                                  int64_t workspace_bytes, void* stream) {
  LLMC_CHECK_ARG(W && Hinv && tmp && mask && losses && workspace && threshold && scales && zeros && R > 0 && C > 0,
                 "spqr_colblock: bad argument");
  LLMC_CHECK_ARG(bit >= 2 && bit <= 8 && s_bit >= 2 && s_bit <= 8 && z_bit >= 2 && z_bit <= 8,
                 "spqr_colblock: bit widths outside 2..8");
  LLMC_CHECK_ARG(!sym, "spqr_colblock: symmetric weights (the reference fails on them, spqr.py:334)");
  LLMC_CHECK_ARG((group == 16 || group == 32 || group == 64 || group == 128) && C % group == 0,
                 "spqr_colblock: group %lld must be 16, 32, 64 or 128 and divide C=%lld",
                 (long long)group, (long long)C);
  LLMC_CHECK_ARG(workspace_bytes >= llmc_gptq_workspace_bytes(R, C), "spqr_colblock: workspace too small");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LLMC_ONCE_PER_DEVICE({
    LLMC_CHECK_CUDA(cudaFuncSetAttribute(spqr_inblock_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSpqrSmem));
  });
  LLMC_CHECK_CUDA(cudaMemsetAsync(losses, 0, R * sizeof(float), st));
  SpqrArgs a{};
  a.W = W; a.Hinv = Hinv; a.R = R; a.C = C; a.ng = C / group;
  a.cfg.w = spqr_qcfg(bit, sym, round_zp);
  a.cfg.loo = spqr_qcfg(bit, sym, 0);                   // spqr.py:56-58
  a.cfg.sc = spqr_qcfg(s_bit, s_sym, s_round_zp);
  a.cfg.zc = spqr_qcfg(z_bit, z_sym, z_round_zp);
  a.cfg.gs = static_cast<int>(group);
  a.thr = threshold; a.simplified = simplified_outliers;
  a.scales = scales; a.zeros = zeros; a.tmp = tmp; a.mask = mask; a.out_perm = out_perm; a.losses = losses;
  a.Rpad = ((R + GB - 1) / GB) * GB;
  return sweep_schedule(W, Hinv, R, C, group, false, workspace, st,
                        [&](int i1, int count, float* err, float* err_hi, float* err_lo, cudaStream_t cs) -> int {
    a.i1 = i1; a.count = count; a.err = err; a.err_hi = err_hi; a.err_lo = err_lo;
    spqr_inblock_kernel<<<static_cast<unsigned>(a.Rpad / SR), SR * SL, kSpqrSmem, cs>>>(a);
    LLMC_CHECK_LAUNCH();
    return LLMC_OK;
  });
}
