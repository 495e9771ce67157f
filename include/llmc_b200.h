/*
 * llmc_b200.h — C ABI of libllmc_b200.so: the H100 (sm_90a) kernels behind llmc's
 * weight-quantization hot path (SURVEY.md §8).
 *
 * The reference (ModelTC/llmc) has no FFI: its plug-in boundary is the Python object
 * protocol of `llmc/compression/quantization/{quant,module_utils,gptq,awq,auto_clip}.py`.
 * Each entry point below names the reference function (file:line, relative to the llmc
 * tree) whose arithmetic it replaces; `llmc_b200/*.py` mirrors the reference classes and
 * calls these through ctypes (see INTEGRATION.md for the binding a maintainer would add).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to caller-owned, contiguous memory (16-byte aligned
 *     base); nothing is allocated, nothing is retained after return;
 *   - every call is asynchronous on `stream` (a cudaStream_t / CUstream handle passed as
 *     void*; NULL = legacy default stream) and never synchronises the host;
 *   - return value: 0 on success, a negative LLMC_E* code otherwise
 *     (llmc_b200_error_string() explains it, llmc_b200_last_error() adds detail);
 *   - dtype enums: LLMC_F32 / LLMC_F16 / LLMC_BF16.  "T-faithful" below means: computed
 *     like torch eager does for a tensor of dtype T — every elementwise op is evaluated in
 *     fp32 and rounded once to T (SURVEY.md Appendix A.1), division is IEEE, rounding is
 *     half-to-even.
 */
#ifndef LLMC_B200_H_
#define LLMC_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LLMC_B200_ABI_VERSION 2

/* dtypes */
enum { LLMC_F32 = 0, LLMC_F16 = 1, LLMC_BF16 = 2 };

/* error codes */
enum {
  LLMC_OK = 0,
  LLMC_EINVAL = -1,      /* bad argument (shape / enum / null pointer)            */
  LLMC_EUNSUPPORTED = -2, /* valid request this build has no kernel for            */
  LLMC_ECUDA = -3,       /* a CUDA runtime / driver call failed (see last_error)  */
  LLMC_EALIGN = -4       /* pointer or leading dimension not suitably aligned     */
};

/* output selector of the quantize kernels */
enum {
  LLMC_OUT_NONE = 0,      /* qparams only                                                      */
  LLMC_OUT_QDQ = 1,       /* fake-quant: dequantised values, dtype = out_dtype                 */
  LLMC_OUT_CODES_I8 = 2,  /* integer codes as int8  (8-bit symmetric; quant.py:890-897)        */
  LLMC_OUT_CODES_U8 = 3,  /* integer codes as uint8 (8-bit asymmetric)                         */
  LLMC_OUT_CODES_I32 = 4, /* one code per int32 (every other bit-width; quant.py:895-896)      */
  LLMC_OUT_PACK_VLLM = 5  /* (code + 2^(bit-1)) packed 32/bit per int32 along the input
                             dimension, element i in bits [bit*i, bit*i+bit), zero padded
                             (VllmRealQuantLinear.pack, module_utils.py:836-862)               */
};
/* OR-ed into out_mode of llmc_quant_static: `round_zp: False` (quant.py:702-707, HQQ's real-valued
 * zero-points): q = clamp(round(x / max(s, 1e-9) + z), qmin, qmax) — the zero-point is added BEFORE
 * the rounding. */
#define LLMC_OUT_FLAG_ZP_INSIDE 0x100

int llmc_b200_abi_version(void);
const char* llmc_b200_error_string(int code);
/* thread-local detail of the most recent failure on the calling thread ("" if none) */
const char* llmc_b200_last_error(void);
/* number of CUDA kernels this library has launched in this process (monotonic) */
long long llmc_b200_launch_count(void);

/* ------------------------------------------------------------------------------------
 * K1+K2  llmc_quant_dynamic — replaces IntegerQuantizer.get_tensor_qparams (quant.py:690-697
 *   = reshape_tensor :612-642 -> get_minmax_range :132-143 -> get_qparams :545-559) followed by
 *   quant :699-708 / dequant :710-712, i.e. fake_quant_weight_dynamic :833-869 (out_mode QDQ),
 *   real_quant_weight_dynamic :916-953 (CODES_*), and VllmRealQuantLinear.pack (PACK_VLLM).
 *
 *   w        [rows, cols] dtype `dtype`, row stride `ld` elements (ld >= cols)
 *   group    elements per quantisation group along a row: group_size (per_group),
 *            cols (per_channel / per_token); cols % group == 0
 *   bit      2..8 ; sym != 0: qmin=-2^(bit-1), qmax=2^(bit-1)-1, zero = 0
 *                    sym == 0: qmin=0, qmax=2^bit-1, zero = clamp(qmin - round(min/scale))
 *   qmin,qmax  override the range when qmin < qmax is given with use_range != 0 (int_range)
 *   col_scale  optional [cols] dtype `dtype`: quantise rT(w * col_scale[c]) instead of w — AWQ's
 *            fake_quantize_weight (awq.py:39-46, 147-164) without touching the weights
 *   scales   [rows * cols/group] dtype `dtype`  (index r*ng + j == the reference's [R*ng,1])
 *   zeros    same shape/dtype, written only when sym == 0 (may be NULL when sym != 0)
 *   out      per out_mode (QDQ: [rows, cols] out_dtype, row stride ld_out;
 *            CODES_*: [rows, cols] dense; PACK_VLLM: [rows, ceil(cols*bit/32)] int32 dense)
 *   All arithmetic is `dtype`-faithful.
 * ------------------------------------------------------------------------------------ */
int llmc_quant_dynamic(const void* w, int64_t rows, int64_t cols, int64_t ld, int dtype,
                       int64_t group, int bit, int sym, int use_range, int qmin, int qmax,
                       const void* col_scale, void* scales, void* zeros, int out_mode, void* out,
                       int64_t ld_out, int out_dtype, void* stream);

/* ------------------------------------------------------------------------------------
 * K2  llmc_quant_static — replaces fake_quant_weight_static (quant.py:785-831),
 *   real_quant_weight_static (:871-914) and GPTQ.w_qdq / w_q (gptq.py:411-452) incl. the
 *   act-order gather `W[:, perm] -> qdq -> [:, invperm]`.
 *
 *   element (r, c) uses qparams[r * q_row_stride + g(c)], g(c) = gmap ? gmap[c] : c / group
 *   (q_row_stride = groups per row; 0 with group = cols selects per_tensor qparams).
 *   (for gptq.py:427-450 pass gmap[c] = invperm[c] / group)
 *   w dtype `w_dtype`; scales/zeros dtype `q_dtype`; arithmetic is faithful to
 *   promote(w_dtype, q_dtype) exactly like torch type promotion (round_dtype = -1), or to
 *   round_dtype = w_dtype with fp32 qparams: torch's CPU path for a 0-dim (per_tensor) scale,
 *   which keeps the scalar in fp32 and rounds every result to the tensor dtype
 *   (ATen BinaryOpsKernel.cpp, scalar-operand branch of div/mul).  zeros may be NULL (= 0).
 *   qmin/qmax: the clamp range.  out as in llmc_quant_dynamic (QDQ written as out_dtype).
 * ------------------------------------------------------------------------------------ */
int llmc_quant_static(const void* w, int64_t rows, int64_t cols, int64_t ld, int w_dtype,
                      const void* scales, const void* zeros, int q_dtype, int round_dtype,
                      int64_t q_row_stride, int64_t group, const int32_t* gmap, int bit,
                      int qmin, int qmax, int out_mode, void* out, int64_t ld_out,
                      int out_dtype, void* stream);

/* ------------------------------------------------------------------------------------
 * llmc_pack_vllm_codes — VllmRealQuantLinear.pack (module_utils.py:836-862) on codes that
 *   are already quantised: codes [rows, cols] int8 (code_bytes 1) or int32 (code_bytes 4)
 *   -> out [rows, ceil(cols / (32/bit))] int32.
 * ------------------------------------------------------------------------------------ */
int llmc_pack_vllm_codes(const void* codes, int code_bytes, int64_t rows, int64_t cols,
                         int bit, int32_t* out, void* stream);

/* ------------------------------------------------------------------------------------
 * llmc_minmax_tensor — per_tensor range (quant.py:133-135): min and max over the whole
 *   tensor written to mm[0], mm[1] (dtype `dtype`).  Two-stage device reduction,
 *   `workspace` >= 2 * 1024 floats.
 * ------------------------------------------------------------------------------------ */
int llmc_minmax_tensor(const void* w, int64_t n, int dtype, void* mm, float* workspace,
                       void* stream);

/* ------------------------------------------------------------------------------------
 * Range search / observers (csrc/range.cu)
 *   llmc_mse_range — `calib_algo: mse`, BaseQuantizer.get_mse_range (quant.py:145-203) on the
 *     reshaped tensor [rows = groups, cols = group elements] (any dtype, evaluated in fp32 like
 *     `tensor.float()`): for i in 0..steps-1 (steps = int(maxshrink * mse_grid), p = 1 - i/grid)
 *     the range (p*min, p*max) is tried with get_qparams (:545-559) + quant_dequant (:699-717) and
 *     the one with the smallest sum |q - x|^norm (norm = 2.4) per row is kept; min_out / max_out
 *     [rows] fp32.  The reference's aliasing of the running range (:165, an improvement shrinks
 *     the base of all later levels) is reproduced.
 *   llmc_histc — torch.histc(x.float(), bins, min=lo, max=hi) for the static histogram observer
 *     (get_static_hist_range, quant.py:462-522): hist [bins] fp32 counts, each the exact count
 *     rounded once (deterministic beyond 2^24 per bin); n < 2^32.
 * ------------------------------------------------------------------------------------ */
int llmc_mse_range(const void* w, int64_t rows, int64_t cols, int dtype, int sym, int qmin,
                   int qmax, int steps, float grid, float norm, float* min_out, float* max_out,
                   void* stream);
int llmc_histc(const void* x, int64_t n, int dtype, int bins, float lo, float hi, float* hist,
               void* stream);

/* ------------------------------------------------------------------------------------
 * K2-awq  llmc_pack_awq — replaces AutoawqRealQuantLinear.gemm_pack (module_utils.py:1004-1065).
 *   w       [R, C] fp16/bf16/fp32 (the module weight)
 *   scales  [R, ng] dtype `dtype`, zeros [R, ng] int32 (as returned by real_quant_weight_*)
 *   intweight(r,c) = round((w + rT(z*s)) / s) computed in `dtype` exactly like :1022-1029
 *   (scales are first cast to fp16, :1008), NOT clamped;
 *   qweight [C, R/8] int32: nibble i of word (c, r8) = intweight(r8*8 + order[i], c),
 *   order = {0,2,4,6,1,3,5,7}; qzeros [ng, R/8] packed the same way; scales_out [ng, R] fp16.
 *   Requires bit == 4, R % 32 == 0.
 * ------------------------------------------------------------------------------------ */
int llmc_pack_awq(const void* w, int64_t R, int64_t C, int dtype, const void* scales,
                  int s_dtype, const int32_t* zeros, int64_t group, int32_t* qweight,
                  int32_t* qzeros, void* scales_out_f16, void* stream);

/* ------------------------------------------------------------------------------------
 * K3  llmc_syrk_accum — replaces GPTQ.add_batch's Hessian update (gptq.py:283-290):
 *       H <- H * n/(n+b) + (2/(n+b)) * X^T X          (fp32 H, bf16/fp16 X)
 *   x   [T, C] row-major activations (tokens x in_features), dtype bf16 or fp16
 *   H   [C, C] fp32, full symmetric matrix on return (upper computed on wgmma tensor
 *       cores with fp32 register accumulation, mirrored into the lower triangle)
 *   n   samples accumulated so far, b = samples in this call (inp.shape[0], :258)
 *   workspace: split-K partials, >= llmc_syrk_workspace_bytes(T, C) bytes
 * ------------------------------------------------------------------------------------ */
int64_t llmc_syrk_workspace_bytes(int64_t T, int64_t C);
int llmc_syrk_accum(const void* x, int64_t T, int64_t C, int dtype, float* H, double n,
                    double b, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------
 * Multi-GPU helpers (csrc/comm.cu) — the reference all-reduces the FULL Hessian after every
 *   hooked batch (gptq.py:292-295); H is symmetric, so only its upper triangle needs to cross
 *   NVLink, once per distinct input:
 *   llmc_tri_pack    packed[i*C - i(i-1)/2 + (j-i)] = H[i][j], j >= i   (llmc_tri_elems(C) floats)
 *   llmc_tri_unpack  H[i][j] = H[j][i] = packed[...] * scale            (scale = 1/world: the mean)
 * ------------------------------------------------------------------------------------ */
int64_t llmc_tri_elems(int64_t C);
int llmc_tri_pack(const float* H, int64_t C, float* packed, void* stream);
int llmc_tri_unpack(const float* packed, int64_t C, float scale, float* H, void* stream);

/* ------------------------------------------------------------------------------------
 * G4 helpers  llmc_gptq_prepare — replaces process_hessian_and_weights (gptq.py:128-171)
 *   up to (not including) the Cholesky triple: dead-column fix, act-order gather of W and H,
 *   damping.  perm NULL = identity.
 *     Hp[i,j] = H[perm[i], perm[j]] (+ percdamp*mean(diag) on the diagonal; dead -> 1)
 *     Wp[r,j] = dead[perm[j]] ? 0 : float(W[r, perm[j]])
 *   diag_mean_out: device float[1] scratch.
 *   Hp == NULL skips the Hessian part, W == NULL the weight part: linears that share one input
 *   (q/k/v, gate/up) need Hp once and one Wp each — written into row slices of ONE buffer, they
 *   are then swept by a single llmc_gptq_colblock call (rows are independent given Hinv).
 * ------------------------------------------------------------------------------------ */
int llmc_gptq_prepare(const float* H, int64_t C, const int64_t* perm, float percdamp,
                      float* Hp, const void* W, int64_t R, int w_dtype, float* Wp,
                      float* diag_scratch, void* stream);

/* ------------------------------------------------------------------------------------
 * K4  llmc_chol_inv_upper — replaces the Cholesky triple (gptq.py:172-174):
 *       U = cholesky( cholesky_inverse( cholesky(H) ), upper )
 *   computed as U = R^-1 where H = R R^T, R upper triangular (one reverse-ordered
 *   factorisation + one triangular inverse instead of potrf + potri + potrf; DESIGN.md).
 *   A  [C, C] fp32 in: SPD H; only its upper triangle (diagonal included) is read;
 *                 out: U in the upper triangle, zeros below.
 *   info: device int[1]: 0 if H is positive-definite, else k = the order of the first leading minor
 *         of the index-REVERSED matrix J H J that is not positive (the factorisation runs bottom-up).
 *   C must be a multiple of 8.  The inverse chain runs on a library-owned side stream (one per
 *   device) that forks from and joins back into `stream`: on return everything is ordered on
 *   `stream`, nothing has synchronised with the host.  One host thread per device.
 * ------------------------------------------------------------------------------------ */
int64_t llmc_chol_workspace_bytes(int64_t C);
int llmc_chol_inv_upper(float* A, int64_t C, void* workspace, int64_t workspace_bytes,
                        int* info, void* stream);

/* ------------------------------------------------------------------------------------
 * fp32-accurate tensor-core GEMM building block ("3xTF32", csrc/tf32.cu) used by K4 and K5:
 *   llmc_split_tf32:  hi = tf32(x), lo = tf32(x - hi)            (x, hi, lo: [rows, cols], ld)
 *   llmc_gemm_f32x3:  C[M,N] = (mode 1) or C -= (mode 0)  A * B  with
 *       A(i,k) = a[i*lda + k],  B(j,k) = b[j*ldb + k]     (both K-major)
 *     evaluated as A_hi*B_hi + A_lo*B_hi + A_hi*B_lo per k8 step with fp32 register
 *     accumulation on wgmma tf32; lower_only != 0 restricts the update to tiles touching
 *     col <= row.
 *   These replace the fp32 cuBLAS SGEMMs of gptq.py:244 and the potrf/potri updates of :172-174.
 * ------------------------------------------------------------------------------------ */
int llmc_split_tf32(const float* x, int64_t rows, int64_t cols, int64_t ld, float* hi,
                    float* lo, void* stream);
int llmc_gemm_f32x3(const float* a_hi, const float* a_lo, int64_t lda, const float* b_hi,
                    const float* b_lo, int64_t ldb, float* c, int64_t ldc, int64_t M, int64_t N,
                    int64_t K, int mode, int lower_only, void* stream);

/* ------------------------------------------------------------------------------------
 * K5  llmc_gptq_colblock — replaces GPTQ.weight_transform (gptq.py:198-244) incl.
 *   search_column_qparams (:358-366).
 *   W      [R, C] fp32, permuted weights; overwritten (scratch)
 *   Hinv   [C, C] fp32 upper factor from llmc_chol_inv_upper
 *   tmp    [R, C] fp32 out: compensated, un-rounded weights (gptq.py:237)
 *   losses [R] fp32 out: per-row sum of (w-q)^2/(2 d^2)  (sum over rows == Losses.sum(), :184)
 *   dynamic groups (static_groups == 0): qparams searched on the compensated columns
 *     [idx, idx+group) when idx % group == 0; written to scales/zeros [R, ng] fp32 in
 *     PERMUTED column order (update_model_qparams, :397-409)
 *   static groups: scales/zeros [R, ng] are inputs, dtype q_dtype; column idx uses group
 *     gmap[idx] (= perm[idx] / group, :225-227) or idx / group when gmap is NULL
 *   group == C means per-channel (qparams always static inputs, search_layer_qparams :368-377).
 *   blocksize must be 128 and group % 128 == 0 or 128 % group == 0.
 *   out_perm [C] int64 or NULL: tmp column i is written to column out_perm[i] (pass the act-order
 *     perm to get tmp[:, invperm] of gptq.py:186-188 without a second pass).
 *   The trailing update W[:, i2:] -= Err1 @ Hinv[i1:i2, i2:] (:244) is applied lazily per 512
 *   columns (same terms, fp32 summation order differs); workspace >= llmc_gptq_workspace_bytes.
 * ------------------------------------------------------------------------------------ */
int64_t llmc_gptq_workspace_bytes(int64_t R, int64_t C);
int llmc_gptq_colblock(float* W, const float* Hinv, int64_t R, int64_t C, int64_t group,
                       int bit, int sym, int static_groups, const int32_t* gmap,
                       void* scales, void* zeros, int q_dtype, float* tmp,
                       const int64_t* out_perm, float* losses, void* workspace,
                       int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------
 * K5  llmc_gptq_colblock_fp8 — the same sweep on an FP8 grid: FloatQuantizer with
 *   `use_qtorch: True` (quant.py:963-1081), e5m2 = 0 for e4m3fn (finfo.max 448), 1 for e5m2
 *   (57344).  Symmetric, zero-point 0, so there are no zeros.  Per column (gptq.py:229-235):
 *   s == 0 -> 1 (quant.py:1062), q = float_quantize(w / s + 0) * s in fp32, the rounding
 *   clamped to +-finfo.max then round-to-nearest-even (the cvt.rn.satfinite of llmc_fp8_quant;
 *   parity with qtorch unpinned).  Dynamic groups: s = max(|max|, |min|).clamp(1e-5) / finfo.max
 *   in fp32, written to scales [R, ng] in permuted order.  Everything else (W, Hinv, tmp,
 *   losses, group / static_groups / gmap / q_dtype, out_perm, workspace) as llmc_gptq_colblock.
 * ------------------------------------------------------------------------------------ */
int llmc_gptq_colblock_fp8(float* W, const float* Hinv, int64_t R, int64_t C, int64_t group,
                           int e5m2, int static_groups, const int32_t* gmap, void* scales,
                           int q_dtype, float* tmp, const int64_t* out_perm, float* losses,
                           void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------
 * K5s llmc_spqr_colblock — SpQR's column sweep (llmc/compression/quantization/spqr.py:172-268,
 *   326-351), the sibling of llmc_gptq_colblock: same Hessian / Cholesky inputs, same block /
 *   super-panel schedule and trailing updates; the in-block step is SpQR's — per group of `group`
 *   columns (16 | 32 | 64 | 128) the leave-one-out outlier search on the current weights
 *   (:174-192, 232-241), group statistics with outliers replaced by the group mean, scale and zero
 *   pushed through the second-level quantizers (s_* / z_*: special.scale / special.zero,
 *   :326-351); per column quantise -> err, unstructured outlier mask err^2 > threshold (:255-259;
 *   outliers keep their weight), rank-1 update.
 *   W [R,C] fp32 permuted weights (consumed), Hinv [C,C] upper factor (llmc_chol_inv_upper).
 *   bit/sym/round_zp: the weight quantizer (symmetric weights are refused by the reference
 *     itself, spqr.py:334; here sym must be 0).
 *   threshold: DEVICE fp32 scalar = relative_threshold * mean(var(W, 0) / diag(Hinv)^2)
 *     (:194-195), +inf disables both outlier mechanisms; simplified_outliers: skip the
 *     leave-one-out search only.
 *   Outputs: scales / zeros [R, C/group] fp32 (second-level quantised, permuted group order),
 *     tmp [R,C] fp32 and mask [R,C] uint8 scattered through out_perm (tmp[:, invperm],
 *     mask[:, invperm], :163-165), losses [R] = sum of err^2 per row.
 *   Workspace as llmc_gptq_colblock (llmc_gptq_workspace_bytes).
 *   The per-row arithmetic is csrc/spqr_row.cuh, which the CPU tests build for the host and
 *   compare bit for bit with the oracle.
 * ------------------------------------------------------------------------------------ */
int llmc_spqr_colblock(float* W, const float* Hinv, int64_t R, int64_t C, int64_t group,
                       int bit, int sym, int round_zp, int s_bit, int s_sym, int s_round_zp,
                       int z_bit, int z_sym, int z_round_zp, const float* threshold,
                       int simplified_outliers, float* scales, float* zeros, float* tmp,
                       uint8_t* mask, const int64_t* out_perm, float* losses, void* workspace,
                       int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------
 * K6  llmc_gemm_bf16 — Y[M,N] = X[M,K] · W[N,K]^T (+ bias[N]); X, W, Y bf16 or fp16,
 *   fp32 accumulation in registers (wgmma.mma_async), TMA-fed.  This is F.linear of
 *   FakeQuantLinear / EffcientFakeQuantLinear.forward (module_utils.py:643, 719).
 * ------------------------------------------------------------------------------------ */
int llmc_gemm_bf16(const void* x, const void* w, const void* bias, void* y, int64_t M,
                   int64_t N, int64_t K, int dtype, void* stream);

/* K6 with the block glue that follows it fused into the epilogue, bit for bit llmc_gemm_bf16
 * followed by the block_ops kernel named (no bias; checks as llmc_gemm_bf16's, plus those listed):
 *   llmc_gemm_rope_qkv  w_qkv = [Wq; Wk; Wv] [n_q + n_k + n_v, K]: q[M, n_q], k[M, n_k], v[M, n_v]
 *                       with llmc_rope (head_dim 128, cos / sin [seq, 128]) applied to q and k;
 *                       row r is position r % seq.  n_q, n_k multiples of 256, n_v of 8,
 *                       M a multiple of seq.
 *   llmc_gemm_swiglu    w_gate_up [2 * inter, K] = gate and up interleaved in 128-row blocks
 *                       (gate rows 0..127, up rows 0..127, gate rows 128..255, ...):
 *                       act[M, inter] = llmc_silu_mul(gate, up); inter a multiple of 128.
 *   llmc_gemm_residual  y[M, N] = llmc_add(res, X W^T); y may be res; N a multiple of 8. */
int llmc_gemm_rope_qkv(const void* x, const void* w_qkv, void* q, void* k, void* v,
                       const void* cosv, const void* sinv, int64_t M, int64_t n_q, int64_t n_k,
                       int64_t n_v, int64_t K, int64_t seq, int dtype, void* stream);
int llmc_gemm_swiglu(const void* x, const void* w_gate_up, void* act, int64_t M, int64_t inter,
                     int64_t K, int dtype, void* stream);
int llmc_gemm_residual(const void* x, const void* w, const void* res, void* y, int64_t M,
                       int64_t N, int64_t K, int dtype, void* stream);

/* K6 with the projections of DeepSeek-V2's multi-head latent attention (MLA, no q LoRA) in its
 * epilogue: heads of 192 = nope 128 | pe 64 for q and k, 128 for v, a 64-wide rotary slice.  Both
 * write into the buffers SDPA then reads as [B, S, H, D] views: q [M, H * 192], k [M, H * 192],
 * v [M, H * 128].  Bit for bit llmc_gemm_bf16 followed by the torch glue of DeepseekV2Attention
 * (split, apply_rotary_emb, broadcast of k_pe, cat).  Checks as llmc_gemm_bf16's, plus those listed.
 *   llmc_gemm_mla_qkv   w_qkva = [W_q; W_kv_a] [H * 192 + kv_lora + 64, K]: q as q_proj lays it
 *                       out with each head's pe slice rotated; latent [M, kv_lora] the first kv_lora
 *                       columns of kv_a_proj_with_mqa; its last 64 columns (k_pe) rotated and written
 *                       to the pe slot of every head of k.  The rotation (apply_rotary_emb) takes
 *                       interleaved pairs (a, b) = rT(acc) and stores rT(a c - b s), rT(a s + b c) in
 *                       fp32, one rounding per operation; cos / sin fp32 [seq, 32]; row r is position
 *                       r % seq.  H a multiple of 4 (q a whole number of 256-wide n-tiles), kv_lora of
 *                       64, M a multiple of seq.
 *   llmc_gemm_mla_kv_b  w_kv_b [H * 256, K] (kv_b_proj): each head's first 128 columns to k's nope
 *                       slot (columns h * 192 .. h * 192 + 127), its last 128 to v. */
int llmc_gemm_mla_qkv(const void* x, const void* w_qkva, void* q, void* k, void* latent,
                      const float* cosv, const float* sinv, int64_t M, int64_t heads, int64_t kv_lora,
                      int64_t K, int64_t seq, int dtype, void* stream);
int llmc_gemm_mla_kv_b(const void* x, const void* w_kv_b, void* k, void* v, int64_t M, int64_t heads,
                       int64_t K, int dtype, void* stream);

/* ------------------------------------------------------------------------------------
 * K6 grouped: a sparse-MoE layer's experts (Mixtral: w2(silu(w1 x) * w3 x) per expert) as one
 * launch per projection, bit for bit the eager per-expert loop (gather x[tok], llmc_gemm_bf16,
 * F.silu * up, * w[tok, slot], index_add_ into zeros).  The routing stays on the device:
 *   xp [rows, K]      the routed rows of x gathered in expert order (rows = tokens * top_k);
 *                     expert e owns rows [offsets[e], offsets[e+1])
 *   offsets [E + 1]   int32 device array, offsets[0] = 0, offsets[E] = rows; read by the kernel,
 *                     never by the host, so no call synchronises
 *   w1, w3, w2        HOST arrays of E device pointers to each expert's weight: w1 / w3
 *                     [inter, K], w2 [N, inter]
 * Launches are sized by the bound ceil(rows / 128) + E m-tiles per column of n-tiles.  Each
 * expert's weight has its own tensor map in the kernel's parameters, which caps the number of
 * experts at LLMC_MOE_MAX_EXPERTS; more return LLMC_EINVAL.  At 64 experts the largest argument
 * list is about 20 KB, past the 4 KB kernel-parameter limit of older toolkits: the library needs
 * CUDA 12.1 or later and a driver of R530 or later (32,764 parameter bytes on Volta and newer).
 * bf16 / fp16, pointers 16-byte aligned, K a multiple of 8.
 *   llmc_moe_gemm_swiglu  act[rows, inter] = llmc_silu_mul(xp W1_e^T, xp W3_e^T) per segment;
 *                         inter a multiple of 128.
 *   llmc_moe_gemm_down    y[rows, N] = rT(rT(act W2_e^T) * w_route[row]) per segment; w_route
 *                         [rows] the routing weights in xp's row order (dtype); N a multiple of 8.
 *   llmc_moe_combine      out[T, N] = the sum of y's rows rows[t, 0], ..., rows[t, top_k - 1]
 *                         (int64 device array), added left to right with one rounding per add;
 *                         N a multiple of 8.
 *   llmc_moe_combine_shared  out[t] = rT(routed[t] + rT(rT(sigmoid(g[t])) * s[t])): routed[t] the
 *                         sum llmc_moe_combine writes, g [T] the shared expert's gate logit (one per
 *                         token, dtype), s [T, N] the shared expert's output; the roundings of
 *                         Qwen2-MoE's block (index_add_ into zeros, F.sigmoid(gate(x)) * shared, the
 *                         add).  top_k > 0, N a multiple of 8, pointers 16-byte aligned; scalar checks,
 *                         then the T == 0 no-op, then pointer checks, all before any CUDA call.
 *   llmc_moe_combine_weighted  out[t] = rT(acc + s[t]), acc = rT(...rT(rT(y[r0] w[r0]) + rT(y[r1]
 *                         w[r1]))...) over r = rows[t, 0], ..., rows[t, top_k - 1]: w fp32 [rows] the
 *                         routing weights in y's row order, s [T, N] the shared experts' output; the
 *                         roundings of DeepSeek-V2's block (expert(x) * w in fp32 rounded once,
 *                         index_add_ into zeros, + shared_experts(x)).  y holds the experts' unscaled
 *                         outputs: llmc_moe_gemm_down with unit routing weights of the dtype, for which
 *                         rT(rT(acc) * 1) = rT(acc).  Checks as llmc_moe_combine_shared's. */
#define LLMC_MOE_MAX_EXPERTS 64
int llmc_moe_gemm_swiglu(const void* xp, const void* const* w1, const void* const* w3,
                         const int32_t* offsets, void* act, int64_t rows, int64_t inter, int64_t K,
                         int64_t n_experts, int dtype, void* stream);
int llmc_moe_gemm_down(const void* act, const void* const* w2, const int32_t* offsets,
                       const void* w_route, void* y, int64_t rows, int64_t N, int64_t inter,
                       int64_t n_experts, int dtype, void* stream);
int llmc_moe_combine(const void* y, const int64_t* rows, void* out, int64_t T, int64_t top_k,
                     int64_t N, int dtype, void* stream);
int llmc_moe_combine_shared(const void* y, const int64_t* rows, const void* gate_logit,
                            const void* shared, void* out, int64_t T, int64_t top_k, int64_t N,
                            int dtype, void* stream);
int llmc_moe_combine_weighted(const void* y, const int64_t* rows, const float* w, const void* shared,
                              void* out, int64_t T, int64_t top_k, int64_t N, int dtype, void* stream);

/* The same two grouped projections on PACKED experts (the llmc_gemm_w4a16 / w8a16 dequant GEMM,
 * grouped): bit for bit the per-expert loop over llmc_gemm_w{4,8}a16[_gidx] with the same operands.
 * bits 4 or 8; each expert linear's codes wq [N_lin, K * bits / 32] int32 (LLMC_OUT_PACK_VLLM),
 * scales / zeros in qparam_dtype (LLMC_F32 or dtype), g_idx int32 [K].  The qparam arrays are HOST
 * arrays of E device pointers like the weights; a zeros array may be NULL (2^(bits-1), symmetric)
 * and a g_idx array NULL (contiguous groups), but within a call either every expert linear has
 * them or none has.  One form per call: bits, qparam dtype, layout (group < 0: qparams [ng, N_lin],
 * else [N_lin, ng]) and ng; without g_idx ng = K / |group|.  K, |group| and (swiglu) inter
 * multiples of 64, |group| dividing K; N a multiple of 8; no bias.  rows == 0 is a no-op; every
 * argument error is returned before any CUDA call (misaligned xp / act / y / wq / g_idx:
 * LLMC_EALIGN).
 *   llmc_moe_gemm_packed_swiglu  act[rows, inter] = llmc_silu_mul(xp W1_e^T, xp W3_e^T) per segment,
 *                                W1_e / W3_e dequantised from wq1 / wq3 [inter, K * bits / 32].
 *   llmc_moe_gemm_packed_down    y[rows, N] = rT(rT(act W2_e^T) * w_route[row]) per segment, W2_e
 *                                from wq2 [N, inter * bits / 32]; K = inter. */
int llmc_moe_gemm_packed_swiglu(const void* xp, int bits, const int32_t* const* wq1,
                                const int32_t* const* wq3, const void* const* s1, const void* const* s3,
                                const void* const* z1, const void* const* z3, const int32_t* const* gidx1,
                                const int32_t* const* gidx3, int qparam_dtype, int64_t group, int64_t ng,
                                const int32_t* offsets, void* act, int64_t rows, int64_t inter, int64_t K,
                                int64_t n_experts, int dtype, void* stream);
int llmc_moe_gemm_packed_down(const void* act, int bits, const int32_t* const* wq2, const void* const* s2,
                              const void* const* z2, const int32_t* const* gidx2, int qparam_dtype,
                              int64_t group, int64_t ng, const int32_t* offsets, const void* w_route, void* y,
                              int64_t rows, int64_t N, int64_t inter, int64_t n_experts, int dtype,
                              void* stream);
/* The same pair on FP8 experts (the llmc_gemm_fp8a16 dequant GEMM, grouped): bit for bit the
 * per-expert loop over llmc_gemm_fp8a16[_gidx] with the same operands.  e5m2 1: e5m2 bytes, 0:
 * e4m3, for every expert linear alike.  Each expert linear's wq is its fp8 bytes [N_lin, K] viewed
 * as int32 [N_lin, K/4]; dequant = rT(fmul_rn(fp32(byte), s)), s = 1 where the scale is 0.  No
 * zero-point arguments; otherwise the operands, layouts and rules of the packed pair above (scales
 * and g_idx HOST arrays of E device pointers, one form per call, rows == 0 a no-op, every argument
 * error before any CUDA call, misalignment LLMC_EALIGN).
 *   llmc_moe_gemm_fp8a16_swiglu  act[rows, inter] = llmc_silu_mul(xp W1_e^T, xp W3_e^T) per segment.
 *   llmc_moe_gemm_fp8a16_down    y[rows, N] = rT(rT(act W2_e^T) * w_route[row]) per segment; K = inter. */
int llmc_moe_gemm_fp8a16_swiglu(const void* xp, int e5m2, const int32_t* const* wq1, const int32_t* const* wq3,
                                const void* const* s1, const void* const* s3, const int32_t* const* gidx1,
                                const int32_t* const* gidx3, int qparam_dtype, int64_t group, int64_t ng,
                                const int32_t* offsets, void* act, int64_t rows, int64_t inter, int64_t K,
                                int64_t n_experts, int dtype, void* stream);
int llmc_moe_gemm_fp8a16_down(const void* act, int e5m2, const int32_t* const* wq2, const void* const* s2,
                              const int32_t* const* gidx2, int qparam_dtype, int64_t group, int64_t ng,
                              const int32_t* offsets, const void* w_route, void* y, int64_t rows, int64_t N,
                              int64_t inter, int64_t n_experts, int dtype, void* stream);

/* The same two grouped projections on W8A8 experts (the llmc_gemm_w8a8_i8 / _fp8 GEMM, grouped): bit
 * for bit the per-expert loop over llmc_gemm_w8a8_* with the same codes and scales, no bias.  fp8 0:
 * int8 codes, else e4m3, for xq / actq and every expert weight alike.  s_x [rows] fp32, one scale
 * per row of xq / actq (a per-tensor static scale repeated per row, in that row order).  Each expert
 * linear's codes w [N_lin, K] with its own fp32 scales s_w (HOST arrays of E device pointers like
 * the weights): N_lin values each when s_w_stride is 1, one each when it is 0.  Output bf16 / fp16
 * (dtype).  K a multiple of 16 (int8: at most llmc_gemm_w8a8_i8's limit); N a multiple of 8.
 * rows == 0 is a no-op; every argument error is returned before any CUDA call (misaligned xq / actq
 * / act / y / codes: LLMC_EALIGN).
 *   llmc_moe_gemm_w8a8_swiglu  act[rows, inter] = llmc_silu_mul(G, U) per segment, G / U the
 *                              llmc_gemm_w8a8_* outputs of xq on w1 / w3 [inter, K] before their
 *                              rounding; inter a multiple of 64.
 *   llmc_moe_gemm_w8a8_down    y[rows, N] = rT(rT(S) * w_route[row]) per segment, S the
 *                              llmc_gemm_w8a8_* output of actq on w2 [N, inter] before its rounding;
 *                              K = inter. */
int llmc_moe_gemm_w8a8_swiglu(const void* xq, const float* s_x, int fp8, const void* const* w1,
                              const void* const* w3, const float* const* s_w1, const float* const* s_w3,
                              int64_t s_w_stride, const int32_t* offsets, void* act, int64_t rows,
                              int64_t inter, int64_t K, int64_t n_experts, int dtype, void* stream);
int llmc_moe_gemm_w8a8_down(const void* actq, const float* s_x, int fp8, const void* const* w2,
                            const float* const* s_w2, int64_t s_w_stride, const int32_t* offsets,
                            const void* w_route, void* y, int64_t rows, int64_t N, int64_t inter,
                            int64_t n_experts, int dtype, void* stream);

/* ------------------------------------------------------------------------------------
 * K6  llmc_gemm_w4a16 — fake-quant forward on PACKED weights:
 *   Y[M,N] = X[M,K] · dequant(Wq)[N,K]^T (+ bias), dequant(Wq)[n,k] =
 *   rT((code - zero) * scale) rounded to `dtype` exactly like the materialised weight of
 *   FakeQuantLinear (module_utils.py:626-643); group-wise dequant runs inside the wgmma
 *   operand pipeline.
 *   wq      [N, K/8] int32, LLMC_OUT_PACK_VLLM layout of UNSIGNED codes (code+2^(bit-1) for
 *           symmetric, code for asymmetric)
 *   scales  [N, K/group], zeros [N, K/group] (integer valued; for symmetric pass NULL ->
 *           zero = 2^(bit-1)), both of type `qparam_dtype`:
 *             LLMC_F32  (GPTQ dynamic groups): fp32 arithmetic, one rounding to `dtype`;
 *           A NEGATIVE `group` (-group_size) says that scales / zeros are stored TRANSPOSED,
 *           [K/group, N]: the 32 rows of a dequant warp then read one coalesced segment per group
 *           instead of 32 strided sectors (what EffcientFakeQuantLinear hands over).
 *             == dtype  (RTN / AWQ / exported checkpoints): the same value computed with packed
 *                       half2 / bf16x2 arithmetic — (q - z) is exact and the product of two
 *                       `dtype` numbers rounds once either way — at 2.4 instead of 4.2
 *                       instructions per weight.
 * ------------------------------------------------------------------------------------ */
/* ------------------------------------------------------------------------------------
 * K8 / K9  AWQ pieces (csrc/awq.cu)
 *   llmc_absmean_cols  get_act_scale (awq.py:74-85): out[c] = mean_t |x[t,c]|  (fp32 accumulate,
 *                      rounded to dtype); workspace >= min(256, T/64) * C floats
 *   llmc_div_cols      scaling_input (base_blockwise_quantization.py:876-889): out = x / s[c]
 *   llmc_mse           calculate_loss (awq.py:134-145): out[0] = mean(((a - b) in dtype).float()^2);
 *                      workspace >= 1024 floats; result stays on the device (no host sync)
 *   llmc_awq_clip      AutoClipper.auto_clip_layer (auto_clip.py:83-191), clip_version v1, w_only:
 *                      w [R,C], x [ns,C] = the sampled tokens, 10 shrink levels (max_shrink 0.5,
 *                      n_grid 20); best_max / best_min [R, ng] dtype; workspace >= R*ng*10 floats.
 * ------------------------------------------------------------------------------------ */
int llmc_absmean_cols(const void* x, int64_t T, int64_t C, int dtype, void* out,
                      float* workspace, int64_t workspace_floats, void* stream);
int llmc_div_cols(const void* x, const void* s, int64_t T, int64_t C, int dtype, void* out,
                  void* stream);
int llmc_mse(const void* a, const void* b, int64_t n, int dtype, float* out, float* workspace,
             void* stream);
int llmc_awq_clip(const void* w, int64_t R, int64_t C, const void* x, int64_t ns, int dtype,
                  int64_t group, int bit, int sym, int clip_sym, void* best_max, void* best_min,
                  float* workspace, int64_t workspace_floats, void* stream);

/* ------------------------------------------------------------------------------------
 * llmc_fp8_quant — FloatQuantizer with use_qtorch (quant.py:963-1229), e4m3 (e5m2 != 0: e5m2).
 *   PARITY UNPINNED: qtorch.float_quantize is third-party and absent; restated as IEEE RNE onto
 *   the fp8 grid with saturation to the finite max (csrc/fp8.cu header).
 *   dynamic != 0: per (row, group) scale = rT(max(absmax, 1e-5) / finfo.max) written to `scales`
 *                 (dtype), then out_mode 1: QDQ (dtype) | 2: fp8 bytes | 0: scales only.
 *                 A NaN in a group makes its scale NaN (the absmax propagates NaN, as amax does).
 *   A scale of 0 (a 16-bit scale that underflowed, or a static 0) quantises with 1 (quant.py:1062);
 *   the scale written is still 0, and FloatQuantizer exports 1 for it.
 *   dynamic == 0: `scales` is an input: [rows * q_row_stride] dtype, or ONE per-tensor scale
 *                 (q_row_stride 0), fp32 when scale_f32 != 0 (torch's CPU scalar-operand path).
 * ------------------------------------------------------------------------------------ */
int llmc_fp8_quant(const void* w, int64_t rows, int64_t cols, int dtype, int64_t group, int e5m2,
                   int dynamic, void* scales, int q_row_stride, int scale_f32, int out_mode,
                   void* out, void* stream);

/* ------------------------------------------------------------------------------------
 * Q10  128 x 128 block FP8 (DeepSeek-V3 / R1 checkpoints), csrc/fp8.cu — PARITY UNPINNED like
 *   llmc_fp8_quant (qtorch):
 *   llmc_fp8_block_quant    weight_cast_to_fp8 (quant.py:32-43) = FloatQuantizer(e4m3, per_block)
 *       .real_quant_weight_dynamic: per [block x block] tile scale = max(absmax, 1e-5) / finfo.max
 *       (fp32, written to scales [ceil(M/block), ceil(N/block)]), q = fp8(x.float() / scale);
 *       out_mode 0 scales only | 1 QDQ (`dtype`) | 2 fp8 bytes.
 *   llmc_fp8_block_dequant  weight_cast_to_bf16 (quant.py:18-29): bf16(fp8.float() * scale_inv).
 *   (LlmcFp8Linear dequantises once with llmc_fp8_block_dequant and runs the bf16 wgmma GEMM — the
 *   reference's non-Hopper branch, module_utils.py:171-178 — unless its USE_FP8GEMM_KERNEL switch
 *   selects the FP8 tensor-core forward below.)
 * ------------------------------------------------------------------------------------ */
int llmc_fp8_block_quant(const void* w, int64_t M, int64_t N, int dtype, int block, int e5m2,
                         float* scales, int out_mode, void* out, void* stream);
int llmc_fp8_block_dequant(const void* w_fp8, int64_t M, int64_t N, int block, int e5m2,
                           const float* scale_inv, void* out_bf16, void* stream);

/* ------------------------------------------------------------------------------------
 * Block-FP8 linear forward on the FP8 tensor cores: the reference's Triton act_quant / fp8_gemm
 *   pair (kernel.py:7-53, 153-242) behind block_wise_fp8_forward_func (module_utils.py:40-45).
 *   llmc_fp8_act_quant  (csrc/fp8.cu) x [rows, K] `dtype`, K % 128 == 0: per contiguous group of 128
 *       elements s = max|x| / 448 and y = e4m3(x / s), both divisions the approximate div.full.f32
 *       the reference's kernel compiles to, the cast cvt.rn.satfinite; y [rows, K] e4m3 bytes,
 *       scales [rows, K/128] fp32.  No clamp: an all-zero group gives s = 0 and NaN codes.  The
 *       max (max.f32) skips NaN elements unless the whole group is NaN (s = NaN); +-inf gives
 *       s = inf, +-0 codes for the finite elements and NaN for the infinite ones.
 *   llmc_gemm_fp8_block (csrc/gemm_8bit.cu) out[M, N] = sum over 128-deep K blocks kb, ascending,
 *       acc = fma(dot_kb * a_s[m, kb], b_s[n / 128, kb], acc), the dot on wgmma e4m3 (Hopper's
 *       reduced-precision accumulator, fresh per K block).  a [M, K], b [N, K] e4m3 (K-major),
 *       a_s [M, K/128], b_s [ceil(N/128), K/128] fp32; K % 128 == 0, N >= 1, M == 0 is a no-op.
 *       out_dtype LLMC_F32: out = acc (fp8_gemm's default-dtype output; bias must be NULL).
 *       out_dtype LLMC_BF16: out = bf16(acc), or with a bias [N] of `bias_dtype` (F32 / F16 / BF16)
 *       bf16(float(bf16(acc)) + float(bias)) — the rounding, then the bias, as module_utils.py:42-44.
 *       Each output element's arithmetic does not depend on M, N or the tile schedule.
 * ------------------------------------------------------------------------------------ */
int llmc_fp8_act_quant(const void* x, int64_t rows, int64_t K, int dtype, void* y, float* scales,
                       void* stream);
int llmc_gemm_fp8_block(const void* a, const float* a_s, const void* b, const float* b_s,
                        const void* bias, int bias_dtype, void* out, int out_dtype, int64_t M,
                        int64_t N, int64_t K, void* stream);

/* ------------------------------------------------------------------------------------
 * Block-forward glue (csrc/block_ops.cu) for F2 block_forward
 * (base_blockwise_quantization.py:367-390): one pass each instead of the HF modules' eager chains.
 *   llmc_rmsnorm   y = weight * (x.float() * rsqrt(mean(x^2) + eps)).to(dtype)     x,y [rows, cols]
 *   llmc_rope      x[B,S,H,D] <- x*cos + rotate_half(x)*sin  (in place; cos/sin [S, D], dtype)
 *   llmc_silu_mul  y = silu(gate) * up                                             n elements
 *   llmc_add       y = a + b
 * ------------------------------------------------------------------------------------ */
int llmc_rmsnorm(const void* x, const void* weight, void* y, int64_t rows, int64_t cols, float eps,
                 int dtype, void* stream);
int llmc_rope(void* x, const void* cosv, const void* sinv, int64_t B, int64_t S, int64_t H,
              int64_t D, int dtype, void* stream);
int llmc_silu_mul(const void* gate, const void* up, void* y, int64_t n, int dtype, void* stream);
int llmc_add(const void* a, const void* b, void* y, int64_t n, int dtype, void* stream);

int llmc_gemm_w4a16(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                    int qparam_dtype, const void* bias, void* y, int64_t M, int64_t N, int64_t K,
                    int64_t group, int dtype, void* stream);
/* llmc_gemm_w8a16 — the same fused forward for INT8 weights (W8A16: rtn_w8a16.yml and the
 *   per-channel W8 configs): wq [N, K/4] int32 = 4 UNSIGNED codes per word along K (code + 128
 *   for symmetric; zeros NULL -> 128), group = K for per-channel.  Dequant in fp32
 *   ((q - z) * s, one rounding to `dtype`), bit-identical to the materialised weight. */
int llmc_gemm_w8a16(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                    int qparam_dtype, const void* bias, void* y, int64_t M, int64_t N, int64_t K,
                    int64_t group, int dtype, void* stream);
/* llmc_gemm_w4a16_gidx / llmc_gemm_w8a16_gidx — the same fused forward with a per-column group
 *   index: replaces GPTQ.w_qdq with act-order (gptq.py:424-452: W[:, perm] -> qdq in groups of
 *   the permuted order -> [:, invperm]) followed by F.linear of EffcientFakeQuantLinear
 *   (module_utils.py:719).  Column k dequantises with group g_idx[k] = invperm[k] / group_size:
 *   g_idx   [K] int32, 0 <= g_idx[k] < ng (a precondition of the caller, not checked on the device)
 *   scales / zeros  [N, ng], or [ng, N] when q_transposed != 0, of type `qparam_dtype`
 *   Arithmetic per element as llmc_gemm_w4a16 (fp32 qparams: one rounding of the fp32 product),
 *   K in its original order, so the result equals llmc_gemm_bf16 on the materialised weight bit
 *   for bit; with g_idx[k] = k / group it equals the contiguous call.  K % 64 == 0, 1 <= ng <= K,
 *   g_idx 16-byte aligned; wq as llmc_gemm_w4a16 / llmc_gemm_w8a16. */
int llmc_gemm_w4a16_gidx(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                         int qparam_dtype, const int32_t* g_idx, int64_t ng, int q_transposed,
                         const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype,
                         void* stream);
/* llmc_gemm_w4a16_awq — the same fused forward on the AutoAWQ GEMM export as stored
 *   (AutoawqRealQuantLinear / MlcllmRealQuantLinear, module_utils.py:1004-1065):
 *   qweight [K, N/8] int32 packed along N: nibble i of word (k, j) is column 8j + AWQ_ORDER[i],
 *           AWQ_ORDER = {0, 2, 4, 6, 1, 3, 5, 7}
 *   qzeros  [K/group, N/8] int32, packed the same way; scales_f16 [K/group, N] fp16 (for bf16
 *           models too: widened in the kernel)
 *   w[n, k] = rT(fp32(q - z) * fp32(s)) with q, z the STORED nibbles (the packer does not clamp, so a
 *   code outside 0..15 has carried into its neighbours; the forward decodes the word as held), one
 *   rounding; the result equals llmc_gemm_bf16 on that weight (+ bias) bit for bit.  bias [N] of
 *   `dtype` or NULL.  K % 64 == 0, group a multiple of 64 dividing K, N % 32 == 0 (as llmc_pack_awq
 *   requires), pointers 16-byte aligned. */
int llmc_gemm_w4a16_awq(const void* x, const int32_t* qweight, const void* scales_f16, const int32_t* qzeros,
                        const void* bias, void* y, int64_t M, int64_t N, int64_t K, int64_t group, int dtype,
                        void* stream);
int llmc_gemm_w8a16_gidx(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                         int qparam_dtype, const int32_t* g_idx, int64_t ng, int q_transposed,
                         const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype,
                         void* stream);
/* llmc_gemm_fp8a16 / llmc_gemm_fp8a16_gidx — the same fused forward for FP8 weights
 *   (FloatQuantizer's e4m3 / e5m2 fake-quant weights; e5m2 != 0: e5m2, else e4m3):
 *   Y = X · dequant(Wq)^T (+ bias),  dequant(Wq)[n,k] = rT(fmul_rn(fp32(byte[n,k]), s)), s the
 *   row's group scale, or 1 where that scale is 0 (quant.py:1062).  This is the QDQ value
 *   llmc_fp8_quant writes (mode 1) computed from the bytes it writes (mode 2), so the result equals
 *   llmc_gemm_bf16 on the materialised weight bit for bit.  fp8 value x 16-bit scale is exact in
 *   fp32; fp32 scales round once in fp32, then to `dtype`.
 *   wq      the fp8 bytes [N, K] viewed as int32 [N, K/4] (byte i of word w = element 4w + i)
 *   scales  as llmc_gemm_w8a16 / llmc_gemm_w8a16_gidx (fp32 or `dtype`, [N, ng] or transposed)
 *   zeros   must be NULL (the grid is symmetric)
 *   Otherwise as llmc_gemm_w8a16 (group: negative for transposed qparams) / llmc_gemm_w8a16_gidx. */
int llmc_gemm_fp8a16(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                     int qparam_dtype, const void* bias, void* y, int64_t M, int64_t N, int64_t K,
                     int64_t group, int dtype, int e5m2, void* stream);
int llmc_gemm_fp8a16_gidx(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                          int qparam_dtype, const int32_t* g_idx, int64_t ng, int q_transposed,
                          const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype,
                          int e5m2, void* stream);
/* llmc_gemm_w2a16 / llmc_gemm_w3a16 (+ _gidx) — the same fused forward for INT2 / INT3 weights
 *   (the W2A16 g64 / W3A16 g128 AWQ recipes, GPTQ at 2 or 3 bits), arguments and rules as
 *   llmc_gemm_w4a16 / llmc_gemm_w4a16_gidx; UNSIGNED codes, zeros NULL -> 2 (W2) / 4 (W3).
 *   W2: wq [N, K/16] int32, LLMC_OUT_PACK_VLLM (code i of word w = element 16w + i, bits 2i..2i+1).
 *   W3: wq [ceil(N/2), 12*K/64] int32 — rows 2r and 2r+1 share a row: for each 64-column step s,
 *       words 12s..12s+5 hold row 2r, 12s+6..12s+11 row 2r+1 (an odd N pads a zero row).  A row's
 *       six words of a step: word l < 4 the low two bits of codes 16l..16l+15 (code 16l+i in bits
 *       2i..2i+1), word 4+m the third bits of codes 32m..32m+31 (code 32m+c at bit c with bits 3
 *       and 4 of c swapped).  Exactly 3 bits per code; llmc_pack_w3_codes writes it.
 *   Bit for bit llmc_gemm_bf16 on the materialised weight rT((code - zero) * scale). */
int llmc_gemm_w2a16(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                    int qparam_dtype, const void* bias, void* y, int64_t M, int64_t N, int64_t K,
                    int64_t group, int dtype, void* stream);
int llmc_gemm_w3a16(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                    int qparam_dtype, const void* bias, void* y, int64_t M, int64_t N, int64_t K,
                    int64_t group, int dtype, void* stream);
int llmc_gemm_w2a16_gidx(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                         int qparam_dtype, const int32_t* g_idx, int64_t ng, int q_transposed,
                         const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype,
                         void* stream);
int llmc_gemm_w3a16_gidx(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                         int qparam_dtype, const int32_t* g_idx, int64_t ng, int q_transposed,
                         const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype,
                         void* stream);
/* llmc_pack_w3_codes — the W3 layout above from SIGNED int32 codes [rows, cols] (code - 4 for an
 *   asymmetric grid, as llmc_pack_vllm_codes takes them), stored as code + 4:
 *   out [ceil(rows/2), 12*cols/64] int32; cols % 64 == 0. */
int llmc_pack_w3_codes(const int32_t* codes, int64_t rows, int64_t cols, int32_t* out, void* stream);
/* llmc_gemm_w2a16_rz / w3a16_rz / w4a16_rz / w8a16_rz — the same fused forward with REAL-VALUED
 *   zero-points (HQQ, SpQR: round_zp False), fp32 qparams only:
 *   dequant(Wq)[n,k] = rT(fmul_rn(fsub_rn(code, z), s)) in fp32, one rounding to `dtype` — the value
 *   of quant.py:710-717 followed by .to(dtype).  code = the stored unsigned code, minus 2^(bit-1)
 *   when sym != 0 (the code is exact; the zero-point is never shifted); zeros NULL -> z = 0.
 *   wq      the layout of each width: W2 / W4 / W8 [N, K*bit/32] LLMC_OUT_PACK_VLLM, W3 the row-pair
 *           layout of llmc_gemm_w3a16
 *   group_axis 0 (groups along K; HQQ axis 1, SpQR): column k uses group g_idx[k] of ng:
 *           scales / zeros [ng, N] fp32, s = scales[g_idx[k] * N + n]; g_idx [K] int32 required,
 *           16-byte aligned, 0 <= g_idx[k] < ng (not checked on the device), 1 <= ng <= K;
 *           contiguous groups pass g_idx[k] = k / group.  `group` is ignored.
 *   group_axis 1 (groups along N; HQQ axis 0, which quantises W^T): row n uses group n / group:
 *           scales / zeros [K, N/group] fp32, s = scales[k * (N/group) + n / group] (HQQ's
 *           buf_scales / buf_zeros as stored); N % group == 0.  g_idx and ng are ignored.
 *   outlier_rows [N+1] int32, outlier_cols [nnz] int32 (ascending within a row, original column
 *           order), outlier_vals [nnz] in `dtype`: CSR of weights kept unquantised (SpQR).  Each
 *           value REPLACES its dequantised element.  All three or none (NULL).
 *   Bit for bit llmc_gemm_bf16 on the materialised weight.  K % 64 == 0; argument errors are
 *   returned before any launch. */
int llmc_gemm_w2a16_rz(const void* x, const int32_t* wq, const float* scales, const float* zeros, int sym,
                       int group_axis, int64_t group, const int32_t* g_idx, int64_t ng,
                       const int32_t* outlier_rows, const int32_t* outlier_cols, const void* outlier_vals,
                       const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype, void* stream);
int llmc_gemm_w3a16_rz(const void* x, const int32_t* wq, const float* scales, const float* zeros, int sym,
                       int group_axis, int64_t group, const int32_t* g_idx, int64_t ng,
                       const int32_t* outlier_rows, const int32_t* outlier_cols, const void* outlier_vals,
                       const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype, void* stream);
int llmc_gemm_w4a16_rz(const void* x, const int32_t* wq, const float* scales, const float* zeros, int sym,
                       int group_axis, int64_t group, const int32_t* g_idx, int64_t ng,
                       const int32_t* outlier_rows, const int32_t* outlier_cols, const void* outlier_vals,
                       const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype, void* stream);
int llmc_gemm_w8a16_rz(const void* x, const int32_t* wq, const float* scales, const float* zeros, int sym,
                       int group_axis, int64_t group, const int32_t* g_idx, int64_t ng,
                       const int32_t* outlier_rows, const int32_t* outlier_cols, const void* outlier_vals,
                       const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype, void* stream);

/* ------------------------------------------------------------------------------------
 * K7  llmc_gemm_w8a8_i8 / llmc_gemm_w8a8_fp8 (csrc/gemm_8bit.cu) — the forward of the exported
 *   W8A8 linears (VllmRealQuantLinear and its Sgl / Lightllm / Lightx2v aliases): both operands
 *   8-bit on the tensor cores, one scale per token and one per output channel.
 *   x    [M, K] activation codes: int8 (i8) or e4m3 bytes (fp8), K-major, row stride K
 *   w    [N, K] weight codes of the same type (the exported `weight`), row stride K
 *   s_x  fp32 activation scales, s_x[m * s_x_stride]; s_w fp32 weight scales, s_w[n * s_w_stride];
 *        a stride of 0 passes one per-tensor scale, 1 a vector
 *   bias [N] of `dtype` or NULL; y [M, N] `dtype` (LLMC_BF16 / LLMC_F16)
 *   Numerics, per output element, independent of M, N and the tile schedule:
 *     acc  = sum_k x[m, k] * w[n, k]
 *            i8:  wgmma s32.s8.s8, the exact integer sum (K <= 131056 keeps it below 2^31 for any
 *                 int8 codes), converted with cvt.rn.f32.s32
 *            fp8: wgmma f32.e4m3.e4m3 with a fresh fp32 dot per 128-deep K block, the blocks summed
 *                 in ascending K order with fadd.rn into an fp32 register (Hopper's tensor core adds
 *                 the products of one block at reduced precision; only that differs from an fp32 sum
 *                 of exact products)
 *     y    = rT(fmul.rn(fmul.rn(acc, s_w[n]), s_x[m]))             without a bias
 *     y    = rT(fadd.rn(fmul.rn(fmul.rn(acc, s_w[n]), s_x[m]), bias[n]))   with one
 *     fp32 throughout, one rounding to `dtype`.
 *   The codes and scales are what the activation quantizer of the same config writes
 *   (llmc_quant_dynamic / llmc_quant_static with LLMC_OUT_CODES_I8, llmc_fp8_quant out_mode 2),
 *   widened to fp32.  K % 16 == 0 (16-byte rows; the K tail of a 128-deep block is zero-filled),
 *   N >= 1, M == 0 is a no-op; x, w, y 16-byte aligned.  Argument errors are returned before any
 *   launch. */
int llmc_gemm_w8a8_i8(const void* x, const float* s_x, int64_t s_x_stride, const void* w, const float* s_w,
                      int64_t s_w_stride, const void* bias, void* y, int64_t M, int64_t N, int64_t K,
                      int dtype, void* stream);
int llmc_gemm_w8a8_fp8(const void* x, const float* s_x, int64_t s_x_stride, const void* w, const float* s_w,
                       int64_t s_w_stride, const void* bias, void* y, int64_t M, int64_t N, int64_t K,
                       int dtype, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LLMC_B200_H_ */
