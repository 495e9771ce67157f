// gemm_w4.cu — K6: fake-quant forward on PACKED INT2 / INT3 / INT4 / INT8 weights, dequantisation
// fused into the wgmma operand pipeline.
//
//   Y[M,N] = X[M,K] . dequant(Wq)[N,K]^T (+ bias),   dequant(n,k) = rT( fp32((code - zero) * scale) )
//
// which is bit-for-bit the bf16/fp16 weight the reference materialises in FakeQuantLinear /
// EffcientFakeQuantLinear (llmc/compression/quantization/module_utils.py:626-643, 722-741) before
// F.linear — so the result equals llmc_gemm_bf16 on that materialised weight exactly (the same
// m64n128k16 wgmma per output element, same K order), while the weight stream from HBM is 4.25
// bits instead of 16 per element.
//
// Tile 128(M) x 128(N) x 64(K).  Pipeline per K step, TWO tc::Rings so that the TMA latency is
// covered by a deep, cheap ring and the dequantised tile by a short one:
//   ring L (6 x 20 KB): X tile [128 x 64] bf16 (swizzle 128B) + packed W tile [128 x 8] int32
//   ring B (3 x 16 KB): the dequantised, 128B-swizzled wgmma B tile; its full barrier counts the
//                       four warps of the dequant group that wrote it
//   warps 0-7          dequant, NG = 2 groups of four warps taking alternate K steps (one weight
//                      row per thread): nibble -> fp32 via the 2^23 magic constant, (q - z) * s in
//                      fp32, round to bf16/fp16, 16-byte stores into ring B, fence.proxy.async;
//                      the group's scale/zero for its NEXT step is prefetched
//   warpgroups 2, 3    consumers: 64 rows each, wgmma m64n128k16 with fp32 register
//                      accumulators; retiring a step's wgmma group frees its ring-L and ring-B
//                      stages; epilogue (bias -> bf16/fp16 -> global) from registers
//   warp 16            TMA into ring L  (17 warps, 544 threads)
// Weight layout: LLMC_OUT_PACK_VLLM of UNSIGNED codes — 8 nibbles per int32 along K, nibble i =
// element 8*w + i; scales / zeros fp32 [N, K/group] (zeros NULL => 2^(bit-1), the symmetric
// +8 offset of module_utils.py:842-844).
//
// Group-index form (kGidx, GPTQ act-order): column k uses group g_idx[k] of ng, in any order, so
// one 64-deep step can touch 64 different groups.  The dequant warps then gather each element's
// (scale, zero) from global memory (L1 / L2: the qparams of an 8B-model linear are at most 3.7 MB
// in fp32) instead of holding one pair per step in registers; staging the CTA's 128-row slice of
// every group in shared memory would take 112 KB at K = 14336, which the ring needs.  The
// arithmetic per element is the fp32 one, fmul_rn((2^23 + q) - (2^23 + z), s), for both qparam
// flavours (the product of a small integer and a 16-bit qparam is exact in fp32, so it rounds to
// the same value as the packed half2 / bf16x2 path).  The ring, the consumers and the epilogue are
// the contiguous form's; K keeps its order, so the result is still llmc_gemm_bf16's bit for bit.
//
// FP8 weight grids (kGrid e4m3 / e5m2, FloatQuantizer's fake-quant weights): the INT8 configuration
// unchanged — 8 KB packed tile, TMA box and swizzle, rings, consumers, epilogue, tile order — on
// the fp8 byte tensor [N, K] viewed as int32 [N, K/4] (byte i of word w = element 4w + i, the W8
// word layout).  Per element: byte -> fp32 (exact, every e4m3 / e5m2 value is an fp16 value),
// fmul_rn(q, s) with s = 1 where the scale is 0 (quant.py:1062), one rounding to bf16 / fp16 —
// fp8_emit's QDQ value (csrc/fp8.cu) from the bytes of its byte mode.  No zero-point.
//
// INT2 / INT3 weights (kBits 2, 3): the same rings, consumers, epilogue and tile order; only the
// packed tile and its decode differ.  Both dequant a row's 64 codes of a step as four pair words
// u(l, j) = code 16l + j in bits 0..2 and code 16l + j + 8 in bits 16..18 (l = 0..3, j = 0..7), so
// the native-qparam path is the INT4 one — (magic | u) as half2 / bf16x2, one HSUB2 + one HMUL2 —
// and the fp32 path lifts each half to 0x4B0000nn = 2^23 + code with one byte-permute.
//   W2: LLMC_OUT_PACK_VLLM, 16 codes per int32 along K, code i of word w (element 16w + i) in bits
//       2i..2i+1: wq [N, K/16], TMA box [128 rows, 4 words] = 16 B per row, no swizzle (a thread's
//       16-byte row read is already conflict-free).
//   W3: 64 codes are 24 B, and a TMA box row must be a multiple of 16 B, so rows 2r and 2r+1 share
//       one tensor row: wq [ceil(N/2), 12 K/64] int32, words 12 s .. 12 s + 11 = K step s of row 2r
//       (6 words) then of row 2r+1 (6 words); an odd N pads one all-zero row.  Box [64 row pairs,
//       12 words] = 48 B, no swizzle; in shared memory row r's 24 bytes of the step sit at 24 r.
//       The 6 words of a row's step: words 0..3 the low two bits of codes 0..63 in the W2 layout
//       (code 16l + i in bits 2i..2i+1 of word l), words 4, 5 the third bit of codes 0..31 and
//       32..63: code 32m + c at bit c' of word 4 + m, c' = c with its bits 3 and 4 swapped (an
//       involution), so that one shift and one AND move the third bits of codes 16l + j and
//       16l + j + 8 under bits 2 and 18 of u(l, j).  Exactly 3 bits per code (plus the odd-N row);
//       llmc_pack_w3_codes writes it.
//
// Real-valued zero-points (kRz, HQQ and SpQR: round_zp False): the group-index form's gather with
// fp32 qparams only; rings, consumers, epilogue, K order and tile order are unchanged.  Per element
// the code is recovered exactly (code - 2^(b-1) on a symmetric grid), then
// rT(__fmul_rn(__fsub_rn(code, z), s)) — quant.py:710-717 in fp32, one rounding — where the 2^23
// formula of the integer forms would round a fractional z.  The zero-point is never shifted.
//   kRzK  groups along K: (s, z) = qparams[g_idx[k], n] of [ng, N] (contiguous groups pass k / group)
//   kRzN  groups along N (HQQ axis 0, which quantises W^T): (s, z) = qparams[k, n / g] of [K, N/g],
//         HQQ's buffers as stored; with g % 32 == 0 a warp's 32 rows read one address (broadcast)
// Outliers (SpQR), optional: CSR over rows, columns ascending in the original (K) order, values in
// `dtype`.  A value REPLACES the dequantised element before the 16-byte store into ring B, so the
// accumulation is llmc_gemm_bf16's on the materialised weight.  Each thread keeps a cursor into its
// row's segment: at every step of its group it skips the columns below the step (the other
// group's steps), then patches the step's columns in order.
//
// AutoAWQ layout (kLayout kPackAwq, the W4 configuration; AutoawqRealQuantLinear's export as stored):
// qweight [K, N/8] and qzeros [K/group, N/8] int32 packed along N, nibble i of word (k, j) = column
// 8j + AWQ_ORDER[i], AWQ_ORDER = {0, 2, 4, 6, 1, 3, 5, 7}; scales [K/group, N] fp16.  The TMA box is
// [64 k-rows x 16 words] of qweight (4 KB, the W4 tile size), SWIZZLE_64B.  Each thread of a dequant
// group takes one 8(n) x 8(k) block: word j = t / 8, k-rows 8 kk .. 8 kk + 7 with kk = t % 8.  It reads
// the 8 words (row 8 kk + (r ^ kk) at read r: with the swizzle a warp's 32 reads hit 32 banks), moves
// them back into k order with three XOR-swap stages, transposes the 8 x 8 nibble block in registers
// (two byte-permute stages and one nibble stage), and so holds for each of its 8 columns the word of
// 8 consecutive k codes that the contiguous W4 layout stores.  That word goes through the contiguous
// form's decode (w4_chunk_native / w4_chunk_f32) into chunk kk of the column's row of the same
// K-major swizzled B tile: the consumers, the epilogue and the K order are those of llmc_gemm_w4a16,
// so the result is llmc_gemm_bf16's on rT((q - z) * s) bit for bit.  The nibbles are decoded as
// stored (the packer's unclamped codes can carry into neighbouring nibbles; the forward reads the
// word the checkpoint holds).  Per thread and group: one qzeros word and its 8 columns' fp16 scales
// (16 B), prefetched one step ahead; fp16 activations take the packed half2 path (the scale is an
// fp16 value), bf16 ones the fp32 path with the scale widened in the kernel.
#include <stdlib.h>

#include <type_traits>

#include <cuda_fp8.h>

#include "tc.cuh"

namespace llmc {

using namespace tc;

namespace w4 {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int kABytes = BM * BK * 2;          // 16 KB
constexpr int kBBytes = BN * BK * 2;          // 16 KB dequantised
constexpr int NG = 2;                         // dequant groups of four warps
// the weight grid: integer codes, or e4m3 / e5m2 bytes (8-bit words, no zero-point)
enum : int { kGridInt = 0, kGridE4M3 = 1, kGridE5M2 = 2 };
// integer zero-points (the 2^23 path), or real-valued ones with groups along K / along N
enum : int { kRzOff = 0, kRzK = 1, kRzN = 2 };
// the packed layout: codes along K per weight row (LLMC_OUT_PACK_VLLM and the W3 row pairs), or
// AutoAWQ's interleaved words along N
enum : int { kPackK = 0, kPackAwq = 1 };
// per weight width: INT2 / INT3 / INT4 -> 2 / 3 / 4 KB packed tile, INT8 -> 8 KB
template <int kBits> struct Cfg {
  static constexpr int kPBytes = BN * BK * kBits / 8;
  static constexpr int kLBytes = kABytes + kPBytes;
  static constexpr int kBStages = 3;
  static constexpr int kLStages = 6;
  static constexpr int kSmemBytes = ring_smem_bytes(kLStages * kLBytes + kBStages * kBBytes);
  static constexpr int kWordsPerRow = BK * kBits / 32;      // int32 per row of the packed tile
  static constexpr int kPackRows = kBits == 3 ? 2 : 1;      // weight rows per row of the packed tensor
  static constexpr int kDequantWarps = 4 * NG;
  static constexpr int kConsumerWarp0 = kDequantWarps;      // first warp of the consumer warpgroups
  static constexpr int kTmaWarp = kDequantWarps + 8;
  static constexpr int kThreads = (kTmaWarp + 1) * 32;
};
struct Params {
  int64_t M, N, K;
  void* out;
  const void* bias;
  const void* scales;       // [N, ng] fp32, or `dtype` when qparam_native
  const void* zeros;        // [N, ng] or null
  int qparam_native;        // qparams are in the activation dtype: packed half2 / bf16x2 dequant
  int q_transposed;         // qparams stored [ng, N] (a warp's 32 rows = one coalesced segment)
  int64_t group;
  int ng;
  const int32_t* g_idx;     // [K] group of each column (group-index form only)
  float zero_default;
  int n_tiles_n, num_units, kb_total, gn;
};
// The real-zero forms' parameters.  A type of their own, so that Params stays within the 128 bytes
// up to which nvcc reads a kernel's struct parameter field by field: the other forms' code is unchanged.
struct ParamsRz : Params {
  int code_shift;           // 2^(bit-1) on a symmetric grid, else 0
  int group_n;              // kRzN: rows per group; the qparams are [K, N / group_n]
  int ngn;                  // kRzN: N / group_n
  const int32_t* o_rows;    // outliers: CSR [N + 1], or null
  const int32_t* o_cols;    // [nnz], ascending within a row
  const uint16_t* o_vals;   // [nnz] in `dtype`
};
template <int kRz> using ParamsOf = std::conditional_t<kRz == kRzOff, Params, ParamsRz>;

// Grouped (sparse-MoE) mode (tc::MoeMode, on packed weights): the gate/up B tile is two 64-row
// boxes of 2 KB (W4) / 4 KB (W8), whole swizzle atoms, so the dequant warps' row swizzle is
// unchanged; rows 0..63 of the tile are w1's, 64..127 w3's.  The epilogue writes act =
// silu(gate) * up for 64 columns (store_swiglu_m64n64).  FP8 grids run in it as in plain mode: the
// W8 configuration on the bytes viewed as words, with no zero-point.
// The grouped operands of one launch, per expert linear (tc::moe_load_b's order): its packed
// codes' tensor map and its qparam and g_idx pointers.  Every linear of a launch has one form:
// bits, qparam dtype and layout, zeros (all null: 2^(bits-1)) and g_idx (all null: contiguous
// groups).  A kernel argument of its own, so that Params stays within its 128 bytes.
struct MoeW4Operands {
  CUtensorMap tmP[2 * LLMC_MOE_MAX_EXPERTS];
  const void* scales[2 * LLMC_MOE_MAX_EXPERTS];
  const void* zeros[2 * LLMC_MOE_MAX_EXPERTS];
  const int32_t* g_idx[2 * LLMC_MOE_MAX_EXPERTS];
  MoeSegments seg;
};
// The whole argument list of the grouped kernel fits the 32,764-byte kernel-parameter space of
// CUDA 12.1+ (driver R530+) at LLMC_MOE_MAX_EXPERTS experts.
static_assert(2 * sizeof(CUtensorMap) + sizeof(Params) + sizeof(MoeW4Operands) <= 32764,
              "LLMC_MOE_MAX_EXPERTS exceeds the kernel-parameter space");

// (a & b) | c in one LOP3
__device__ __forceinline__ uint32_t and_or(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

// ((x2 - zm2) * s2) on two packed 16-bit floats; the subtraction is exact (small integers), the
// product of two T values rounds once — the same value as rT(fp32((q - z) * s)).
template <bool kBf16>
__device__ __forceinline__ uint32_t sub_mul2(uint32_t x2, uint32_t zm2, uint32_t s2) {
  if constexpr (kBf16) {
    const __nv_bfloat162 r = __hmul2(__hsub2(*reinterpret_cast<__nv_bfloat162*>(&x2),
                                             *reinterpret_cast<__nv_bfloat162*>(&zm2)),
                                     *reinterpret_cast<__nv_bfloat162*>(&s2));
    return *reinterpret_cast<const uint32_t*>(&r);
  } else {
    const __half2 r = __hmul2(__hsub2(*reinterpret_cast<__half2*>(&x2), *reinterpret_cast<__half2*>(&zm2)),
                              *reinterpret_cast<__half2*>(&s2));
    return *reinterpret_cast<const uint32_t*>(&r);
  }
}

// four fp8 bytes of a word -> fp32, byte i in f[i]; exact through fp16
template <int G>
__device__ __forceinline__ void fp8x4_to_f32(uint32_t w, float* f) {
  constexpr __nv_fp8_interpretation_t kI = G == kGridE5M2 ? __NV_E5M2 : __NV_E4M3;
  const float2 lo = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w & 0xFFFFu), kI)));
  const float2 hi = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w >> 16), kI)));
  f[0] = lo.x; f[1] = lo.y; f[2] = hi.x; f[3] = hi.y;
}

// quant.py:1062: a zero scale dequantises with 1
__device__ __forceinline__ float fp8_scale(float s) { return s == 0.f ? 1.f : s; }

// W4: one word of 8 codes (nibble e = element e) -> the 16-byte chunk of its 8 dequantised values,
// the arithmetic of the contiguous W4 branch of w4a16_gemm_kernel, for the AutoAWQ layout's
// per-column qparams.  (That branch keeps its inline form: calling these there changes its
// instruction schedule.)  Packed path: 0x6400|q = 1024+q (fp16) / 0x4300|q = 128+q (bf16), two weights per register;
// (magic+q) - (magic+z) and * s are one HSUB2 + one HMUL2 per pair (zm2 = magic + z, s2 = s, both
// halves; both exact in T).
template <bool kBf16>
__device__ __forceinline__ uint4 w4_chunk_native(uint32_t w, uint32_t zm2, uint32_t s2) {
  constexpr uint32_t kMagic2 = kBf16 ? 0x43004300u : 0x64006400u;
  // element pairs (0,4) (1,5) (2,6) (3,7): nibble i in the low half, nibble i+4 in the high
  const uint32_t r04 = sub_mul2<kBf16>(and_or(w, 0x000F000Fu, kMagic2), zm2, s2);
  const uint32_t r15 = sub_mul2<kBf16>(and_or(w >> 4, 0x000F000Fu, kMagic2), zm2, s2);
  const uint32_t r26 = sub_mul2<kBf16>(and_or(w >> 8, 0x000F000Fu, kMagic2), zm2, s2);
  const uint32_t r37 = sub_mul2<kBf16>(and_or(w >> 12, 0x000F000Fu, kMagic2), zm2, s2);
  return make_uint4(__byte_perm(r04, r15, 0x5410), __byte_perm(r26, r37, 0x5410),
                    __byte_perm(r04, r15, 0x7632), __byte_perm(r26, r37, 0x7632));
}

// fp32 path: split the word into even / odd nibbles once, then ONE byte-permute per element builds
// the fp32 bit pattern 0x4B0000nn = 2^23 + nibble; minus zm = 2^23 + z is q - z exactly, times s
// rounds once in fp32, then once to T.
template <int DT>
__device__ __forceinline__ uint4 w4_chunk_f32(uint32_t w, float zm, float s) {
  const uint32_t ev = w & 0x0F0F0F0Fu;           // nibbles 0,2,4,6 in bytes 0..3
  const uint32_t od = (w >> 4) & 0x0F0F0F0Fu;    // nibbles 1,3,5,7
  float v[8];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t be = __byte_perm(ev, 0x4B000000u, 0x7650u + j);
    const uint32_t bo = __byte_perm(od, 0x4B000000u, 0x7650u + j);
    v[2 * j] = fmul_rn(__uint_as_float(be) - zm, s);
    v[2 * j + 1] = fmul_rn(__uint_as_float(bo) - zm, s);
  }
  return make_uint4(pack_pair<DT>(v[0], v[1]), pack_pair<DT>(v[2], v[3]),
                    pack_pair<DT>(v[4], v[5]), pack_pair<DT>(v[6], v[7]));
}

// AutoAWQ: nibble i of a word holds column 8j + AWQ_ORDER[i], AWQ_ORDER = {0, 2, 4, 6, 1, 3, 5, 7}
__device__ __forceinline__ constexpr int awq_column(int i) { return ((i & 3) << 1) | (i >> 2); }

// Transposes the 8 x 8 nibble block w[e] nibble i -> w[i] nibble e: 4 x 4 blocks by 16-bit halves,
// 2 x 2 blocks by bytes, then single nibbles.
__device__ __forceinline__ void transpose_nibbles8(uint32_t* w) {
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const uint32_t a = w[e], b = w[e + 4];
    w[e] = __byte_perm(a, b, 0x5410);
    w[e + 4] = __byte_perm(a, b, 0x7632);
  }
#pragma unroll
  for (int h = 0; h < 4; ++h) {
    const int e = (h & 1) | ((h & 2) << 1);          // 0, 1, 4, 5
    const uint32_t a = w[e], b = w[e + 2];
    w[e] = __byte_perm(a, b, 0x6240);
    w[e + 2] = __byte_perm(a, b, 0x7351);
  }
#pragma unroll
  for (int e = 0; e < 8; e += 2) {
    const uint32_t a = w[e], b = w[e + 1];
    w[e] = (a & 0x0F0F0F0Fu) | ((b << 4) & 0xF0F0F0F0u);
    w[e + 1] = ((a >> 4) & 0x0F0F0F0Fu) | (b & 0xF0F0F0F0u);
  }
}

// W2 / W3: a row's words of one K step in the packed tile (header: 4 words of 2-bit planes, W3 two
// more of third bits).  W3 rows are 24 bytes apart, so the row is read as three 8-byte halves.
template <int kBits>
__device__ __forceinline__ void load_lowbit_row(const uint8_t* pk, int row, uint32_t* w) {
  if constexpr (kBits == 2) {
    const uint4 v = *reinterpret_cast<const uint4*>(pk + row * 16);
    w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
  } else {
    const uint2 a = *reinterpret_cast<const uint2*>(pk + row * 24);
    const uint2 b = *reinterpret_cast<const uint2*>(pk + row * 24 + 8);
    const uint2 c = *reinterpret_cast<const uint2*>(pk + row * 24 + 16);
    w[0] = a.x; w[1] = a.y; w[2] = b.x; w[3] = b.y; w[4] = c.x; w[5] = c.y;
  }
}

// u(l, j): code 16l + j in bits 0..2, code 16l + j + 8 in bits 16..18 (l, j compile-time after unrolling)
template <int kBits>
__device__ __forceinline__ uint32_t lowbit_pair(const uint32_t* w, int l, int j) {
  uint32_t u = (w[l] >> (2 * j)) & 0x00030003u;
  if constexpr (kBits == 3) {
    // third bits of codes 16l + j and 16l + j + 8 sit at bits 8(l & 1) + j and 16 + 8(l & 1) + j
    const int sh = 8 * (l & 1) + j - 2;
    const uint32_t h = sh >= 0 ? w[4 + (l >> 1)] >> sh : w[4 + (l >> 1)] << -sh;
    u = and_or(h, 0x00040004u, u);
  }
  return u;
}

// the outlier cursor's next entry of the row: oc = its column, or INT_MAX past the row's end
__device__ __forceinline__ void next_outlier(const int32_t* cols, int& ocur, int oend, int& oc) {
  ++ocur;
  oc = ocur < oend ? __ldg(cols + ocur) : INT_MAX;
}

// Plain mode: tiles from grouped_tile, B from tmP, qparams from p.  Grouped mode (kMoe): tiles
// from moe_segment_tile, B and the qparams of the tile's expert from `moe`; tmP is unused.
template <bool kBf16, int kBits, bool kGidx, int kGrid, int kRz = kRzOff, int kLayout = kPackK,
          int kMoe = kMoeOff>
__global__ void __launch_bounds__(Cfg<kBits>::kThreads, 1)
w4a16_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmP,
                  const ParamsOf<kRz> p, const __grid_constant__ MoeArg<kMoe, MoeW4Operands> moe) {
  using C = Cfg<kBits>;
  constexpr bool kAwq = kLayout == kPackAwq;
  static_assert(!kAwq || (kBits == 4 && !kGidx && kGrid == kGridInt && kRz == kRzOff),
                "the AutoAWQ layout is a contiguous-group W4 form");
  static_assert(kMoe == kMoeOff || ((kBits == 4 || kBits == 8) && (kGrid == kGridInt || kBits == 8) &&
                                    kRz == kRzOff && !kAwq),
                "the grouped mode runs W4 / W8 integer codes or fp8 bytes in the LLMC_OUT_PACK_VLLM layout");
  constexpr int DT = kBf16 ? LLMC_BF16 : LLMC_F16;
  constexpr int kLStages = C::kLStages;
  constexpr int kLBytes = C::kLBytes;
  constexpr int kBStages = C::kBStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* ringL = ring_base(smem_raw);
  uint8_t* ringB = ringL + kLStages * kLBytes;
  const Ring<kLStages> ring_l(ringB + kBStages * kBBytes);
  const Ring<kBStages> ring_b(ring_l.end());      // full: the dequantised B tile is written
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const MoeW4Operands* g = nullptr;
  if constexpr (kMoe != kMoeOff) g = &moe;
  // the tile of unit u (grouped mode: also its expert, first A row and segment end); false past
  // the last expert's tiles
  auto tile_of = [&](int u, int& e, int& m_blk, int& n_blk, int& row0, int& row_end) -> bool {
    if constexpr (kMoe != kMoeOff) {
      return moe_segment_tile<BM>(g->seg, u, p.n_tiles_n, p.gn, e, m_blk, n_blk, row0, row_end);
    } else {
      grouped_tile(u, p.num_units / p.n_tiles_n, p.n_tiles_n, p.gn, m_blk, n_blk);
      return true;
    }
  };

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    if constexpr (kMoe != kMoeOff) {
      prefetch_moe_tmaps<kMoe>(g->tmP, g->seg);
    } else {
      prefetch_tmap(&tmP);
    }
    ring_l.init(1, 2 + 4);            // empty: both consumer warpgroups + the step's dequant group
    ring_b.init(4, 2);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == C::kTmaWarp) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      PipeState<kLStages> sl;
      for (int u = blockIdx.x; u < p.num_units; u += gridDim.x) {
        int e, m_blk, n_blk, row0, row_end;
        if (!tile_of(u, e, m_blk, n_blk, row0, row_end)) break;
        for (int kb = 0; kb < p.kb_total; ++kb) {
          ring_l.wait_empty(sl);
          uint8_t* a_dst = ringL + sl.stage * kLBytes;
          uint8_t* p_dst = a_dst + kABytes;
          ring_l.expect_tx(sl, kLBytes);
          if constexpr (kMoe != kMoeOff) {
            tma_load_2d(a_dst, &tmA, &ring_l.full[sl.stage], kb * BK, row0);
            moe_load_b<kMoe>(p_dst, g->tmP, &ring_l.full[sl.stage], e, kb * C::kWordsPerRow, n_blk, BN,
                             C::kPBytes / 2);
          } else {
            tma_load_2d(a_dst, &tmA, &ring_l.full[sl.stage], kb * BK, m_blk * BM);
            if constexpr (kAwq)     // [64 k-rows x 16 words] of qweight [K, N/8]
              tma_load_2d(p_dst, &tmP, &ring_l.full[sl.stage], n_blk * (BN / 8), kb * BK);
            else
              tma_load_2d(p_dst, &tmP, &ring_l.full[sl.stage], kb * C::kWordsPerRow * C::kPackRows,
                          n_blk * (BN / C::kPackRows));
          }
          sl.advance();
        }
      }
    }
  } else if (warp >= C::kConsumerWarp0) {
    // ===================== consumers: rows 64 * c .. 64 * c + 63 of the tile =====================
    const int c = (warp - C::kConsumerWarp0) >> 2;
    const int tid = threadIdx.x & 127;
    PipeState<kLStages> sl;
    PipeState<kBStages> sb;
    for (int u = blockIdx.x; u < p.num_units; u += gridDim.x) {
      int e, m_blk, n_blk, row0, row_end;
      if (!tile_of(u, e, m_blk, n_blk, row0, row_end)) break;
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      int prev_l = -1, prev_b = -1;
      for (int kb = 0; kb < p.kb_total; ++kb) {
        ring_l.wait_full(sl);                    // X tile landed
        ring_b.wait_full(sb);                    // W tile dequantised
        wgmma_fence();
        const uint32_t a_addr = smem_u32(ringL + sl.stage * kLBytes) + c * 64 * 128;
        const uint32_t b_addr = smem_u32(ringB + sb.stage * kBBytes);
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t adesc = make_smem_desc(a_addr + k * 32, 16, 1024);
          const uint64_t bdesc = make_smem_desc(b_addr + k * 32, 16, 1024);
          wgmma_m64n128k16<kBf16, 0, 0>(acc, adesc, bdesc, (kb > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();                         // the previous step's group has retired
        if (prev_l >= 0 && tid == 0) {
          ring_l.release(prev_l);
          ring_b.release(prev_b);
        }
        prev_l = sl.stage;
        prev_b = sb.stage;
        sl.advance();
        sb.advance();
      }
      wgmma_wait<0>();
      fence_acc(acc);
      if (prev_l >= 0 && tid == 0) {
        ring_l.release(prev_l);
        ring_b.release(prev_b);
      }
      // ---- epilogue from the accumulator registers ----
      if constexpr (kMoe == kMoeSwiGLU) {
        store_swiglu_m64n64<DT>(acc, static_cast<int64_t>(row0) + c * 64, static_cast<int64_t>(n_blk) * (BN / 2),
                                row_end, p.N, p.out);
      } else if constexpr (kMoe == kMoeDown) {
        store_routed_m64n128<DT>(acc, static_cast<int64_t>(row0) + c * 64, static_cast<int64_t>(n_blk) * BN,
                                 row_end, p.N, p.N, p.out, g->seg.w_route);
      } else {
        store_linear_m64n128<DT>(acc, static_cast<int64_t>(m_blk) * BM + c * 64,
                                 static_cast<int64_t>(n_blk) * BN, p.M, p.N, p.N, p.bias, p.out);
      }
    }
  } else {
    // ===================== dequant warps (4 * NG): one weight row per thread =====================
    // NG groups of four warps take every NG-th K step, so that both groups' dependent
    // unpack -> convert -> store chains are in flight at once.
    const int grp = warp % NG;
    const int row = (warp / NG) * 32 + lane;         // 0..127 inside the group
    uint32_t it = 0;                                 // K steps issued so far (all tiles)
    // grouped mode: the qparams and g_idx of this thread's row's expert linear in the current tile
    // (plain mode reads p's)
    const void* lin_s = nullptr;
    const void* lin_z = nullptr;
    const int32_t* lin_g = nullptr;
    // RAW bits of (scale, zero) — widening / arithmetic happens at use (widen below), so the two
    // loads stay in flight across a whole K step
    auto load_qparams = [&](int64_t n, int gi, uint32_t& s, uint32_t& z) {
      s = 0u; z = 0u;
      if (n >= p.N) return;
      const int64_t qi = p.q_transposed ? static_cast<int64_t>(gi) * p.N + n : n * p.ng + gi;
      if (p.qparam_native) {
        s = __ldg(&reinterpret_cast<const uint16_t*>(kMoe != kMoeOff ? lin_s : p.scales)[qi]);
        if ((kMoe != kMoeOff ? lin_z : p.zeros) != nullptr)
          z = __ldg(&reinterpret_cast<const uint16_t*>(kMoe != kMoeOff ? lin_z : p.zeros)[qi]);
      } else {
        s = __ldg(&reinterpret_cast<const uint32_t*>(kMoe != kMoeOff ? lin_s : p.scales)[qi]);
        if ((kMoe != kMoeOff ? lin_z : p.zeros) != nullptr)
          z = __ldg(&reinterpret_cast<const uint32_t*>(kMoe != kMoeOff ? lin_z : p.zeros)[qi]);
      }
    };
    // AutoAWQ: the qzeros word and the 8 fp16 scales (16 B) of columns n .. n + 7 in group gi
    auto load_awq_qparams = [&](int64_t n, int gi, uint4& s8, uint32_t& zw) {
      s8 = make_uint4(0u, 0u, 0u, 0u); zw = 0u;
      if (n >= p.N) return;
      s8 = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(p.scales) + gi * p.N + n));
      zw = __ldg(static_cast<const uint32_t*>(p.zeros) + gi * (p.N / 8) + n / 8);
    };
    auto widen = [&](uint32_t raw) -> float {
      if (!p.qparam_native) return __uint_as_float(raw);
      return widen16<DT>(static_cast<uint16_t>(raw));
    };
    const bool have_zeros = (kMoe != kMoeOff ? g->zeros[0] : p.zeros) != nullptr;
    const int steps_per_group = static_cast<int>(p.group / BK);
    for (int u = blockIdx.x; u < p.num_units; u += gridDim.x) {
      int e, m_blk, n_blk, row0, row_end;
      if (!tile_of(u, e, m_blk, n_blk, row0, row_end)) break;
      // this thread's weight row (of w1 / w3 for rows 0..63 / 64..127 of a gate/up tile), or with
      // the AutoAWQ layout the first of its 8 columns
      const int64_t n0 = kMoe == kMoeSwiGLU ? static_cast<int64_t>(n_blk) * (BN / 2) + (row & 63)
                                            : static_cast<int64_t>(n_blk) * BN + (kAwq ? 8 * (row >> 3) : row);
      if constexpr (kMoe != kMoeOff) {
        const int lin = kMoe == kMoeSwiGLU ? 2 * e + (row >> 6) : e;
        lin_s = g->scales[lin];
        lin_z = g->zeros[lin];
        lin_g = g->g_idx[lin];
      }
      // real-zero forms: this row's group along N, and its cursor into the outlier CSR (oc = the
      // column of entry ocur, INT_MAX past the row's end)
      int nq = 0, ocur = 0, oend = 0, oc = INT_MAX;
      if constexpr (kRz == kRzN) nq = static_cast<int>(n0 / p.group_n);
      if constexpr (kRz != kRzOff) {
        if (p.o_rows != nullptr && n0 < p.N) {
          ocur = __ldg(p.o_rows + n0);
          oend = __ldg(p.o_rows + n0 + 1);
          oc = ocur < oend ? __ldg(p.o_cols + ocur) : INT_MAX;
        }
      }
      // first K step of this tile that belongs to this group: (it + kb) % NG == grp
      int kb = (grp + NG - static_cast<int>(it % NG)) % NG;
      uint32_t s_cur = 0u, z_cur = 0u;
      uint4 s8_cur = make_uint4(0u, 0u, 0u, 0u);     // AutoAWQ: 8 scales; z_cur is the qzeros word
      if (!kGidx && kb < p.kb_total) {
        if constexpr (kAwq) load_awq_qparams(n0, kb / steps_per_group, s8_cur, z_cur);
        else load_qparams(n0, kb / steps_per_group, s_cur, z_cur);
      }
      for (; kb < p.kb_total; kb += NG) {
        const auto sl = PipeState<kLStages>::at(it + kb);
        const auto sb = PipeState<kBStages>::at(it + kb);
        // qparams of this group's NEXT step are requested now and consumed next iteration
        uint32_t s_nxt = s_cur, z_nxt = z_cur;
        uint4 s8_nxt = s8_cur;
        if (!kGidx && kb + NG < p.kb_total && (kb + NG) / steps_per_group != kb / steps_per_group) {
          if constexpr (kAwq) load_awq_qparams(n0, (kb + NG) / steps_per_group, s8_nxt, z_nxt);
          else load_qparams(n0, (kb + NG) / steps_per_group, s_nxt, z_nxt);
        }
        ring_l.wait_full(sl);
        ring_b.wait_empty(sb);
        const uint8_t* pk = ringL + sl.stage * kLBytes + kABytes;
        uint8_t* bt = ringB + sb.stage * kBBytes;
        const float z_c = have_zeros ? widen(z_cur) : p.zero_default;
        const float zm_cur = 8388608.0f + z_c;        // (2^23 + q) - (2^23 + z) = q - z exactly
        const float s_c = (n0 < p.N) ? widen(s_cur) : 0.f;
        if constexpr (kAwq) {
          // this thread's 8(n) x 8(k) block (header): word j of k-rows 8 kk .. 8 kk + 7
          const int kk = row & 7, j = row >> 3;
          uint32_t w[8];
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            const int k = 8 * kk + (r ^ kk);
            // SWIZZLE_64B: 16-byte chunk c of k-row k sits at chunk c ^ ((k >> 1) & 3)
            w[r] = *reinterpret_cast<const uint32_t*>(pk + k * 64 + ((((j >> 2) ^ ((k >> 1) & 3)) << 4) |
                                                                      ((j & 3) << 2)));
          }
          // w[r] holds k-row 8 kk + (r ^ kk): XOR-swap by the bits of kk so that w[e] holds 8 kk + e
#pragma unroll
          for (int b = 1; b < 8; b <<= 1) {
            const bool f = (kk & b) != 0;
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              if (e & b) continue;
              const uint32_t lo = w[e], hi = w[e | b];
              w[e] = f ? hi : lo;
              w[e | b] = f ? lo : hi;
            }
          }
          transpose_nibbles8(w);   // w[i]: column 8j + awq_column(i), nibble e = k-row 8 kk + e
          const uint32_t sv[4] = {s8_cur.x, s8_cur.y, s8_cur.z, s8_cur.w};
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int col = awq_column(i);
            const uint32_t z = (z_cur >> (4 * i)) & 0xFu;                       // as stored
            const uint32_t sh = (sv[col >> 1] >> (16 * (col & 1))) & 0xFFFFu;   // fp16 bits of the scale
            uint4 o;
            if constexpr (kBf16)   // an fp16 scale is no bf16 value: the fp32 path
              o = w4_chunk_f32<DT>(w[i], __uint_as_float(0x4B000000u | z), __half2float(__ushort_as_half(
                                                                               static_cast<unsigned short>(sh))));
            else                   // fp16 (1024 + z) and s in both halves
              o = w4_chunk_native<false>(w[i], (0x6400u | z) * 0x10001u, sh * 0x10001u);
            // row 8j + col of the K-major SWIZZLE_128B B tile (row & 7 == col), chunk kk
            *reinterpret_cast<uint4*>(bt + (8 * j + col) * 128 + ((kk ^ col) << 4)) = o;
          }
        } else if constexpr (kGidx) {
          // this row's packed words of the step, unswizzled (W4 / W8: word w holds elements 32/kBits * w ..;
          // W2 / W3: the words of load_lowbit_row)
          constexpr int kWords = BK * kBits / 32;
          uint32_t words[kWords];
          if constexpr (kBits == 8) {
            const int sw8 = (row >> 1) & 3;
#pragma unroll
            for (int c4 = 0; c4 < 4; ++c4) {
              const uint4 wv = *reinterpret_cast<const uint4*>(pk + row * 64 + ((c4 ^ sw8) << 4));
              words[4 * c4] = wv.x; words[4 * c4 + 1] = wv.y; words[4 * c4 + 2] = wv.z; words[4 * c4 + 3] = wv.w;
            }
          } else if constexpr (kBits == 4) {
            const int sw = ((row >> 2) & 1) << 4;
            const uint4 w0 = *reinterpret_cast<const uint4*>(pk + row * 32 + sw);
            const uint4 w1 = *reinterpret_cast<const uint4*>(pk + row * 32 + (sw ^ 16));
            words[0] = w0.x; words[1] = w0.y; words[2] = w0.z; words[3] = w0.w;
            words[4] = w1.x; words[5] = w1.y; words[6] = w1.z; words[7] = w1.w;
          } else {
            load_lowbit_row<kBits>(pk, row, words);
          }
          const int4* gk = reinterpret_cast<const int4*>((kMoe != kMoeOff ? lin_g : p.g_idx) +
                                                         static_cast<int64_t>(kb) * BK);
          const int k0 = kb * BK;
          if constexpr (kRz != kRzOff) {
            while (oc < k0) next_outlier(p.o_cols, ocur, oend, oc);   // entries of the other group's steps
          }
#pragma unroll
          for (int c = 0; c < 8; ++c) {              // 16-byte output chunk c = elements 8c .. 8c+7
            uint32_t sr[8], zr[8];
            if constexpr (kRz == kRzN) {
              // row k of the [K, N/g] table (K * N/g < 2^31, checked on the host); a warp's rows
              // share n / g when g % 32 == 0
              const int q0 = (k0 + 8 * c) * p.ngn + nq;
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                sr[e] = 0u; zr[e] = 0u;
                if (n0 < p.N) {
                  sr[e] = __ldg(reinterpret_cast<const uint32_t*>(p.scales) + (q0 + e * p.ngn));
                  if (have_zeros) zr[e] = __ldg(reinterpret_cast<const uint32_t*>(p.zeros) + (q0 + e * p.ngn));
                }
              }
            } else {
              const int4 ga = __ldg(gk + 2 * c), gb = __ldg(gk + 2 * c + 1);   // same for every lane
              const int g[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
#pragma unroll
              for (int e = 0; e < 8; ++e) load_qparams(n0, g[e], sr[e], zr[e]);
            }
            float v[8];
            if constexpr (kGrid != kGridInt) {
              float f[8];
              fp8x4_to_f32<kGrid>(words[2 * c], f);
              fp8x4_to_f32<kGrid>(words[2 * c + 1], f + 4);
#pragma unroll
              for (int e = 0; e < 8; ++e) v[e] = fmul_rn(f[e], fp8_scale(widen(sr[e])));
            } else {
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                uint32_t q;
                if constexpr (kBits == 8) q = (words[2 * c + e / 4] >> (8 * (e % 4))) & 0xFFu;
                else if constexpr (kBits == 4) q = (words[c] >> (4 * e)) & 0xFu;
                else q = (lowbit_pair<kBits>(words, c >> 1, e) >> (16 * (c & 1))) & 0xFFFFu;   // element 8c + e
                if constexpr (kRz != kRzOff) {
                  // exact code, then (code - z) * s as two fp32 ops: no 2^23 offset, no FMA
                  const float code = __int2float_rn(static_cast<int>(q) - p.code_shift);
                  const float z = have_zeros ? __uint_as_float(zr[e]) : 0.f;
                  v[e] = __fmul_rn(__fsub_rn(code, z), __uint_as_float(sr[e]));
                } else {
                  const float zm = 8388608.0f + (have_zeros ? widen(zr[e]) : p.zero_default);
                  v[e] = fmul_rn(__uint_as_float(0x4B000000u | q) - zm, widen(sr[e]));
                }
              }
              if constexpr (kRz != kRzOff) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {          // outliers replace their element (exact: a `dtype` value)
                  if (oc == k0 + 8 * c + e) {
                    v[e] = widen16<DT>(__ldg(p.o_vals + ocur));
                    next_outlier(p.o_cols, ocur, oend, oc);
                  }
                }
              }
            }
            const uint4 o = make_uint4(pack_pair<DT>(v[0], v[1]), pack_pair<DT>(v[2], v[3]),
                                       pack_pair<DT>(v[4], v[5]), pack_pair<DT>(v[6], v[7]));
            *reinterpret_cast<uint4*>(bt + row * 128 + ((c ^ (row & 7)) << 4)) = o;
          }
        } else if constexpr (kBits == 8) {
          // INT8: 64-byte rows, TMA SWIZZLE_64B: 16-byte chunk c of row r sits at c ^ ((r >> 1) & 3).
          // byte -> fp32 through the 2^23 magic (0x4B0000nn), (q - z) * s in fp32, one rounding;
          // bf16 has no exact packed form for 8-bit codes (128 + q needs 9 bits), so both qparam
          // flavours take this path (same value: the product of two T numbers rounds once).
          const int sw8 = (row >> 1) & 3;
#pragma unroll
          for (int c4 = 0; c4 < 4; ++c4) {
            const uint4 wv = *reinterpret_cast<const uint4*>(pk + row * 64 + ((c4 ^ sw8) << 4));
            const uint32_t wd[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              float v[8];
              if constexpr (kGrid != kGridInt) {
                // fp8 bytes: decode, times the scale in fp32
                float f0[4], f1[4];
                fp8x4_to_f32<kGrid>(wd[2 * hh], f0);
                fp8x4_to_f32<kGrid>(wd[2 * hh + 1], f1);
                const float s_f = fp8_scale(s_c);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  v[j] = fmul_rn(f0[j], s_f);
                  v[4 + j] = fmul_rn(f1[j], s_f);
                }
              } else {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  v[j] = fmul_rn(__uint_as_float(__byte_perm(wd[2 * hh], 0x4B000000u, 0x7650u + j)) - zm_cur, s_c);
                  v[4 + j] = fmul_rn(__uint_as_float(__byte_perm(wd[2 * hh + 1], 0x4B000000u, 0x7650u + j)) - zm_cur, s_c);
                }
              }
              const uint4 o = make_uint4(pack_pair<DT>(v[0], v[1]), pack_pair<DT>(v[2], v[3]),
                                         pack_pair<DT>(v[4], v[5]), pack_pair<DT>(v[6], v[7]));
              const int c = c4 * 2 + hh;
              *reinterpret_cast<uint4*>(bt + row * 128 + ((c ^ (row & 7)) << 4)) = o;
            }
          }
        } else if constexpr (kBits < 4) {
          // INT2 / INT3: pair word u(l, j) -> output chunk 2l from its low halves (elements
          // 16l .. 16l+7), chunk 2l+1 from its high halves (16l+8 .. 16l+15)
          uint32_t words[C::kWordsPerRow];
          load_lowbit_row<kBits>(pk, row, words);
          if (p.qparam_native) {
            // as INT4: (magic | u) - (magic + z) is exact, times s rounds once
            constexpr uint32_t kMagic2 = kBf16 ? 0x43004300u : 0x64006400u;
            const uint32_t s2 = pack_pair<DT>(s_c, s_c);
            const uint32_t zm2 = pack_pair<DT>((kBf16 ? 128.f : 1024.f) + z_c, (kBf16 ? 128.f : 1024.f) + z_c);
#pragma unroll
            for (int l = 0; l < 4; ++l) {
              uint32_t r[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) r[j] = sub_mul2<kBf16>(lowbit_pair<kBits>(words, l, j) | kMagic2, zm2, s2);
              const uint4 o0 = make_uint4(__byte_perm(r[0], r[1], 0x5410), __byte_perm(r[2], r[3], 0x5410),
                                          __byte_perm(r[4], r[5], 0x5410), __byte_perm(r[6], r[7], 0x5410));
              const uint4 o1 = make_uint4(__byte_perm(r[0], r[1], 0x7632), __byte_perm(r[2], r[3], 0x7632),
                                          __byte_perm(r[4], r[5], 0x7632), __byte_perm(r[6], r[7], 0x7632));
              *reinterpret_cast<uint4*>(bt + row * 128 + (((2 * l) ^ (row & 7)) << 4)) = o0;
              *reinterpret_cast<uint4*>(bt + row * 128 + (((2 * l + 1) ^ (row & 7)) << 4)) = o1;
            }
          } else {
#pragma unroll
            for (int l = 0; l < 4; ++l) {
              float v[16];
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const uint32_t u = lowbit_pair<kBits>(words, l, j);
                v[j] = fmul_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7650u)) - zm_cur, s_c);
                v[8 + j] = fmul_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7652u)) - zm_cur, s_c);
              }
              const uint4 o0 = make_uint4(pack_pair<DT>(v[0], v[1]), pack_pair<DT>(v[2], v[3]),
                                          pack_pair<DT>(v[4], v[5]), pack_pair<DT>(v[6], v[7]));
              const uint4 o1 = make_uint4(pack_pair<DT>(v[8], v[9]), pack_pair<DT>(v[10], v[11]),
                                          pack_pair<DT>(v[12], v[13]), pack_pair<DT>(v[14], v[15]));
              *reinterpret_cast<uint4*>(bt + row * 128 + (((2 * l) ^ (row & 7)) << 4)) = o0;
              *reinterpret_cast<uint4*>(bt + row * 128 + (((2 * l + 1) ^ (row & 7)) << 4)) = o1;
            }
          }
        } else {
          // packed tile is TMA-swizzled (32B): half h of row r sits at half h ^ ((r >> 2) & 1)
          const int sw = ((row >> 2) & 1) << 4;
          const uint4 w0 = *reinterpret_cast<const uint4*>(pk + row * 32 + sw);
          const uint4 w1 = *reinterpret_cast<const uint4*>(pk + row * 32 + (sw ^ 16));
          const uint32_t words[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
          if (p.qparam_native) {
            // packed path: 0x6400|q = 1024+q (fp16) / 0x4300|q = 128+q (bf16), two weights per
            // register; (magic+q) - (magic+z) and * s are one HSUB2 + one HMUL2 per pair
            constexpr uint32_t kMagic2 = kBf16 ? 0x43004300u : 0x64006400u;
            const uint32_t s2 = pack_pair<DT>(s_c, s_c);                          // exact: s is a T value
            const uint32_t zm2 = pack_pair<DT>((kBf16 ? 128.f : 1024.f) + z_c,
                                               (kBf16 ? 128.f : 1024.f) + z_c);       // exact: <= 8 bits
#pragma unroll
            for (int c = 0; c < 8; ++c) {
              const uint32_t w = words[c];
              // element pairs (0,4) (1,5) (2,6) (3,7): nibble i in the low half, nibble i+4 in the high
              const uint32_t r04 = sub_mul2<kBf16>(and_or(w, 0x000F000Fu, kMagic2), zm2, s2);
              const uint32_t r15 = sub_mul2<kBf16>(and_or(w >> 4, 0x000F000Fu, kMagic2), zm2, s2);
              const uint32_t r26 = sub_mul2<kBf16>(and_or(w >> 8, 0x000F000Fu, kMagic2), zm2, s2);
              const uint32_t r37 = sub_mul2<kBf16>(and_or(w >> 12, 0x000F000Fu, kMagic2), zm2, s2);
              const uint4 o = make_uint4(__byte_perm(r04, r15, 0x5410), __byte_perm(r26, r37, 0x5410),
                                         __byte_perm(r04, r15, 0x7632), __byte_perm(r26, r37, 0x7632));
              // K-major SWIZZLE_128B: 16-byte chunk c of row r lives at chunk (c ^ (r & 7))
              *reinterpret_cast<uint4*>(bt + row * 128 + ((c ^ (row & 7)) << 4)) = o;
            }
          } else {
#pragma unroll
            for (int c = 0; c < 8; ++c) {            // one 16-byte chunk = 8 elements = one word
              // split the word into even / odd nibbles once, then ONE byte-permute per element
              // builds the fp32 bit pattern 0x4B0000nn = 2^23 + nibble
              const uint32_t w = words[c];
              const uint32_t ev = w & 0x0F0F0F0Fu;           // nibbles 0,2,4,6 in bytes 0..3
              const uint32_t od = (w >> 4) & 0x0F0F0F0Fu;    // nibbles 1,3,5,7
              float v[8];
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const uint32_t be = __byte_perm(ev, 0x4B000000u, 0x7650u + j);
                const uint32_t bo = __byte_perm(od, 0x4B000000u, 0x7650u + j);
                v[2 * j] = fmul_rn(__uint_as_float(be) - zm_cur, s_c);
                v[2 * j + 1] = fmul_rn(__uint_as_float(bo) - zm_cur, s_c);
              }
              const uint4 o = make_uint4(pack_pair<DT>(v[0], v[1]), pack_pair<DT>(v[2], v[3]),
                                         pack_pair<DT>(v[4], v[5]), pack_pair<DT>(v[6], v[7]));
              *reinterpret_cast<uint4*>(bt + row * 128 + ((c ^ (row & 7)) << 4)) = o;
            }
          }
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&ring_b.full[sb.stage]);
          ring_l.release(sl.stage);                // packed tile consumed
        }
        s_cur = s_nxt;
        z_cur = z_nxt;
        s8_cur = s8_nxt;
      }
      it += static_cast<uint32_t>(p.kb_total);
    }
  }
}

}  // namespace w4

}  // namespace llmc

using namespace llmc;

template <int kBits, int kGrid, int kRz, int kLayout = w4::kPackK>
static int launch_wNa16(const void* x, const int32_t* wq, const void* bias, void* y, int64_t M, int64_t N,
                        int64_t K, int dtype, void* stream, const char* name, w4::ParamsOf<kRz> p);

template <int kBits, int kGrid = w4::kGridInt>
static int gemm_wNa16(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                      int qparam_dtype, const void* bias, void* y, int64_t M, int64_t N, int64_t K,
                      int64_t group, const int32_t* g_idx, int64_t ng, int dtype, int q_transposed,
                      void* stream, const char* name) {
  using namespace w4;
  LLMC_CHECK_ARG(M >= 0 && N >= 0 && K > 0, "%s: bad shape", name);
  if (M == 0 || N == 0) return LLMC_OK;
  LLMC_CHECK_ARG(x && wq && scales && y, "%s: null pointer", name);
  LLMC_CHECK_ARG(dtype == LLMC_BF16 || dtype == LLMC_F16, "%s: dtype must be bf16 or fp16", name);
  LLMC_CHECK_ARG(qparam_dtype == LLMC_F32 || qparam_dtype == dtype,
                 "%s: qparam_dtype must be fp32 or the activation dtype", name);
  if (g_idx == nullptr) {
    LLMC_CHECK_ARG(group > 0 && K % group == 0 && group % BK == 0,
                   "%s: group %lld must divide K=%lld and be a multiple of %d", name, (long long)group,
                   (long long)K, BK);
    ng = K / group;
  } else {
    LLMC_CHECK_ARG(ng >= 1 && ng <= K, "%s: ng=%lld groups for K=%lld columns", name, (long long)ng,
                   (long long)K);
  }
  if (K % 64 != 0 || !aligned16(x) || !aligned16(wq) || !aligned16(y) || (g_idx && !aligned16(g_idx))) {
    set_last_error("%s: K=%lld must be a multiple of 64 and pointers 16-byte aligned", name, (long long)K);
    return LLMC_EALIGN;
  }
  Params p{};
  p.scales = scales; p.zeros = zeros;
  // packed half2 / bf16x2 dequant exists for INT4 only; INT8 widens native qparams to fp32
  p.qparam_native = (qparam_dtype != LLMC_F32) ? 1 : 0;
  p.q_transposed = q_transposed ? 1 : 0;
  p.group = g_idx ? K : group; p.ng = static_cast<int>(ng);
  p.g_idx = g_idx;
  p.zero_default = static_cast<float>(1 << (kBits - 1));
  return launch_wNa16<kBits, kGrid, w4::kRzOff>(x, wq, bias, y, M, N, K, dtype, stream, name, p);
}

// Tensor maps, tile counts and the launch of a validated call whose dequant fields `p` holds.
template <int kBits, int kGrid, int kRz, int kLayout>
static int launch_wNa16(const void* x, const int32_t* wq, const void* bias, void* y, int64_t M, int64_t N,
                        int64_t K, int dtype, void* stream, const char* name, w4::ParamsOf<kRz> p) {
  using namespace w4;
  using C = Cfg<kBits>;
  constexpr int wpr = C::kWordsPerRow;
  constexpr int pr = C::kPackRows;
  // W4 / W8 rows are 32 / 64 B and TMA-swizzled; the 16-byte W2 rows and 48-byte W3 row pairs are not
  constexpr CUtensorMapSwizzle swz = kBits == 4 ? CU_TENSOR_MAP_SWIZZLE_32B
                                     : kBits == 8 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUtensorMap tmA, tmP;
  if (int rc = encode_tmap_2d(&tmA, x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, M, K, K, BM, BK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  if constexpr (kLayout == kPackAwq) {
    // qweight [K, N/8]: 64 k-rows of 16 words (64 B) per box
    if (int rc = encode_tmap_2d(&tmP, wq, CU_TENSOR_MAP_DATA_TYPE_INT32, 4, K, N / 8, N / 8, BK, BN / 8,
                                CU_TENSOR_MAP_SWIZZLE_64B))
      return rc;
  } else {
    if (int rc = encode_tmap_2d(&tmP, wq, CU_TENSOR_MAP_DATA_TYPE_INT32, 4, (N + pr - 1) / pr, K * kBits / 32 * pr,
                                K * kBits / 32 * pr, BN / pr, wpr * pr, swz))
      return rc;
  }
  p.M = M; p.N = N; p.K = K; p.out = y; p.bias = bias;
  p.n_tiles_n = static_cast<int>((N + BN - 1) / BN);
  const int64_t mt = (M + BM - 1) / BM;
  LLMC_CHECK_ARG(mt * p.n_tiles_n < (1ll << 31), "%s: too many tiles", name);
  p.num_units = static_cast<int>(mt * p.n_tiles_n);
  p.kb_total = static_cast<int>(K / BK);
  // One byte over the packed n-tile's size, so that the tile order, and with it the measured
  // timing, stays as it is: the width is one n-tile narrower than 32 MB allows when the tile bytes
  // divide 32 MB exactly (W8 at K = 4096: 63 n-tiles, not 64).  The width changes no output, only
  // L2 traffic; change it only together with a measurement.
  p.gn = l2_group_width(static_cast<int64_t>(BN) * K * kBits / 8 + 1, p.n_tiles_n);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  constexpr int smem = C::kSmemBytes;
  static_assert(smem <= 227 * 1024, "shared memory budget");
  if constexpr (kRz != kRzOff) {
    // the real-zero forms always gather per element (the group-index dequant)
    auto kernel = dtype == LLMC_BF16 ? w4a16_gemm_kernel<true, kBits, true, kGrid, kRz>
                                     : w4a16_gemm_kernel<false, kBits, true, kGrid, kRz>;
    return launch_persistent(kernel, p.num_units, C::kThreads, smem, st, tmA, tmP, p, nullptr);
  } else if constexpr (kLayout == kPackAwq) {
    auto kernel = dtype == LLMC_BF16 ? w4a16_gemm_kernel<true, kBits, false, kGrid, kRzOff, kPackAwq>
                                     : w4a16_gemm_kernel<false, kBits, false, kGrid, kRzOff, kPackAwq>;
    return launch_persistent(kernel, p.num_units, C::kThreads, smem, st, tmA, tmP, p, nullptr);
  } else {
    auto kernel = p.g_idx ? (dtype == LLMC_BF16 ? w4a16_gemm_kernel<true, kBits, true, kGrid>
                                                : w4a16_gemm_kernel<false, kBits, true, kGrid>)
                          : (dtype == LLMC_BF16 ? w4a16_gemm_kernel<true, kBits, false, kGrid>
                                                : w4a16_gemm_kernel<false, kBits, false, kGrid>);
    return launch_persistent(kernel, p.num_units, C::kThreads, smem, st, tmA, tmP, p, nullptr);
  }
}

extern "C" int llmc_gemm_w4a16(const void* x, const int32_t* wq, const void* scales,
                               const void* zeros, int qparam_dtype, const void* bias, void* y,
                               int64_t M, int64_t N, int64_t K, int64_t group, int dtype,
                               void* stream) {
  // `group` < 0 selects the TRANSPOSED qparam layout [K/|group|, N] (coalesced per-warp loads)
  return gemm_wNa16<4>(x, wq, scales, zeros, qparam_dtype, bias, y, M, N, K, group < 0 ? -group : group,
                       nullptr, 0, dtype, group < 0, stream, "gemm_w4a16");
}

// INT8 weights: wq [N, K/4] int32, 4 UNSIGNED codes per word along K (code + 128 for symmetric,
// zeros NULL => 128), otherwise as llmc_gemm_w4a16.
extern "C" int llmc_gemm_w8a16(const void* x, const int32_t* wq, const void* scales,
                               const void* zeros, int qparam_dtype, const void* bias, void* y,
                               int64_t M, int64_t N, int64_t K, int64_t group, int dtype,
                               void* stream) {
  return gemm_wNa16<8>(x, wq, scales, zeros, qparam_dtype, bias, y, M, N, K, group < 0 ? -group : group,
                       nullptr, 0, dtype, group < 0, stream, "gemm_w8a16");
}

// Group-index form: column k dequantises with the qparams of group g_idx[k] (0 <= g_idx[k] < ng,
// the caller's guarantee; not checked on the device).
extern "C" int llmc_gemm_w4a16_gidx(const void* x, const int32_t* wq, const void* scales,
                                    const void* zeros, int qparam_dtype, const int32_t* g_idx,
                                    int64_t ng, int q_transposed, const void* bias, void* y,
                                    int64_t M, int64_t N, int64_t K, int dtype, void* stream) {
  LLMC_CHECK_ARG(g_idx != nullptr, "gemm_w4a16_gidx: g_idx is NULL");
  return gemm_wNa16<4>(x, wq, scales, zeros, qparam_dtype, bias, y, M, N, K, 0, g_idx, ng, dtype,
                       q_transposed, stream, "gemm_w4a16_gidx");
}

extern "C" int llmc_gemm_w8a16_gidx(const void* x, const int32_t* wq, const void* scales,
                                    const void* zeros, int qparam_dtype, const int32_t* g_idx,
                                    int64_t ng, int q_transposed, const void* bias, void* y,
                                    int64_t M, int64_t N, int64_t K, int dtype, void* stream) {
  LLMC_CHECK_ARG(g_idx != nullptr, "gemm_w8a16_gidx: g_idx is NULL");
  return gemm_wNa16<8>(x, wq, scales, zeros, qparam_dtype, bias, y, M, N, K, 0, g_idx, ng, dtype,
                       q_transposed, stream, "gemm_w8a16_gidx");
}

// AutoAWQ GEMM layout as stored (header): qweight [K, N/8], qzeros [K/group, N/8] int32, scales
// [K/group, N] fp16.  N % 32 == 0: a qweight row is then a multiple of the 16 bytes a TMA row stride
// needs (the AutoAWQ packer, llmc_pack_awq, requires it as well).
extern "C" int llmc_gemm_w4a16_awq(const void* x, const int32_t* qweight, const void* scales_f16,
                                   const int32_t* qzeros, const void* bias, void* y, int64_t M, int64_t N,
                                   int64_t K, int64_t group, int dtype, void* stream) {
  using namespace w4;
  const char* name = "gemm_w4a16_awq";
  LLMC_CHECK_ARG(M >= 0 && N >= 0 && K > 0, "%s: bad shape", name);
  if (M == 0 || N == 0) return LLMC_OK;
  LLMC_CHECK_ARG(x && qweight && scales_f16 && qzeros && y, "%s: null pointer", name);
  LLMC_CHECK_ARG(dtype == LLMC_BF16 || dtype == LLMC_F16, "%s: dtype must be bf16 or fp16", name);
  LLMC_CHECK_ARG(N % 32 == 0, "%s: N=%lld must be a multiple of 32", name, (long long)N);
  LLMC_CHECK_ARG(group > 0 && K % group == 0 && group % BK == 0,
                 "%s: group %lld must divide K=%lld and be a multiple of %d", name, (long long)group,
                 (long long)K, BK);
  if (K % 64 != 0 || !aligned16(x) || !aligned16(qweight) || !aligned16(scales_f16) || !aligned16(qzeros) ||
      !aligned16(y)) {
    set_last_error("%s: K=%lld must be a multiple of 64 and pointers 16-byte aligned", name, (long long)K);
    return LLMC_EALIGN;
  }
  Params p{};
  p.scales = scales_f16; p.zeros = qzeros;
  p.qparam_native = dtype == LLMC_F16 ? 1 : 0;   // fp16 scales are native to fp16 activations only
  p.q_transposed = 1;
  p.group = group; p.ng = static_cast<int>(K / group);
  return launch_wNa16<4, kGridInt, kRzOff, kPackAwq>(x, qweight, bias, y, M, N, K, dtype, stream, name, p);
}

// INT2 weights: wq [N, K/16] (LLMC_OUT_PACK_VLLM, zeros NULL => 2); INT3 weights: wq
// [ceil(N/2), 12 K/64] in the row-pair layout of the header (llmc_pack_w3_codes, zeros NULL => 4).
// Otherwise as llmc_gemm_w4a16 / llmc_gemm_w4a16_gidx.
extern "C" int llmc_gemm_w2a16(const void* x, const int32_t* wq, const void* scales,
                               const void* zeros, int qparam_dtype, const void* bias, void* y,
                               int64_t M, int64_t N, int64_t K, int64_t group, int dtype,
                               void* stream) {
  return gemm_wNa16<2>(x, wq, scales, zeros, qparam_dtype, bias, y, M, N, K, group < 0 ? -group : group,
                       nullptr, 0, dtype, group < 0, stream, "gemm_w2a16");
}

extern "C" int llmc_gemm_w3a16(const void* x, const int32_t* wq, const void* scales,
                               const void* zeros, int qparam_dtype, const void* bias, void* y,
                               int64_t M, int64_t N, int64_t K, int64_t group, int dtype,
                               void* stream) {
  return gemm_wNa16<3>(x, wq, scales, zeros, qparam_dtype, bias, y, M, N, K, group < 0 ? -group : group,
                       nullptr, 0, dtype, group < 0, stream, "gemm_w3a16");
}

extern "C" int llmc_gemm_w2a16_gidx(const void* x, const int32_t* wq, const void* scales,
                                    const void* zeros, int qparam_dtype, const int32_t* g_idx,
                                    int64_t ng, int q_transposed, const void* bias, void* y,
                                    int64_t M, int64_t N, int64_t K, int dtype, void* stream) {
  LLMC_CHECK_ARG(g_idx != nullptr, "gemm_w2a16_gidx: g_idx is NULL");
  return gemm_wNa16<2>(x, wq, scales, zeros, qparam_dtype, bias, y, M, N, K, 0, g_idx, ng, dtype,
                       q_transposed, stream, "gemm_w2a16_gidx");
}

extern "C" int llmc_gemm_w3a16_gidx(const void* x, const int32_t* wq, const void* scales,
                                    const void* zeros, int qparam_dtype, const int32_t* g_idx,
                                    int64_t ng, int q_transposed, const void* bias, void* y,
                                    int64_t M, int64_t N, int64_t K, int dtype, void* stream) {
  LLMC_CHECK_ARG(g_idx != nullptr, "gemm_w3a16_gidx: g_idx is NULL");
  return gemm_wNa16<3>(x, wq, scales, zeros, qparam_dtype, bias, y, M, N, K, 0, g_idx, ng, dtype,
                       q_transposed, stream, "gemm_w3a16_gidx");
}

// ---- the INT3 weight layout (header): one thread per output word ----
namespace llmc {
namespace w4 {
__global__ void __launch_bounds__(256)
pack_w3_codes_kernel(const int32_t* __restrict__ codes, int64_t rows, int64_t cols, int32_t* __restrict__ out) {
  const int64_t wpp = cols / BK * 12;                       // words per row pair
  const int64_t total = (rows + 1) / 2 * wpp;
  for (int64_t u = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < total;
       u += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t pair = u / wpp, rem = u - pair * wpp;
    const int64_t step = rem / 12;
    const int w = static_cast<int>(rem % 12);
    const int64_t r = 2 * pair + w / 6;
    uint32_t word = 0;
    if (r < rows) {
      const int32_t* c = codes + r * cols + step * BK;
      const int f = w % 6;
      if (f < 4) {                                          // low two bits of codes 16f .. 16f + 15
        for (int i = 0; i < 16; ++i) word |= (static_cast<uint32_t>(c[16 * f + i] + 4) & 3u) << (2 * i);
      } else {                                              // third bits of codes 32m .. 32m + 31
        const int m = f - 4;
        for (int b = 0; b < 32; ++b) {
          const int cc = (b & ~24) | ((b & 8) << 1) | ((b & 16) >> 1);   // b with bits 3 and 4 swapped
          word |= ((static_cast<uint32_t>(c[32 * m + cc] + 4) >> 2) & 1u) << b;
        }
      }
    }
    out[u] = static_cast<int32_t>(word);
  }
}
}  // namespace w4
}  // namespace llmc

// codes [rows, cols] int32, SIGNED (code - 4 for an asymmetric grid, as llmc_pack_vllm_codes takes
// them); stored as code + 4 in 3 bits.  out [ceil(rows/2), 12 cols/64] int32.
extern "C" int llmc_pack_w3_codes(const int32_t* codes, int64_t rows, int64_t cols, int32_t* out, void* stream) {
  LLMC_CHECK_ARG(rows >= 0 && cols >= 0, "pack_w3_codes: bad shape");
  LLMC_CHECK_ARG(cols % w4::BK == 0, "pack_w3_codes: cols=%lld must be a multiple of %d", (long long)cols, w4::BK);
  if (rows == 0 || cols == 0) return LLMC_OK;
  LLMC_CHECK_ARG(codes && out, "pack_w3_codes: null pointer");
  int64_t blocks = ((rows + 1) / 2 * (cols / w4::BK * 12) + 255) / 256;
  if (blocks > kNumSMs * 32) blocks = kNumSMs * 32;
  w4::pack_w3_codes_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(codes, rows, cols, out);
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

// FP8 weights (e5m2 != 0: e5m2, else e4m3): wq = the fp8 bytes [N, K] viewed as int32 [N, K/4],
// scales as llmc_gemm_w8a16, zeros must be NULL.  dequant = rT(fmul_rn(fp32(byte), s)), s = 1
// where the scale is 0.
static int gemm_fp8a16(const void* x, const int32_t* wq, const void* scales, const void* zeros,
                       int qparam_dtype, const void* bias, void* y, int64_t M, int64_t N, int64_t K,
                       int64_t group, const int32_t* g_idx, int64_t ng, int dtype, int q_transposed,
                       int e5m2, void* stream, const char* name) {
  LLMC_CHECK_ARG(zeros == nullptr, "%s: an fp8 grid has no zero-point (zeros must be NULL)", name);
  LLMC_CHECK_ARG(e5m2 == 0 || e5m2 == 1, "%s: e5m2 must be 0 (e4m3) or 1 (e5m2), got %d", name, e5m2);
  if (e5m2)
    return gemm_wNa16<8, w4::kGridE5M2>(x, wq, scales, nullptr, qparam_dtype, bias, y, M, N, K, group, g_idx,
                                        ng, dtype, q_transposed, stream, name);
  return gemm_wNa16<8, w4::kGridE4M3>(x, wq, scales, nullptr, qparam_dtype, bias, y, M, N, K, group, g_idx,
                                      ng, dtype, q_transposed, stream, name);
}

extern "C" int llmc_gemm_fp8a16(const void* x, const int32_t* wq, const void* scales,
                                const void* zeros, int qparam_dtype, const void* bias, void* y,
                                int64_t M, int64_t N, int64_t K, int64_t group, int dtype, int e5m2,
                                void* stream) {
  return gemm_fp8a16(x, wq, scales, zeros, qparam_dtype, bias, y, M, N, K, group < 0 ? -group : group,
                     nullptr, 0, dtype, group < 0, e5m2, stream, "gemm_fp8a16");
}

extern "C" int llmc_gemm_fp8a16_gidx(const void* x, const int32_t* wq, const void* scales,
                                     const void* zeros, int qparam_dtype, const int32_t* g_idx,
                                     int64_t ng, int q_transposed, const void* bias, void* y,
                                     int64_t M, int64_t N, int64_t K, int dtype, int e5m2,
                                     void* stream) {
  LLMC_CHECK_ARG(g_idx != nullptr, "gemm_fp8a16_gidx: g_idx is NULL");
  return gemm_fp8a16(x, wq, scales, zeros, qparam_dtype, bias, y, M, N, K, 0, g_idx, ng, dtype, q_transposed,
                     e5m2, stream, "gemm_fp8a16_gidx");
}

// Real-valued zero-points (HQQ, SpQR): fp32 scales / zeros, dequant rT(fmul(fsub(code, z), s)) with
// the exact code (minus 2^(bit-1) when sym), zeros NULL => 0.  group_axis 0: column k uses group
// g_idx[k] of ng, qparams [ng, N]; group_axis 1: rows n use group n / group, qparams [K, N/group].
// Outliers (rows [N+1], cols [nnz], vals [nnz] in `dtype`; all three or none) replace their element.
template <int kBits>
static int gemm_wNa16_rz(const void* x, const int32_t* wq, const float* scales, const float* zeros, int sym,
                         int group_axis, int64_t group, const int32_t* g_idx, int64_t ng,
                         const int32_t* outlier_rows, const int32_t* outlier_cols, const void* outlier_vals,
                         const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype, void* stream,
                         const char* name) {
  using namespace w4;
  LLMC_CHECK_ARG(M >= 0 && N >= 0 && K > 0, "%s: bad shape", name);
  if (M == 0 || N == 0) return LLMC_OK;
  LLMC_CHECK_ARG(x && wq && scales && y, "%s: null pointer", name);
  LLMC_CHECK_ARG(dtype == LLMC_BF16 || dtype == LLMC_F16, "%s: dtype must be bf16 or fp16", name);
  LLMC_CHECK_ARG(sym == 0 || sym == 1, "%s: sym must be 0 or 1, got %d", name, sym);
  LLMC_CHECK_ARG(group_axis == 0 || group_axis == 1, "%s: group_axis must be 0 (K) or 1 (N), got %d", name,
                 group_axis);
  const int n_outlier_args = (outlier_rows != nullptr) + (outlier_cols != nullptr) + (outlier_vals != nullptr);
  LLMC_CHECK_ARG(n_outlier_args == 0 || n_outlier_args == 3,
                 "%s: outlier rows, cols and vals must be given together or not at all", name);
  if (group_axis == 0) {
    LLMC_CHECK_ARG(g_idx != nullptr, "%s: group_axis 0 needs g_idx", name);
    LLMC_CHECK_ARG(ng >= 1 && ng <= K, "%s: ng=%lld groups for K=%lld columns", name, (long long)ng,
                   (long long)K);
  } else {
    LLMC_CHECK_ARG(group > 0 && N % group == 0, "%s: group %lld must divide N=%lld", name, (long long)group,
                   (long long)N);
    LLMC_CHECK_ARG(K * (N / group) < (1ll << 31), "%s: qparam table [K, N/group] over 2^31 entries", name);
  }
  if (K % 64 != 0 || !aligned16(x) || !aligned16(wq) || !aligned16(y) || (g_idx && !aligned16(g_idx))) {
    set_last_error("%s: K=%lld must be a multiple of 64 and pointers 16-byte aligned", name, (long long)K);
    return LLMC_EALIGN;
  }
  ParamsRz p{};
  p.scales = scales; p.zeros = zeros;
  p.qparam_native = 0;
  p.q_transposed = 1;
  p.group = K;
  p.code_shift = sym ? 1 << (kBits - 1) : 0;
  p.o_rows = outlier_rows; p.o_cols = outlier_cols;
  p.o_vals = static_cast<const uint16_t*>(outlier_vals);
  if (group_axis == 0) {
    p.ng = static_cast<int>(ng);
    p.g_idx = g_idx;
    return launch_wNa16<kBits, kGridInt, kRzK>(x, wq, bias, y, M, N, K, dtype, stream, name, p);
  }
  p.group_n = static_cast<int>(group);
  p.ngn = static_cast<int>(N / group);
  return launch_wNa16<kBits, kGridInt, kRzN>(x, wq, bias, y, M, N, K, dtype, stream, name, p);
}

extern "C" int llmc_gemm_w2a16_rz(const void* x, const int32_t* wq, const float* scales, const float* zeros,
                                  int sym, int group_axis, int64_t group, const int32_t* g_idx, int64_t ng,
                                  const int32_t* outlier_rows, const int32_t* outlier_cols,
                                  const void* outlier_vals, const void* bias, void* y, int64_t M, int64_t N,
                                  int64_t K, int dtype, void* stream) {
  return gemm_wNa16_rz<2>(x, wq, scales, zeros, sym, group_axis, group, g_idx, ng, outlier_rows, outlier_cols,
                           outlier_vals, bias, y, M, N, K, dtype, stream, "gemm_w2a16_rz");
}

extern "C" int llmc_gemm_w3a16_rz(const void* x, const int32_t* wq, const float* scales, const float* zeros,
                                  int sym, int group_axis, int64_t group, const int32_t* g_idx, int64_t ng,
                                  const int32_t* outlier_rows, const int32_t* outlier_cols,
                                  const void* outlier_vals, const void* bias, void* y, int64_t M, int64_t N,
                                  int64_t K, int dtype, void* stream) {
  return gemm_wNa16_rz<3>(x, wq, scales, zeros, sym, group_axis, group, g_idx, ng, outlier_rows, outlier_cols,
                           outlier_vals, bias, y, M, N, K, dtype, stream, "gemm_w3a16_rz");
}

extern "C" int llmc_gemm_w4a16_rz(const void* x, const int32_t* wq, const float* scales, const float* zeros,
                                  int sym, int group_axis, int64_t group, const int32_t* g_idx, int64_t ng,
                                  const int32_t* outlier_rows, const int32_t* outlier_cols,
                                  const void* outlier_vals, const void* bias, void* y, int64_t M, int64_t N,
                                  int64_t K, int dtype, void* stream) {
  return gemm_wNa16_rz<4>(x, wq, scales, zeros, sym, group_axis, group, g_idx, ng, outlier_rows, outlier_cols,
                           outlier_vals, bias, y, M, N, K, dtype, stream, "gemm_w4a16_rz");
}

extern "C" int llmc_gemm_w8a16_rz(const void* x, const int32_t* wq, const float* scales, const float* zeros,
                                  int sym, int group_axis, int64_t group, const int32_t* g_idx, int64_t ng,
                                  const int32_t* outlier_rows, const int32_t* outlier_cols,
                                  const void* outlier_vals, const void* bias, void* y, int64_t M, int64_t N,
                                  int64_t K, int dtype, void* stream) {
  return gemm_wNa16_rz<8>(x, wq, scales, zeros, sym, group_axis, group, g_idx, ng, outlier_rows, outlier_cols,
                           outlier_vals, bias, y, M, N, K, dtype, stream, "gemm_w8a16_rz");
}

// ---- grouped (sparse-MoE) mode on packed experts ---------------------------------------------
// g: the checked qparam and g_idx pointers of every expert linear; its maps and segments are set here.
template <int kBits, int kGrid, int kMoe>
static int launch_moe_packed(const MoeLaunch<kMoe>& m, w4::MoeW4Operands& g, int qparam_dtype, int64_t group,
                             int q_transposed, int64_t ng, int n_tiles, int units, void* stream) {
  using namespace w4;
  using C = Cfg<kBits>;
  constexpr CUtensorMapSwizzle swz = kBits == 4 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUtensorMap tmA;
  if (int rc = encode_tmap_2d(&tmA, m.a, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, m.rows, m.K, m.K, BM, BK,
                              CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  if (int rc = m.encode_tmaps(g.tmP, CU_TENSOR_MAP_DATA_TYPE_INT32, 4, m.K * kBits / 32, BN, C::kWordsPerRow, swz))
    return rc;
  g.seg = m.segments();
  const bool gidx = g.g_idx[0] != nullptr;
  Params p{};
  p.M = m.rows; p.N = m.N; p.K = m.K; p.out = m.out;
  p.qparam_native = qparam_dtype != LLMC_F32 ? 1 : 0;
  p.q_transposed = q_transposed;
  p.group = gidx ? m.K : group; p.ng = static_cast<int>(ng);
  p.zero_default = static_cast<float>(1 << (kBits - 1));
  p.n_tiles_n = n_tiles;
  p.num_units = units;
  p.kb_total = static_cast<int>(m.K / BK);
  p.gn = l2_group_width(static_cast<int64_t>(BN) * m.K * kBits / 8 + 1, p.n_tiles_n);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool bf16 = m.dtype == LLMC_BF16;
  auto kernel = gidx ? (bf16 ? w4a16_gemm_kernel<true, kBits, true, kGrid, kRzOff, kPackK, kMoe>
                             : w4a16_gemm_kernel<false, kBits, true, kGrid, kRzOff, kPackK, kMoe>)
                     : (bf16 ? w4a16_gemm_kernel<true, kBits, false, kGrid, kRzOff, kPackK, kMoe>
                             : w4a16_gemm_kernel<false, kBits, false, kGrid, kRzOff, kPackK, kMoe>);
  return launch_persistent(kernel, p.num_units, C::kThreads, C::kSmemBytes, st, tmA, CUtensorMap{}, p, g);
}

// Checks and launches the grouped packed GEMM over m.rows gathered rows (the codes are m's
// weights); the *_a / *_b arrays are the qparams and g_idx of w_a / w_b.  grid: integer codes of
// `bits` (4 or 8) with optional zeros, or fp8 bytes (kGridE4M3 / kGridE5M2, bits 8, no zeros).
template <int kMoe>
static int moe_packed(const MoeLaunch<kMoe>& m, int bits, int grid, const void* const* s_a, const void* const* s_b,
                      const void* const* z_a, const void* const* z_b, const int32_t* const* g_a,
                      const int32_t* const* g_b, int qparam_dtype, int64_t group, int64_t ng, void* stream) {
  using namespace w4;
  const char* name = m.what;
  int n_tiles, units;
  if (int rc = m.check_values(BM, BN)) return rc;
  LLMC_CHECK_ARG(bits == 4 || bits == 8, "%s: bits=%d must be 4 or 8", name, bits);
  LLMC_CHECK_ARG(m.K % BK == 0, "%s: K=%lld must be a multiple of %d", name, (long long)m.K, BK);
  const int64_t ag = group < 0 ? -group : group;
  LLMC_CHECK_ARG(ag > 0 && ag % BK == 0 && m.K % ag == 0, "%s: group %lld must divide K=%lld and be a multiple of %d",
                 name, (long long)ag, (long long)m.K, BK);
  LLMC_CHECK_ARG(qparam_dtype == LLMC_F32 || qparam_dtype == m.dtype,
                 "%s: qparam_dtype must be fp32 or the activation dtype", name);
  if (int rc = m.plan(BM, BN, n_tiles, units)) return rc;
  if (m.rows == 0) return LLMC_OK;
  if (int rc = m.check_pointers()) return rc;
  LLMC_CHECK_ARG(s_a && (!m.kSwiGLU || s_b), "%s: null pointer", name);
  MoeW4Operands g{};
  const void** z = g.zeros;
  const int32_t** gi = g.g_idx;
  for (int i = 0; i < m.linears(); ++i) {
    g.scales[i] = m.linear(s_a, s_b, i);
    z[i] = m.linear(z_a, z_b, i);
    gi[i] = m.linear(g_a, g_b, i);
    LLMC_CHECK_ARG(g.scales[i], "%s: null codes or scales of expert %d", name, m.expert_of(i));
  }
  for (int i = 1; i < m.linears(); ++i) {
    const int e = m.expert_of(i);
    LLMC_CHECK_ARG((z[i] == nullptr) == (z[0] == nullptr), "%s: zeros of expert %d %s while expert 0's %s", name, e,
                   z[i] ? "given" : "null", z[0] ? "are given" : "are null");
    LLMC_CHECK_ARG((gi[i] == nullptr) == (gi[0] == nullptr), "%s: g_idx of expert %d %s while expert 0's %s", name,
                   e, gi[i] ? "given" : "null", gi[0] ? "is given" : "is null");
  }
  if (gi[0] == nullptr)
    LLMC_CHECK_ARG(ng == m.K / ag, "%s: ng=%lld, but K=%lld in groups of %lld is %lld groups", name, (long long)ng,
                   (long long)m.K, (long long)ag, (long long)(m.K / ag));
  else
    LLMC_CHECK_ARG(ng >= 1 && ng <= m.K, "%s: ng=%lld groups for K=%lld columns", name, (long long)ng,
                   (long long)m.K);
  for (int i = 0; i < m.linears(); ++i) {
    if (gi[i] && !aligned16(gi[i])) {
      set_last_error("%s: g_idx of expert %d not 16-byte aligned", name, m.expert_of(i));
      return LLMC_EALIGN;
    }
  }
  const int qt = group < 0 ? 1 : 0;
  if (grid == kGridE4M3) return launch_moe_packed<8, kGridE4M3>(m, g, qparam_dtype, ag, qt, ng, n_tiles, units, stream);
  if (grid == kGridE5M2) return launch_moe_packed<8, kGridE5M2>(m, g, qparam_dtype, ag, qt, ng, n_tiles, units, stream);
  if (bits == 4) return launch_moe_packed<4, kGridInt>(m, g, qparam_dtype, ag, qt, ng, n_tiles, units, stream);
  return launch_moe_packed<8, kGridInt>(m, g, qparam_dtype, ag, qt, ng, n_tiles, units, stream);
}

// The packed codes arrays, as MoeLaunch's untyped per-expert weight arrays.
static const void* const* codes(const int32_t* const* wq) { return reinterpret_cast<const void* const*>(wq); }

extern "C" int llmc_moe_gemm_packed_swiglu(const void* xp, int bits, const int32_t* const* wq1,
                                           const int32_t* const* wq3, const void* const* s1, const void* const* s3,
                                           const void* const* z1, const void* const* z3, const int32_t* const* gidx1,
                                           const int32_t* const* gidx3, int qparam_dtype, int64_t group, int64_t ng,
                                           const int32_t* offsets, void* act, int64_t rows, int64_t inter,
                                           int64_t K, int64_t n_experts, int dtype, void* stream) {
  return moe_packed<kMoeSwiGLU>({"moe_gemm_packed_swiglu", xp, act, codes(wq1), codes(wq3), offsets, nullptr, rows,
                                 inter, K, n_experts, dtype, "codes or scales"},
                                bits, w4::kGridInt, s1, s3, z1, z3, gidx1, gidx3, qparam_dtype, group, ng, stream);
}

extern "C" int llmc_moe_gemm_packed_down(const void* act, int bits, const int32_t* const* wq2,
                                         const void* const* s2, const void* const* z2, const int32_t* const* gidx2,
                                         int qparam_dtype, int64_t group, int64_t ng, const int32_t* offsets,
                                         const void* w_route, void* y, int64_t rows, int64_t N, int64_t inter,
                                         int64_t n_experts, int dtype, void* stream) {
  return moe_packed<kMoeDown>({"moe_gemm_packed_down", act, y, codes(wq2), nullptr, offsets, w_route, rows, N, inter,
                               n_experts, dtype, "codes or scales"},
                              bits, w4::kGridInt, s2, nullptr, z2, nullptr, gidx2, nullptr, qparam_dtype, group, ng,
                              stream);
}

// FP8 experts: the fp8 bytes [N_lin, K] of each expert linear viewed as int32 [N_lin, K/4], as
// llmc_gemm_fp8a16; no zero-points.  e5m2 is checked with the other scalars, before rows == 0.
static int fp8_grid(int e5m2) { return e5m2 == 1 ? w4::kGridE5M2 : w4::kGridE4M3; }

extern "C" int llmc_moe_gemm_fp8a16_swiglu(const void* xp, int e5m2, const int32_t* const* wq1,
                                           const int32_t* const* wq3, const void* const* s1, const void* const* s3,
                                           const int32_t* const* gidx1, const int32_t* const* gidx3,
                                           int qparam_dtype, int64_t group, int64_t ng, const int32_t* offsets,
                                           void* act, int64_t rows, int64_t inter, int64_t K, int64_t n_experts,
                                           int dtype, void* stream) {
  const char* name = "moe_gemm_fp8a16_swiglu";
  LLMC_CHECK_ARG(e5m2 == 0 || e5m2 == 1, "%s: e5m2 must be 0 (e4m3) or 1 (e5m2), got %d", name, e5m2);
  return moe_packed<kMoeSwiGLU>({name, xp, act, codes(wq1), codes(wq3), offsets, nullptr, rows, inter, K, n_experts,
                                 dtype, "codes or scales"},
                                8, fp8_grid(e5m2), s1, s3, nullptr, nullptr, gidx1, gidx3, qparam_dtype, group, ng,
                                stream);
}

extern "C" int llmc_moe_gemm_fp8a16_down(const void* act, int e5m2, const int32_t* const* wq2,
                                         const void* const* s2, const int32_t* const* gidx2, int qparam_dtype,
                                         int64_t group, int64_t ng, const int32_t* offsets, const void* w_route,
                                         void* y, int64_t rows, int64_t N, int64_t inter, int64_t n_experts,
                                         int dtype, void* stream) {
  const char* name = "moe_gemm_fp8a16_down";
  LLMC_CHECK_ARG(e5m2 == 0 || e5m2 == 1, "%s: e5m2 must be 0 (e4m3) or 1 (e5m2), got %d", name, e5m2);
  return moe_packed<kMoeDown>({name, act, y, codes(wq2), nullptr, offsets, w_route, rows, N, inter, n_experts, dtype,
                               "codes or scales"},
                              8, fp8_grid(e5m2), s2, nullptr, nullptr, nullptr, gidx2, nullptr, qparam_dtype, group,
                              ng, stream);
}
