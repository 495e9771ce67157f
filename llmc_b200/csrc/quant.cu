// quant.cu — K1/K2: fused group min/max -> (scale, zero) -> quantise (-> pack | dequantise).
//
// Replaces the eager chain IntegerQuantizer.get_tensor_qparams / quant / dequant /
// real_quant_weight_* (llmc/compression/quantization/quant.py:132-143, 545-559, 690-717,
// 833-953) and VllmRealQuantLinear.pack (module_utils.py:836-862).
//
// HBM-bound integer/byte work: one pass over W with 16-byte loads, qparams in registers,
// 4..32-byte stores.  Bit-exactness against torch comes from reproducing torch's rounding
// points ("T-faithful", common.cuh) — see DESIGN.md §numerics.
#include <type_traits>

#include "common.cuh"
#include "quant_math.cuh"

namespace llmc {

struct QuantArgs {
  const void* w;
  int64_t rows, cols, ld;
  int64_t group, ng;       // elements per group, groups per row
  float qmin, qmax;
  int sym;
  int bit;
  void* scales;            // [rows*ng] DT  (dynamic: out)
  void* zeros;             // [rows*ng] DT  (dynamic: out, asym only)
  int out_mode;
  void* out;
  int64_t ld_out;          // QDQ row stride (elements)
  int out_dtype;
  int64_t packed_cols;     // PACK_VLLM: words per row
  const void* col_scale;   // optional [cols] DT: w' = rT(w * s[c]) first (AWQ, awq.py:39-46)
};

// x / s, correctly rounded to fp32 (then the caller rounds to T): the reciprocal divider for
// 16-bit operands, the IEEE divide for fp32 (quant_math.cuh).
template <int DT>
using Divider = std::conditional_t<DT == LLMC_F32, IeeeDiv, RecipDiv>;

// Emit 8 consecutive codes/values of row r starting at column c (c % 8 == 0).
template <int DT>
__device__ __forceinline__ void emit8(const QuantArgs& a, int64_t r, int64_t c,
                                      const float (&q)[8], float s, float z) {
  switch (a.out_mode) {
    case LLMC_OUT_QDQ: {
      float y[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) y[i] = dequant<DType<DT>>(q[i], s, z);
      store8_as(a.out_dtype, a.out, r * a.ld_out + c, y);
      break;
    }
    case LLMC_OUT_CODES_I8:
    case LLMC_OUT_CODES_U8: {
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        lo |= (static_cast<uint32_t>(static_cast<int>(q[i])) & 0xffu) << (8 * i);
        hi |= (static_cast<uint32_t>(static_cast<int>(q[i + 4])) & 0xffu) << (8 * i);
      }
      *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(a.out) + r * a.cols + c) =
          make_uint2(lo, hi);
      break;
    }
    case LLMC_OUT_CODES_I32: {
      int4* p = reinterpret_cast<int4*>(reinterpret_cast<int32_t*>(a.out) + r * a.cols + c);
      p[0] = make_int4((int)q[0], (int)q[1], (int)q[2], (int)q[3]);
      p[1] = make_int4((int)q[4], (int)q[5], (int)q[6], (int)q[7]);
      break;
    }
    case LLMC_OUT_PACK_VLLM: {
      // module_utils.py:842-856: (code + 2^(bit-1)).to(uint8) << bit*i, OR-ed.
      const int off = 1 << (a.bit - 1);
      int32_t* o = reinterpret_cast<int32_t*>(a.out) + r * a.packed_cols;
      if (a.bit == 4) {
        uint32_t wd = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          wd |= (static_cast<uint32_t>(static_cast<int>(q[i]) + off) & 0xffu) << (4 * i);
        o[c >> 3] = static_cast<int32_t>(wd);
      } else {  // bit == 8
        uint32_t lo = 0, hi = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          lo |= (static_cast<uint32_t>(static_cast<int>(q[i]) + off) & 0xffu) << (8 * i);
          hi |= (static_cast<uint32_t>(static_cast<int>(q[i + 4]) + off) & 0xffu) << (8 * i);
        }
        *reinterpret_cast<uint2*>(o + (c >> 2)) = make_uint2(lo, hi);
      }
      break;
    }
    default: break;
  }
}

// ---- fast path: a sub-warp of LPG lanes owns one group; CH 8-element chunks per lane -----
template <int DT, int CH>
__global__ void __launch_bounds__(256)
quant_dynamic_warp_kernel(QuantArgs a, int lpg, int64_t total_groups) {
  using D = DType<DT>;
  const int lane = threadIdx.x & 31;
  const int sub = lane & (lpg - 1);
  const int gpw = 32 / lpg;                       // groups per warp
  const int64_t warp_global = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t warp_stride = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  const int chunks = static_cast<int>(a.group >> 3);

  for (int64_t gbase = warp_global * gpw; gbase < total_groups; gbase += warp_stride * gpw) {
    const int64_t g = gbase + lane / lpg;
    const bool active = g < total_groups;
    // 32-bit divide (the launcher guarantees total_groups < 2^31); a 64-bit one is ~100 instrs
    const uint32_t r32 = active ? static_cast<uint32_t>(g) / static_cast<uint32_t>(a.ng) : 0u;
    const int64_t r = r32;
    const int64_t j = active ? g - r * a.ng : 0;
    const int64_t col0 = j * a.group;
    float v[CH][8];
    float mn = INFINITY, mx = -INFINITY;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int ch = c * lpg + sub;
      if (active && ch < chunks) {
        load8<DT>(a.w, r * a.ld + col0 + ch * 8, v[c]);
        if (a.col_scale != nullptr) {
          float cs[8];
          load8<DT>(a.col_scale, col0 + ch * 8, cs);
#pragma unroll
          for (int i = 0; i < 8; ++i) v[c][i] = D::rT(fmul_rn(v[c][i], cs[i]));
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) { mn = fminf(mn, v[c][i]); mx = fmaxf(mx, v[c][i]); }
      }
    }
    mn = warp_min(mn, lpg);
    mx = warp_max(mx, lpg);
    float s, z;
    qparams<DType<DT>>(mn, mx, a.sym, 1, a.qmin, a.qmax, s, z);
    if (active && sub == 0) {
      D::store(a.scales, g, s);
      if (!a.sym && a.zeros) D::store(a.zeros, g, z);
    }
    if (a.out_mode == LLMC_OUT_NONE) continue;
    const Divider<DT> div{s};
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int ch = c * lpg + sub;
      if (active && ch < chunks) {
        float q[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) q[i] = quant_code<DType<DT>>(v[c][i], div, z, a.qmin, a.qmax);
        emit8<DT>(a, r, col0 + ch * 8, q, s, z);
      }
    }
  }
}

__device__ __forceinline__ void block_minmax(float& mn, float& mx) {
  __shared__ float smn[32], smx[32];
  mn = warp_min(mn);
  mx = warp_max(mx);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  if (l == 0) { smn[w] = mn; smx[w] = mx; }
  __syncthreads();
  mn = (l < nw) ? smn[l] : INFINITY;
  mx = (l < nw) ? smx[l] : -INFINITY;
  mn = warp_min(mn);
  mx = warp_max(mx);
  __syncthreads();
}

// ---- large groups (per_channel / per_token rows): one CTA per group, second pass from L2 ---
template <int DT>
__global__ void __launch_bounds__(256)
quant_dynamic_block_kernel(QuantArgs a, int64_t total_groups) {
  using D = DType<DT>;
  const int chunks = static_cast<int>(a.group >> 3);
  for (int64_t g = blockIdx.x; g < total_groups; g += gridDim.x) {
    const int64_t r = g / a.ng, j = g - r * a.ng;
    const int64_t base = r * a.ld + j * a.group;
    float mn = INFINITY, mx = -INFINITY;
    for (int ch = threadIdx.x; ch < chunks; ch += blockDim.x) {
      float v[8];
      load8<DT>(a.w, base + ch * 8, v);
      if (a.col_scale != nullptr) {
        float cs[8];
        load8<DT>(a.col_scale, j * a.group + ch * 8, cs);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = D::rT(fmul_rn(v[i], cs[i]));
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) { mn = fminf(mn, v[i]); mx = fmaxf(mx, v[i]); }
    }
    block_minmax(mn, mx);
    float s, z;
    qparams<DType<DT>>(mn, mx, a.sym, 1, a.qmin, a.qmax, s, z);
    if (threadIdx.x == 0) {
      D::store(a.scales, g, s);
      if (!a.sym && a.zeros) D::store(a.zeros, g, z);
    }
    if (a.out_mode == LLMC_OUT_NONE) continue;
    const Divider<DT> div{s};
    for (int ch = threadIdx.x; ch < chunks; ch += blockDim.x) {
      float v[8], q[8];
      load8<DT>(a.w, base + ch * 8, v);
      if (a.col_scale != nullptr) {
        float cs[8];
        load8<DT>(a.col_scale, j * a.group + ch * 8, cs);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = D::rT(fmul_rn(v[i], cs[i]));
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) q[i] = quant_code<DType<DT>>(v[i], div, z, a.qmin, a.qmax);
      emit8<DT>(a, r, j * a.group + ch * 8, q, s, z);
    }
  }
}

// ---- generic qparams (any group size / alignment): one CTA per group, scalar loads --------
template <int DT>
__global__ void __launch_bounds__(256)
qparams_generic_kernel(QuantArgs a, int64_t total_groups) {
  using D = DType<DT>;
  for (int64_t g = blockIdx.x; g < total_groups; g += gridDim.x) {
    const int64_t r = g / a.ng, j = g - r * a.ng;
    const int64_t base = r * a.ld + j * a.group;
    float mn = INFINITY, mx = -INFINITY;
    for (int64_t i = threadIdx.x; i < a.group; i += blockDim.x) {
      float v = D::load(a.w, base + i);
      mn = fminf(mn, v);
      mx = fmaxf(mx, v);
    }
    block_minmax(mn, mx);
    float s, z;
    qparams<DType<DT>>(mn, mx, a.sym, 1, a.qmin, a.qmax, s, z);
    if (threadIdx.x == 0) {
      D::store(a.scales, g, s);
      if (!a.sym && a.zeros) D::store(a.zeros, g, z);
    }
  }
}

// ---- static quantisation: qparams given ----------------------------------------------------
struct StaticArgs {
  const void* w;
  int64_t rows, cols, ld;
  const void* scales;
  const void* zeros;       // may be null
  int64_t q_row_stride;    // ng, or 0 for per_tensor
  int64_t group;
  const int32_t* gmap;     // optional column -> group index
  float qmin, qmax;
  int bit;
  int out_mode;
  void* out;
  int64_t ld_out;
  int out_dtype;
  int64_t packed_cols;
  int unit;                // elements per thread (8, or 32/bit for PACK with odd widths)
  int zp_inside;           // round_zp False: zero-point added before rounding, scale clamped at 1e-9
};

template <int WT>
__device__ __forceinline__ float load_w(const void* p, int64_t i) { return DType<WT>::load(p, i); }

// CT = rounding dtype of every op (normally promote(w dtype, qparam dtype)); WT = weight storage
// dtype; QT = qparam storage dtype.  CT == WT != QT == fp32 is torch's CPU "scalar operand"
// path: a 0-dim fp32 scale keeps its fp32 value while results round to the tensor dtype.
// The reciprocal-based divide is only exact when x and s both have <= 11 significant bits.
#define LLMC_DV ((WT == QT && WT == CT) ? CT : LLMC_F32)
// QT (qparam storage) == CT unless CT is fp32 and qparams are 16-bit, handled by QT.
template <int CT, int WT, int QT>
__global__ void __launch_bounds__(256)
quant_static_kernel(StaticArgs a) {
  const int64_t units_per_row = (a.cols + a.unit - 1) / a.unit;
  const int64_t total = a.rows * units_per_row;
  for (int64_t u = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < total;
       u += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = u / units_per_row;
    const int64_t c0 = (u - r * units_per_row) * a.unit;
    uint32_t word = 0;
    const int off = 1 << (a.bit - 1);
    int64_t last_g = -1;
    float s = 1.f, z = 0.f;
    Divider<LLMC_DV> div{1.f};
    for (int i = 0; i < a.unit; ++i) {
      const int64_t c = c0 + i;
      if (c >= a.cols) break;
      const int64_t g = a.gmap ? a.gmap[c] : c / a.group;
      if (g != last_g) {
        s = DType<QT>::load(a.scales, r * a.q_row_stride + g);
        z = a.zeros ? DType<QT>::load(a.zeros, r * a.q_row_stride + g) : 0.f;
        div = Divider<LLMC_DV>{a.zp_inside ? fmaxf(s, 1e-9f) : s};
        last_g = g;
      }
      const float x = load_w<WT>(a.w, r * a.ld + c);
      const float q = a.zp_inside ? quant_code_zp<DType<CT>>(x, div, z, a.qmin, a.qmax)
                                  : quant_code<DType<CT>>(x, div, z, a.qmin, a.qmax);
      switch (a.out_mode) {
        case LLMC_OUT_QDQ: {
          store_as(a.out_dtype, a.out, r * a.ld_out + c, dequant<DType<CT>>(q, s, z));
          break;
        }
        case LLMC_OUT_CODES_I8:
        case LLMC_OUT_CODES_U8:
          reinterpret_cast<uint8_t*>(a.out)[r * a.cols + c] =
              static_cast<uint8_t>(static_cast<int>(q));
          break;
        case LLMC_OUT_CODES_I32:
          reinterpret_cast<int32_t*>(a.out)[r * a.cols + c] = static_cast<int>(q);
          break;
        case LLMC_OUT_PACK_VLLM:
          word |= (static_cast<uint32_t>(static_cast<int>(q) + off) & 0xffu) << (a.bit * i);
          break;
        default: break;
      }
    }
    if (a.out_mode == LLMC_OUT_PACK_VLLM)
      reinterpret_cast<int32_t*>(a.out)[r * a.packed_cols + c0 / a.unit] =
          static_cast<int32_t>(word);
  }
}

// vectorised static path: 8 aligned columns per thread, one group per 8 columns unless gmap.
template <int CT, int WT, int QT>
__global__ void __launch_bounds__(256)
quant_static_vec8_kernel(StaticArgs a, QuantArgs e) {
  const int64_t units_per_row = a.cols >> 3;
  const int64_t total = a.rows * units_per_row;
  for (int64_t u = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < total;
       u += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = u / units_per_row;
    const int64_t c0 = (u - r * units_per_row) << 3;
    float x[8], q[8];
    load8<WT>(a.w, r * a.ld + c0, x);
    if (a.gmap == nullptr) {
      const int64_t g = c0 / a.group;
      const float s = DType<QT>::load(a.scales, r * a.q_row_stride + g);
      const float z = a.zeros ? DType<QT>::load(a.zeros, r * a.q_row_stride + g) : 0.f;
      const Divider<LLMC_DV> div{a.zp_inside ? fmaxf(s, 1e-9f) : s};
#pragma unroll
      for (int i = 0; i < 8; ++i)
        q[i] = a.zp_inside ? quant_code_zp<DType<CT>>(x[i], div, z, a.qmin, a.qmax)
                           : quant_code<DType<CT>>(x[i], div, z, a.qmin, a.qmax);
      emit8<CT>(e, r, c0, q, s, z);
    } else {
      // act-order gather: every column may belong to a different group; only QDQ/CODES.
      float y[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int64_t g = a.gmap[c0 + i];
        const float s = DType<QT>::load(a.scales, r * a.q_row_stride + g);
        const float z = a.zeros ? DType<QT>::load(a.zeros, r * a.q_row_stride + g) : 0.f;
        const Divider<LLMC_DV> div{a.zp_inside ? fmaxf(s, 1e-9f) : s};
        q[i] = a.zp_inside ? quant_code_zp<DType<CT>>(x[i], div, z, a.qmin, a.qmax)
                           : quant_code<DType<CT>>(x[i], div, z, a.qmin, a.qmax);
        y[i] = dequant<DType<CT>>(q[i], s, z);
      }
      if (a.out_mode == LLMC_OUT_QDQ) {
        store8_as(a.out_dtype, a.out, r * a.ld_out + c0, y);
      } else {
        emit8<CT>(e, r, c0, q, 1.f, 0.f);
      }
    }
  }
}

// ---- per_tensor min / max ---------------------------------------------------------------------
template <int DT>
__global__ void __launch_bounds__(256) minmax_stage1(const void* w, int64_t n, float* ws) {
  float mn = INFINITY, mx = -INFINITY;
  const int64_t n8 = n >> 3;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float v[8];
    load8<DT>(w, i << 3, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) { mn = fminf(mn, v[k]); mx = fmaxf(mx, v[k]); }
  }
  if (blockIdx.x == 0)
    for (int64_t i = (n8 << 3) + threadIdx.x; i < n; i += blockDim.x) {
      float v = DType<DT>::load(w, i);
      mn = fminf(mn, v);
      mx = fmaxf(mx, v);
    }
  block_minmax(mn, mx);
  if (threadIdx.x == 0) { ws[blockIdx.x] = mn; ws[1024 + blockIdx.x] = mx; }
}

template <int DT>
__global__ void __launch_bounds__(256) minmax_stage2(const float* ws, int nblocks, void* mm) {
  float mn = INFINITY, mx = -INFINITY;
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) {
    mn = fminf(mn, ws[i]);
    mx = fmaxf(mx, ws[1024 + i]);
  }
  block_minmax(mn, mx);
  if (threadIdx.x == 0) { DType<DT>::store(mm, 0, mn); DType<DT>::store(mm, 1, mx); }
}

static int promote(int a, int b) { return a == b ? a : LLMC_F32; }

// ---- round-2 fast path: one THREAD per group, tile staged through shared memory --------------
// The warp kernel above spends ~20 instructions per element (index arithmetic, runtime out_mode
// switch, cross-lane min/max) and was issue-bound at 0.29 of the HBM roof.  Here a CTA of 128
// threads copies 128 consecutive groups (dense rows => one contiguous 16/32 KB span) into shared
// memory with 16-byte cp.async (swizzled so that the per-thread 16-byte reads of "my group" are
// conflict free), double buffered; each thread then owns one whole group in registers: min/max
// on PACKED half2/bf16x2 (1 instruction per element pair and statistic), qparams once, and the
// exact T-faithful quantise chain per element with the output mode fixed at compile time.
namespace qf {

constexpr int TG = 128;                    // groups per tile == threads per CTA
enum { M_NONE = 0, M_PACK = 1, M_QDQ = 2, M_CODES8 = 3 };

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

template <int DT>
__device__ __forceinline__ uint32_t min2(uint32_t a, uint32_t b) {
  if constexpr (DT == LLMC_BF16) {
    const __nv_bfloat162 r = __hmin2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b));
    return *reinterpret_cast<const uint32_t*>(&r);
  } else {
    const __half2 r = __hmin2(*reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&b));
    return *reinterpret_cast<const uint32_t*>(&r);
  }
}
template <int DT>
__device__ __forceinline__ uint32_t max2(uint32_t a, uint32_t b) {
  if constexpr (DT == LLMC_BF16) {
    const __nv_bfloat162 r = __hmax2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b));
    return *reinterpret_cast<const uint32_t*>(&r);
  } else {
    const __half2 r = __hmax2(*reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&b));
    return *reinterpret_cast<const uint32_t*>(&r);
  }
}
template <int DT>
__device__ __forceinline__ float lo_f(uint32_t w) {
  if constexpr (DT == LLMC_BF16) return __uint_as_float(w << 16);
  else return __half2float(__ushort_as_half(static_cast<uint16_t>(w & 0xffffu)));
}
template <int DT>
__device__ __forceinline__ float hi_f(uint32_t w) {
  if constexpr (DT == LLMC_BF16) return __uint_as_float(w & 0xffff0000u);
  else return __half2float(__ushort_as_half(static_cast<uint16_t>(w >> 16)));
}
template <int DT>
__device__ __forceinline__ uint32_t pack_T(float a, float b) {
  if constexpr (DT == LLMC_BF16) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  } else {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  }
}

// The per-chunk tail shared by the two fast kernels: 8 packed T values -> QDQ chunk | packed codes.
//   v = yb + Ce does rint, + zero and the storage offset in one float add (see the kernel comment).
template <int DT, int MODE, int BITS>
__device__ __forceinline__ void fast_tail(const uint4& xin, const Divider<DT>& div, float s, float Ce,
                                          float vlo, float vhi, uint32_t ob, int sym, uint4& out) {
  constexpr uint32_t kMb = 0x4B400000u;
  const uint32_t wd[4] = {xin.x, xin.y, xin.z, xin.w};
  float v[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    // rT(x / s): exact quotient, then ONE rounding to T for the pair (cvt.rn.{bf16,f16}x2)
    const uint32_t yb = pack_T<DT>(div(lo_f<DT>(wd[i])), div(hi_f<DT>(wd[i])));
    v[2 * i] = fminf(fmaxf(fadd_rn(lo_f<DT>(yb), Ce), vlo), vhi);
    v[2 * i + 1] = fminf(fmaxf(fadd_rn(hi_f<DT>(yb), Ce), vlo), vhi);
  }
  if constexpr (MODE == M_QDQ) {
    // (q - z) = v - Ce exactly; * s rounds once to T (quant.py:710-712)
    out.x = pack_T<DT>(fmul_rn(v[0] - Ce, s), fmul_rn(v[1] - Ce, s));
    out.y = pack_T<DT>(fmul_rn(v[2] - Ce, s), fmul_rn(v[3] - Ce, s));
    out.z = pack_T<DT>(fmul_rn(v[4] - Ce, s), fmul_rn(v[5] - Ce, s));
    out.w = pack_T<DT>(fmul_rn(v[6] - Ce, s), fmul_rn(v[7] - Ce, s));
  } else if constexpr (MODE == M_PACK && BITS == 4) {
    // sym: nibble_i = code_i + 8 in [0, 15]; word = sum nibble_i * 16^i.
    // asym: the codes are packed plain (C) and the reference's (code + 8) << 4i, OR-ed
    // (module_utils.py:842-856) is applied on the word: the low nibble of code + 8 is code ^ 8 and
    // its carry (code >= 8) lands on bit 0 of the next field, the last one falling off the word.
    uint32_t w4 = __float_as_uint(v[7]);
#pragma unroll
    for (int i = 6; i >= 0; --i) w4 = w4 * 16u + __float_as_uint(v[i]);
    w4 = w4 - kMb * 0x11111111u + ob * 0x11111111u;
    out.x = sym ? w4 : ((w4 ^ 0x88888888u) | ((w4 & 0x88888888u) << 1));
  } else {
    uint32_t lo = __float_as_uint(v[3]), hi = __float_as_uint(v[7]);
#pragma unroll
    for (int i = 2; i >= 0; --i) {
      lo = lo * 256u + __float_as_uint(v[i]);
      hi = hi * 256u + __float_as_uint(v[4 + i]);
    }
    const uint32_t fix = ob * 0x01010101u - kMb * 0x01010101u;
    lo += fix;
    hi += fix;
    // CODES8 signed: offset-binary -> int8; PACK unsigned: (code + 128).to(uint8) = code ^ 0x80
    if ((MODE == M_CODES8 && sym) || (MODE == M_PACK && !sym)) { lo ^= 0x80808080u; hi ^= 0x80808080u; }
    out.x = lo;
    out.y = hi;
  }
}

// Per-group constants of fast_tail.
template <int MODE, int BITS>
__device__ __forceinline__ void fast_consts(float z, float qmin, float qmax, int sym, float& Ce,
                                            float& vlo, float& vhi, uint32_t& ob) {
  constexpr float kM = 12582912.0f;                   // 1.5 * 2^23 = 0x4B400000
  constexpr float OFFE = (MODE == M_PACK || MODE == M_CODES8) ? static_cast<float>(1 << (BITS - 1)) : 0.f;
  const float zo = static_cast<float>(static_cast<int>(z) & 1);
  // offset-binary internally for signed codes, plain for unsigned (asymmetric) ones
  const float offe = sym ? OFFE : 0.f;
  Ce = kM + (z - zo) + offe;
  vlo = qmin + kM - zo + offe;
  vhi = qmax + kM - zo + offe;
  ob = static_cast<uint32_t>(zo);
}

template <int DT, int G, int MODE, int BITS>
__global__ void __launch_bounds__(TG)
quant_group_fast_kernel(QuantArgs a, int64_t total_groups) {
  constexpr int CPG = G / 8;               // 16-byte chunks per group
  constexpr int RB = G * 2;                // bytes per group row
  constexpr int TILE = TG * RB;
  extern __shared__ __align__(16) uint8_t qsm[];
  const int t = threadIdx.x;
  const int64_t n_tiles = (total_groups + TG - 1) / TG;
  const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(a.w);

  auto prefetch = [&](int64_t tile, int buf) {
    const int64_t g0 = tile * TG;
    const int64_t nvalid = (total_groups - g0) < TG ? (total_groups - g0) : TG;
    const int nchunks = static_cast<int>(nvalid) * CPG;
    uint8_t* dst = qsm + buf * TILE;
    const uint8_t* src = wsrc + g0 * RB;
#pragma unroll
    for (int k = 0; k < CPG; ++k) {
      const int q = k * TG + t;
      if (q < nchunks) {
        const int row = q / CPG, c = q % CPG;
        cp_async16(dst + row * RB + ((c ^ (row & (CPG - 1))) << 4), src + static_cast<int64_t>(q) * 16);
      }
    }
    cp_async_commit();
  };

  int64_t tile = blockIdx.x;
  if (tile >= n_tiles) return;
  prefetch(tile, 0);
  int buf = 0;
  for (; tile < n_tiles; tile += gridDim.x, buf ^= 1) {
    const int64_t next = tile + gridDim.x;
    if (next < n_tiles) { prefetch(next, buf ^ 1); cp_async_wait<1>(); }
    else cp_async_wait<0>();
    __syncthreads();
    const int64_t g0 = tile * TG;
    const int64_t g = g0 + t;
    uint8_t* tb = qsm + buf * TILE;
    if (g < total_groups) {
      uint4 x[CPG];
#pragma unroll
      for (int c = 0; c < CPG; ++c)
        x[c] = *reinterpret_cast<const uint4*>(tb + t * RB + ((c ^ (t & (CPG - 1))) << 4));
      if (a.col_scale != nullptr) {
        // AWQ: quantise rT(w * s[c]) (awq.py:39-46, 147-164) — one multiply and one rounding per
        // element, the scaled values replace the loaded ones for everything that follows
        const uint4* cs = reinterpret_cast<const uint4*>(
            reinterpret_cast<const uint16_t*>(a.col_scale) + (g % a.ng) * G);
#pragma unroll
        for (int c = 0; c < CPG; ++c) {
          const uint4 sv = __ldg(cs + c);
          x[c].x = pack_T<DT>(fmul_rn(lo_f<DT>(x[c].x), lo_f<DT>(sv.x)), fmul_rn(hi_f<DT>(x[c].x), hi_f<DT>(sv.x)));
          x[c].y = pack_T<DT>(fmul_rn(lo_f<DT>(x[c].y), lo_f<DT>(sv.y)), fmul_rn(hi_f<DT>(x[c].y), hi_f<DT>(sv.y)));
          x[c].z = pack_T<DT>(fmul_rn(lo_f<DT>(x[c].z), lo_f<DT>(sv.z)), fmul_rn(hi_f<DT>(x[c].z), hi_f<DT>(sv.z)));
          x[c].w = pack_T<DT>(fmul_rn(lo_f<DT>(x[c].w), lo_f<DT>(sv.w)), fmul_rn(hi_f<DT>(x[c].w), hi_f<DT>(sv.w)));
        }
      }
      uint32_t mn2 = x[0].x, mx2 = x[0].x;
#pragma unroll
      for (int c = 0; c < CPG; ++c) {
        mn2 = min2<DT>(min2<DT>(mn2, x[c].x), min2<DT>(x[c].y, min2<DT>(x[c].z, x[c].w)));
        mx2 = max2<DT>(max2<DT>(mx2, x[c].x), max2<DT>(x[c].y, max2<DT>(x[c].z, x[c].w)));
      }
      const float mn = fminf(lo_f<DT>(mn2), hi_f<DT>(mn2));
      const float mx = fmaxf(lo_f<DT>(mx2), hi_f<DT>(mx2));
      float s, z;
      qparams<DType<DT>>(mn, mx, a.sym, 1, a.qmin, a.qmax, s, z);
      DType<DT>::store(a.scales, g, s);
      if (!a.sym && a.zeros) DType<DT>::store(a.zeros, g, z);
      if constexpr (MODE != M_NONE) {
        // Tail of the chain after the exact division, with the rounding done by ONE float add:
        //   v = yb + Ce,  Ce = 1.5*2^23 + (z - o) + OFFE  (o = parity of z, OFFE = even storage offset)
        // Ce is an even integer in [2^23, 2^24), so RN-even of the sum is rint(yb) + Ce (ties keep
        // their parity) and rint(yb) + z = v - 1.5*2^23 + o - OFFE.  Clamping v against the shifted
        // bounds is clamp(rint + z, qmin, qmax); the float BITS of the clamped v are
        // 0x4B400000 + (code + OFFE - o), which the integer packing below consumes directly
        // (multiply-add chain, the constant parts subtracted once per word).
        const Divider<DT> div{s};
        float Ce, vlo, vhi;
        uint32_t ob;
        fast_consts<MODE, BITS>(z, a.qmin, a.qmax, a.sym, Ce, vlo, vhi, ob);
#pragma unroll
        for (int c = 0; c < CPG; ++c) {
          uint4 o;
          fast_tail<DT, MODE, BITS>(x[c], div, s, Ce, vlo, vhi, ob, a.sym, o);
          if constexpr (MODE == M_QDQ) {
            *reinterpret_cast<uint4*>(tb + t * RB + ((c ^ (t & (CPG - 1))) << 4)) = o;
          } else {
            x[c] = o;                       // packed word(s) in .x (4-bit) or .x/.y (8-bit)
          }
        }
        if constexpr (MODE == M_PACK && BITS == 4) {
          uint4* o = reinterpret_cast<uint4*>(reinterpret_cast<int32_t*>(a.out) + g * (G / 8));
#pragma unroll
          for (int c = 0; c < CPG; c += 4) o[c / 4] = make_uint4(x[c].x, x[c + 1].x, x[c + 2].x, x[c + 3].x);
        } else if constexpr (MODE == M_PACK || MODE == M_CODES8) {
          uint4* o = reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(a.out) + g * G);
#pragma unroll
          for (int c = 0; c < CPG; c += 2) o[c / 2] = make_uint4(x[c].x, x[c].y, x[c + 1].x, x[c + 1].y);
        }
      }
    }
    if constexpr (MODE == M_QDQ) {
      __syncthreads();
      const int64_t nvalid = (total_groups - g0) < TG ? (total_groups - g0) : TG;
      const int nchunks = static_cast<int>(nvalid) * CPG;
      uint8_t* dst = reinterpret_cast<uint8_t*>(a.out) + g0 * RB;
#pragma unroll
      for (int k = 0; k < CPG; ++k) {
        const int q = k * TG + t;
        if (q < nchunks) {
          const int row = q / CPG, c = q % CPG;
          *reinterpret_cast<uint4*>(dst + static_cast<int64_t>(q) * 16) =
              *reinterpret_cast<const uint4*>(tb + row * RB + ((c ^ (row & (CPG - 1))) << 4));
        }
      }
    }
    __syncthreads();
  }
}

// ---- per_channel / per_token rows (one group = one row, 512 <= cols <= 8192): a CTA of 256
// threads owns a row, every thread keeps <= 4 16-byte chunks in registers (ONE pass over the
// row instead of the block kernel's second read), packed min/max + one block reduction, then the
// same fast tail.  Coalesced 16-byte loads and 8/16-byte stores; no shared-memory staging needed.
template <int DT, int MODE, int BITS, int CH>
__global__ void __launch_bounds__(256, CH == 4 ? 4 : 6)
quant_row_fast_kernel(QuantArgs a) {
  __shared__ uint32_t smn[8], smx[8];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int chunks = static_cast<int>(a.cols >> 3);
  auto load_row = [&](int64_t r, uint4 (&x)[CH]) {
    const uint4* src = reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(a.w) + r * a.ld);
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int ch = c * 256 + t;
      if (ch < chunks) x[c] = __ldg(src + ch);
    }
  };
  int64_t r = blockIdx.x;
  if (r >= a.rows) return;
  uint4 x[CH] = {};
  load_row(r, x);
  for (; r < a.rows; r += gridDim.x) {
    // the next row's loads stay in flight across this row's reduction, tail and stores
    uint4 xn[CH] = {};
    if (r + gridDim.x < a.rows) load_row(r + gridDim.x, xn);
    uint32_t mn2 = 0, mx2 = 0;
    bool first = true;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int ch = c * 256 + t;
      if (ch < chunks) {
        const uint32_t lo = min2<DT>(min2<DT>(x[c].x, x[c].y), min2<DT>(x[c].z, x[c].w));
        const uint32_t hi = max2<DT>(max2<DT>(x[c].x, x[c].y), max2<DT>(x[c].z, x[c].w));
        mn2 = first ? lo : min2<DT>(mn2, lo);
        mx2 = first ? hi : max2<DT>(mx2, hi);
        first = false;
      }
    }
    if (first) { mn2 = 0x7f807f80u; mx2 = 0xff80ff80u; if (DT == LLMC_F16) { mn2 = 0x7c007c00u; mx2 = 0xfc00fc00u; } }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn2 = min2<DT>(mn2, __shfl_xor_sync(0xffffffffu, mn2, o));
      mx2 = max2<DT>(mx2, __shfl_xor_sync(0xffffffffu, mx2, o));
    }
    if (lane == 0) { smn[warp] = mn2; smx[warp] = mx2; }
    __syncthreads();
    mn2 = smn[0]; mx2 = smx[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) { mn2 = min2<DT>(mn2, smn[w]); mx2 = max2<DT>(mx2, smx[w]); }
    __syncthreads();
    const float mn = fminf(lo_f<DT>(mn2), hi_f<DT>(mn2));
    const float mx = fmaxf(lo_f<DT>(mx2), hi_f<DT>(mx2));
    float s, z;
    qparams<DType<DT>>(mn, mx, a.sym, 1, a.qmin, a.qmax, s, z);
    if (t == 0) {
      DType<DT>::store(a.scales, r, s);
      if (!a.sym && a.zeros) DType<DT>::store(a.zeros, r, z);
    }
    if constexpr (MODE != M_NONE) {
      const Divider<DT> div{s};
      float Ce, vlo, vhi;
      uint32_t ob;
      fast_consts<MODE, BITS>(z, a.qmin, a.qmax, a.sym, Ce, vlo, vhi, ob);
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const int ch = c * 256 + t;
        if (ch < chunks) {
          uint4 o;
          fast_tail<DT, MODE, BITS>(x[c], div, s, Ce, vlo, vhi, ob, a.sym, o);
          if constexpr (MODE == M_QDQ) {
            reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(a.out) + r * a.ld_out)[ch] = o;
          } else if constexpr (MODE == M_PACK && BITS == 4) {
            (reinterpret_cast<uint32_t*>(a.out) + r * a.packed_cols)[ch] = o.x;
          } else {
            reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(a.out) + r * a.cols)[ch] = make_uint2(o.x, o.y);
          }
        }
      }
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) x[c] = xn[c];
  }
}

template <int DT>
static int launch_row_fast(const QuantArgs& a, int mode, int bits, cudaStream_t st) {
  // chunk slots per thread: 2 up to 4096 columns (6 resident CTAs per SM), 4 up to 8192 (4 CTAs)
  const bool small = a.cols <= 4096;
  const int64_t cap = static_cast<int64_t>(kNumSMs) * (small ? 6 : 4);
  const int grid = static_cast<int>(a.rows < cap ? a.rows : cap);
#define QR_GO(MODE, BITS)                                                              \
  do {                                                                                 \
    if (small) quant_row_fast_kernel<DT, MODE, BITS, 2><<<grid, 256, 0, st>>>(a);      \
    else quant_row_fast_kernel<DT, MODE, BITS, 4><<<grid, 256, 0, st>>>(a);            \
  } while (0)
  if (mode == M_NONE) QR_GO(M_NONE, 4);
  else if (mode == M_QDQ) QR_GO(M_QDQ, 4);
  else if (mode == M_PACK && bits == 4) QR_GO(M_PACK, 4);
  else if (mode == M_PACK && bits == 8) QR_GO(M_PACK, 8);
  else if (mode == M_CODES8) QR_GO(M_CODES8, 8);
  else return LLMC_EUNSUPPORTED;
#undef QR_GO
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

template <int DT, int G>
static int launch_fast(const QuantArgs& a, int mode, int bits, int64_t total_groups, cudaStream_t st) {
  constexpr int smem = 2 * TG * G * 2;
  const int64_t n_tiles = (total_groups + TG - 1) / TG;
  const int64_t cap = static_cast<int64_t>(kNumSMs) * (G == 128 ? 3 : 6);
  const int grid = static_cast<int>(n_tiles < cap ? n_tiles : cap);
#define QF_GO(MODE, BITS)                                                                          \
  do {                                                                                             \
    auto kern = quant_group_fast_kernel<DT, G, MODE, BITS>;                                        \
    LLMC_ONCE_PER_DEVICE({                                                                         \
      LLMC_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); \
    });                                                                                            \
    kern<<<grid, TG, smem, st>>>(a, total_groups);                                                 \
  } while (0)
  if (mode == M_NONE) QF_GO(M_NONE, 4);
  else if (mode == M_QDQ) QF_GO(M_QDQ, 4);
  else if (mode == M_PACK && bits == 4) QF_GO(M_PACK, 4);
  else if (mode == M_PACK && bits == 8) QF_GO(M_PACK, 8);
  else if (mode == M_CODES8) QF_GO(M_CODES8, 8);
  else return LLMC_EUNSUPPORTED;
#undef QF_GO
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

// Which (mode, bits) of the fast kernel serves this call, or -1.
static int fast_mode(const QuantArgs& a, int dtype) {
  if (a.ld != a.cols && !(a.ng == 1 && a.ld % 8 == 0)) return -1;      // groups need dense rows
  if (a.col_scale != nullptr && !((a.group == 64 || a.group == 128) && a.ld == a.cols)) return -1;
  if (dtype != LLMC_F16 && dtype != LLMC_BF16) return -1;
  const bool row_kind = a.ng == 1 && a.group == a.cols && a.cols >= 512 && a.cols <= 8192 && a.cols % 8 == 0;
  if (a.group != 64 && a.group != 128 && !row_kind) return -1;
  if (a.rows * a.ng >= (1ll << 40)) return -1;
  if (row_kind && a.out_mode == LLMC_OUT_QDQ && (a.ld_out % 8 != 0)) return -1;
  switch (a.out_mode) {
    case LLMC_OUT_NONE: return M_NONE;
    case LLMC_OUT_QDQ: return (a.out_dtype == dtype && (a.ld_out == a.cols || a.ng == 1)) ? M_QDQ : -1;
    // asymmetric codes + the +2^(bit-1) storage offset overflow their field and the reference ORs
    // the overlapping bits (module_utils.py:842-856): fast_tail reproduces that on the packed word
    case LLMC_OUT_PACK_VLLM: return (a.bit == 4 || a.bit == 8) ? M_PACK : -1;
    case LLMC_OUT_CODES_I8:
    case LLMC_OUT_CODES_U8: return a.bit == 8 ? M_CODES8 : -1;
    default: return -1;
  }
}

}  // namespace qf

template <int DT>
static int launch_dynamic(const QuantArgs& a, bool vec_ok, cudaStream_t st) {
  const int64_t total_groups = a.rows * a.ng;
  if (total_groups == 0 || a.cols == 0) return LLMC_OK;
  if constexpr (DT != LLMC_F32) {
    const int fm = vec_ok ? qf::fast_mode(a, DT) : -1;
    if (fm >= 0) {
      if (a.group == 128 && a.ld == a.cols) return qf::launch_fast<DT, 128>(a, fm, a.bit, total_groups, st);
      if (a.group == 64 && a.ld == a.cols) return qf::launch_fast<DT, 64>(a, fm, a.bit, total_groups, st);
      if (a.ng == 1) return qf::launch_row_fast<DT>(a, fm, a.bit, st);
    }
  }
  if (vec_ok && a.group <= 1024) {
    // 32 elements (4 x 16-byte loads in flight) per lane wherever the group allows it: the
    // per-group scalar work (qparams: four IEEE divides) is then amortised over 4x more
    // elements — with 8 elements per lane the kernel was issue-bound at ~1.1 warp-instr/element.
    const int64_t chunks = a.group >> 3;
    int lpg = 1;
    while (lpg * 4 < chunks) lpg *= 2;               // smallest power of two with <= 4 chunks/lane
    const int ch = static_cast<int>((chunks + lpg - 1) / lpg);
    if (total_groups >= (1ll << 31)) {
      set_last_error("quant_dynamic: %lld groups exceed the 2^31 limit", (long long)total_groups);
      return LLMC_EUNSUPPORTED;
    }
    const int64_t warps_needed = (total_groups + (32 / lpg) - 1) / (32 / lpg);
    int64_t blocks = (warps_needed + 7) / 8;
    const int64_t cap = static_cast<int64_t>(kNumSMs) * 16;
    if (blocks > cap) blocks = cap;
    if (ch == 1) quant_dynamic_warp_kernel<DT, 1><<<(int)blocks, 256, 0, st>>>(a, lpg, total_groups);
    else if (ch == 2) quant_dynamic_warp_kernel<DT, 2><<<(int)blocks, 256, 0, st>>>(a, lpg, total_groups);
    else quant_dynamic_warp_kernel<DT, 4><<<(int)blocks, 256, 0, st>>>(a, lpg, total_groups);
  } else if (vec_ok) {
    int64_t blocks = total_groups;
    const int64_t cap = static_cast<int64_t>(kNumSMs) * 32;
    if (blocks > cap) blocks = cap;
    quant_dynamic_block_kernel<DT><<<(int)blocks, 256, 0, st>>>(a, total_groups);
  } else {
    return LLMC_EUNSUPPORTED;  // caller falls back to qparams_generic + static generic
  }
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

template <int CT, int WT, int QT>
static int launch_static_t(const StaticArgs& s, const QuantArgs& e, bool vec_ok, cudaStream_t st) {
  if (s.rows == 0 || s.cols == 0) return LLMC_OK;
  if (vec_ok) {
    int64_t total = s.rows * (s.cols >> 3);
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = static_cast<int64_t>(kNumSMs) * 32;
    if (blocks > cap) blocks = cap;
    quant_static_vec8_kernel<CT, WT, QT><<<(int)blocks, 256, 0, st>>>(s, e);
  } else {
    int64_t total = s.rows * ((s.cols + s.unit - 1) / s.unit);
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = static_cast<int64_t>(kNumSMs) * 32;
    if (blocks > cap) blocks = cap;
    quant_static_kernel<CT, WT, QT><<<(int)blocks, 256, 0, st>>>(s);
  }
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

static int launch_static(const StaticArgs& s, const QuantArgs& e, int w_dtype, int q_dtype,
                         int round_dtype, bool vec_ok, cudaStream_t st) {
  const int ct = round_dtype >= 0 ? round_dtype : promote(w_dtype, q_dtype);
#define CASE(CT, WT, QT) \
  if (ct == CT && w_dtype == WT && q_dtype == QT) return launch_static_t<CT, WT, QT>(s, e, vec_ok, st);
  CASE(LLMC_F32, LLMC_F32, LLMC_F32)
  CASE(LLMC_F16, LLMC_F16, LLMC_F16)
  CASE(LLMC_BF16, LLMC_BF16, LLMC_BF16)
  CASE(LLMC_F32, LLMC_F32, LLMC_F16)
  CASE(LLMC_F32, LLMC_F32, LLMC_BF16)
  CASE(LLMC_F32, LLMC_F16, LLMC_F32)
  CASE(LLMC_F32, LLMC_BF16, LLMC_F32)
  CASE(LLMC_F32, LLMC_F16, LLMC_BF16)
  CASE(LLMC_F32, LLMC_BF16, LLMC_F16)
  CASE(LLMC_F16, LLMC_F16, LLMC_F32)
  CASE(LLMC_BF16, LLMC_BF16, LLMC_F32)
#undef CASE
  set_last_error("quant_static: unsupported dtype combination w=%d q=%d", w_dtype, q_dtype);
  return LLMC_EUNSUPPORTED;
}

static int check_out_mode(int out_mode, int bit, const void* out) {
  if (out_mode < LLMC_OUT_NONE || out_mode > LLMC_OUT_PACK_VLLM) {
    set_last_error("bad out_mode %d", out_mode);
    return LLMC_EINVAL;
  }
  if (out_mode != LLMC_OUT_NONE && out == nullptr) {
    set_last_error("out is NULL for out_mode %d", out_mode);
    return LLMC_EINVAL;
  }
  if (bit < 2 || bit > 8) {
    set_last_error("bit %d outside 2..8", bit);
    return LLMC_EINVAL;
  }
  return LLMC_OK;
}

}  // namespace llmc

using namespace llmc;

extern "C" int llmc_quant_dynamic(const void* w, int64_t rows, int64_t cols, int64_t ld,
                                  int dtype, int64_t group, int bit, int sym, int use_range,
                                  int qmin, int qmax, const void* col_scale, void* scales,
                                  void* zeros, int out_mode, void* out, int64_t ld_out,
                                  int out_dtype, void* stream) {
  LLMC_CHECK_ARG(rows >= 0 && cols >= 0 && ld >= cols, "quant_dynamic: bad shape %lld x %lld ld %lld",
                 (long long)rows, (long long)cols, (long long)ld);
  if (rows == 0 || cols == 0) return LLMC_OK;
  LLMC_CHECK_ARG(w && scales, "quant_dynamic: null pointer");
  LLMC_CHECK_ARG(dtype >= LLMC_F32 && dtype <= LLMC_BF16, "quant_dynamic: bad dtype %d", dtype);
  LLMC_CHECK_ARG(group > 0 && cols % group == 0,
                 "quant_dynamic: cols %lld not divisible by group %lld", (long long)cols,
                 (long long)group);
  LLMC_CHECK_ARG(sym || zeros, "quant_dynamic: zeros is NULL for asymmetric quantisation");
  if (int rc = check_out_mode(out_mode, bit, out)) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  QuantArgs a{};
  a.w = w; a.rows = rows; a.cols = cols; a.ld = ld;
  a.group = group; a.ng = cols / group;
  a.sym = sym; a.bit = bit;
  if (use_range) { a.qmin = (float)qmin; a.qmax = (float)qmax; }
  else int_range(bit, sym, a.qmin, a.qmax);
  a.scales = scales; a.zeros = zeros; a.col_scale = col_scale;
  a.out_mode = out_mode; a.out = out;
  a.ld_out = (out_mode == LLMC_OUT_QDQ) ? (ld_out > 0 ? ld_out : cols) : cols;
  a.out_dtype = out_dtype;
  const int pf = 32 / bit;
  a.packed_cols = (cols + pf - 1) / pf;

  const bool pack_fast = out_mode != LLMC_OUT_PACK_VLLM || bit == 4 || bit == 8;
  const bool vec_ok = pack_fast && (group % 8 == 0) && (ld % 8 == 0) && aligned16(w) &&
                      (out == nullptr || aligned16(out)) &&
                      (out_mode != LLMC_OUT_QDQ || a.ld_out % 8 == 0);
  if (col_scale != nullptr && !(vec_ok && aligned16(col_scale))) {
    set_last_error("quant_dynamic: col_scale needs the vectorised path (group, ld %% 8 == 0, aligned)");
    return LLMC_EUNSUPPORTED;
  }
  if (vec_ok) {
#define CALL(DT) return launch_dynamic<DT>(a, true, st)
    LLMC_DISPATCH_DT("quant_dynamic", dtype, CALL);
#undef CALL
  }
  // generic: qparams kernel, then the scalar static kernel
  {
    int64_t total_groups = rows * a.ng;
    int64_t blocks = total_groups < kNumSMs * 32 ? total_groups : kNumSMs * 32;
#define CALL(DT) qparams_generic_kernel<DT><<<(int)blocks, 256, 0, st>>>(a, total_groups)
    LLMC_DISPATCH_DT("quant_dynamic", dtype, CALL);
#undef CALL
    LLMC_CHECK_LAUNCH();
  }
  if (out_mode == LLMC_OUT_NONE) return LLMC_OK;
  StaticArgs s{};
  s.w = w; s.rows = rows; s.cols = cols; s.ld = ld;
  s.scales = scales; s.zeros = sym ? nullptr : zeros;
  s.q_row_stride = a.ng; s.group = group; s.gmap = nullptr;
  s.qmin = a.qmin; s.qmax = a.qmax; s.bit = bit;
  s.out_mode = out_mode; s.out = out; s.ld_out = a.ld_out; s.out_dtype = out_dtype;
  s.packed_cols = a.packed_cols;
  s.unit = (out_mode == LLMC_OUT_PACK_VLLM) ? pf : 8;
  return launch_static(s, a, dtype, dtype, -1, false, st);
}

extern "C" int llmc_quant_static(const void* w, int64_t rows, int64_t cols, int64_t ld,
                                 int w_dtype, const void* scales, const void* zeros,
                                 int q_dtype, int round_dtype, int64_t q_row_stride,
                                 int64_t group,
                                 const int32_t* gmap, int bit, int qmin, int qmax,
                                 int out_mode, void* out, int64_t ld_out, int out_dtype,
                                 void* stream) {
  LLMC_CHECK_ARG(rows >= 0 && cols >= 0 && ld >= cols, "quant_static: bad shape");
  if (rows == 0 || cols == 0) return LLMC_OK;
  LLMC_CHECK_ARG(w && scales, "quant_static: null pointer");
  LLMC_CHECK_ARG(group > 0, "quant_static: group must be positive");
  LLMC_CHECK_ARG(qmin < qmax, "quant_static: qmin %d >= qmax %d", qmin, qmax);
  const int zp_inside = (out_mode & LLMC_OUT_FLAG_ZP_INSIDE) ? 1 : 0;
  out_mode &= ~LLMC_OUT_FLAG_ZP_INSIDE;
  LLMC_CHECK_ARG(out_mode != LLMC_OUT_NONE, "quant_static: out_mode NONE makes no sense");
  if (int rc = check_out_mode(out_mode, bit, out)) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int pf = 32 / bit;

  StaticArgs s{};
  s.w = w; s.rows = rows; s.cols = cols; s.ld = ld;
  s.scales = scales; s.zeros = zeros;
  s.q_row_stride = q_row_stride; s.group = group; s.gmap = gmap;
  s.qmin = (float)qmin; s.qmax = (float)qmax; s.bit = bit;
  s.out_mode = out_mode; s.out = out;
  s.ld_out = (out_mode == LLMC_OUT_QDQ) ? (ld_out > 0 ? ld_out : cols) : cols;
  s.out_dtype = out_dtype;
  s.packed_cols = (cols + pf - 1) / pf;
  s.unit = (out_mode == LLMC_OUT_PACK_VLLM) ? pf : 8;
  s.zp_inside = zp_inside;

  QuantArgs e{};
  e.rows = rows; e.cols = cols; e.bit = bit; e.out_mode = out_mode; e.out = out;
  e.ld_out = s.ld_out; e.out_dtype = out_dtype; e.packed_cols = s.packed_cols;

  const bool pack_fast = out_mode != LLMC_OUT_PACK_VLLM || ((bit == 4 || bit == 8) && !gmap);
  const bool vec_ok = pack_fast && (cols % 8 == 0) && (ld % 8 == 0) && aligned16(w) &&
                      aligned16(out) && (gmap || group % 8 == 0) &&
                      (out_mode != LLMC_OUT_QDQ || s.ld_out % 8 == 0);
  return launch_static(s, e, w_dtype, q_dtype, round_dtype, vec_ok, st);
}

extern "C" int llmc_minmax_tensor(const void* w, int64_t n, int dtype, void* mm,
                                  float* workspace, void* stream) {
  LLMC_CHECK_ARG(w && mm && workspace && n > 0, "minmax_tensor: bad argument");
  LLMC_CHECK_ARG(aligned16(w), "minmax_tensor: w not 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t blocks = ((n >> 3) + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > 1024) blocks = 1024;
#define CALL(DT)                                                                \
  minmax_stage1<DT><<<(int)blocks, 256, 0, st>>>(w, n, workspace);              \
  minmax_stage2<DT><<<1, 256, 0, st>>>(workspace, (int)blocks, mm)
  LLMC_DISPATCH_DT("minmax_tensor", dtype, CALL);
#undef CALL
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}

// ---- pack already-quantised codes (API parity with VllmRealQuantLinear.pack(weight, ...)) ----
namespace llmc {
template <typename CodeT>
__global__ void __launch_bounds__(256)
pack_vllm_codes_kernel(const CodeT* __restrict__ codes, int64_t rows, int64_t cols, int bit,
                       int32_t* __restrict__ out, int64_t packed_cols) {
  const int pf = 32 / bit;
  const int off = 1 << (bit - 1);
  const int64_t total = rows * packed_cols;
  for (int64_t u = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < total;
       u += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = u / packed_cols, pc = u - r * packed_cols;
    uint32_t word = 0;
    for (int i = 0; i < pf; ++i) {
      const int64_t c = pc * pf + i;
      if (c < cols)
        word |= (static_cast<uint32_t>(static_cast<int>(codes[r * cols + c]) + off) & 0xffu)
                << (bit * i);
    }
    out[u] = static_cast<int32_t>(word);
  }
}
}  // namespace llmc

extern "C" int llmc_pack_vllm_codes(const void* codes, int code_bytes, int64_t rows, int64_t cols,
                                    int bit, int32_t* out, void* stream) {
  LLMC_CHECK_ARG(codes && out && rows >= 0 && cols >= 0, "pack_vllm_codes: bad argument");
  LLMC_CHECK_ARG(bit >= 2 && bit <= 8, "pack_vllm_codes: bit %d outside 2..8", bit);
  LLMC_CHECK_ARG(code_bytes == 1 || code_bytes == 4, "pack_vllm_codes: codes must be int8 or int32");
  if (rows == 0 || cols == 0) return LLMC_OK;
  const int pf = 32 / bit;
  const int64_t packed_cols = (cols + pf - 1) / pf;
  int64_t blocks = (rows * packed_cols + 255) / 256;
  if (blocks > kNumSMs * 32) blocks = kNumSMs * 32;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (code_bytes == 1)
    pack_vllm_codes_kernel<int8_t><<<(int)blocks, 256, 0, st>>>(
        reinterpret_cast<const int8_t*>(codes), rows, cols, bit, out, packed_cols);
  else
    pack_vllm_codes_kernel<int32_t><<<(int)blocks, 256, 0, st>>>(
        reinterpret_cast<const int32_t*>(codes), rows, cols, bit, out, packed_cols);
  LLMC_CHECK_LAUNCH();
  return LLMC_OK;
}
