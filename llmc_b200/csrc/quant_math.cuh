// quant_math.cuh — the arithmetic of IntegerQuantizer (llmc/compression/quantization/quant.py:
// 545-559 get_qparams, 661-678 the integer range, 699-717 quant / dequant), written ONCE for every
// quantising kernel (quant.cu, awq.cu, gptq.cu, spqr_row.cuh) and for the host build of
// spqr_row.cuh that the CPU tests pin to the oracle.
//
// Bit-exactness comes from rounding at the same points as torch: every op is one IEEE fp32 op
// (__f*_rn on the device, so nothing is contracted into an FMA; compile host code with
// -ffp-contract=off) followed by `Round::rT`, the rounding of the result to the tensor dtype T
// (DType<DT> of common.cuh on the device, F32Round for fp32 on either side).  The divider of
// x / s is a parameter: the three below give the same correctly rounded quotient on the operands
// each is used for, at different cost.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define LLMC_HD __host__ __device__ __forceinline__
#else
#define LLMC_HD inline
#endif

namespace llmc {

// ---- one rounding per op ---------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
LLMC_HD float mul(float a, float b) { return __fmul_rn(a, b); }
LLMC_HD float add(float a, float b) { return __fadd_rn(a, b); }
LLMC_HD float sub(float a, float b) { return __fsub_rn(a, b); }
LLMC_HD float dvd(float a, float b) { return __fdiv_rn(a, b); }
LLMC_HD float rcp(float a) { return __frcp_rn(a); }
#else
LLMC_HD float mul(float a, float b) { return a * b; }
LLMC_HD float add(float a, float b) { return a + b; }
LLMC_HD float sub(float a, float b) { return a - b; }
LLMC_HD float dvd(float a, float b) { return a / b; }
LLMC_HD float rcp(float a) { return 1.f / a; }
#endif

// Rounding policy of fp32 tensors: none.
struct F32Round {
  LLMC_HD static float rT(float x) { return x; }
};

// quant.py:666-672: the default [qmin, qmax] of a `bit`-bit quantizer.
LLMC_HD void int_range(int bit, int sym, float& qmin, float& qmax) {
  if (sym) { qmin = -static_cast<float>(1 << (bit - 1)); qmax = static_cast<float>((1 << (bit - 1)) - 1); }
  else { qmin = 0.f; qmax = static_cast<float>((1 << bit) - 1); }
}

// quant.py:545-559 (get_qparams) on a (min, max) pair.  torch's clamp(min=1e-5) converts the
// python scalar to T first.  round_zp = false keeps the real-valued zero-point qmin - min / s.
template <class Round>
LLMC_HD void qparams(float mn, float mx, int sym, int round_zp, float qmin, float qmax, float& s, float& z) {
  const float eps = Round::rT(1e-5f);
  if (sym) {
    s = Round::rT(dvd(fmaxf(fmaxf(fabsf(mx), fabsf(mn)), eps), qmax));
    z = 0.f;
  } else {
    s = Round::rT(dvd(fmaxf(Round::rT(sub(mx, mn)), eps), sub(qmax, qmin)));
    if (round_zp) z = fminf(fmaxf(Round::rT(sub(qmin, rintf(Round::rT(dvd(mn, s))))), qmin), qmax);
    else z = Round::rT(sub(qmin, Round::rT(dvd(mn, s))));
  }
}

// quant.py:699-701: clamp(round(x / s) + z, qmin, qmax), the integer-valued code.  `div(x)` is x / s.
template <class Round, class Div>
LLMC_HD float quant_code(float x, const Div& div, float z, float qmin, float qmax) {
  const float q = rintf(Round::rT(div(x))) + z;   // integers: exact whenever the result survives the clamp
  return fminf(fmaxf(q, qmin), qmax);
}

// round_zp = false (quant.py:702-707, real-valued zero-points):
//   clamp(round(x / s.clamp_min(1e-9) + z), qmin, qmax) — the zero-point goes INSIDE the rounding.
// `div` must have been built from the clamped scale.
template <class Round, class Div>
LLMC_HD float quant_code_zp(float x, const Div& div, float z, float qmin, float qmax) {
  const float t = Round::rT(add(Round::rT(div(x)), z));
  return fminf(fmaxf(rintf(t), qmin), qmax);
}

// quant.py:710-712: (q - z) * s, both ops rounded to T.  q - z is exact for integer zero-points;
// the real-valued ones of round_zp = false need its rounding.
template <class Round>
LLMC_HD float dequant(float q, float s, float z) {
  return Round::rT(mul(Round::rT(sub(q, z)), s));
}

// ---- dividers: x / s for a fixed s, correctly rounded to fp32 ---------------------------------
// The IEEE divide.
struct IeeeDiv {
  float s;
  LLMC_HD float operator()(float x) const { return dvd(x, s); }
};

#if defined(__CUDACC__)
// For 16-bit T: both x and s carry <= 11 significant bits, so q0 = RN(x*r), r = RN(1/s),
// followed by one exact-remainder correction is the correctly rounded quotient (the remainder
// x - q0*s is exact in fp32 and the corrected value is within 2^-47 of x/s while fp32 rounding
// boundaries are >= 2^-36 away; DESIGN.md §3).  Not exact for wider operands.
// Domain: finite quotients.  Where IEEE gives a non-finite quotient of a finite x — |x / s| beyond
// fp32 range (bf16 only) or s = inf (a group holding +-inf) — this returns NaN (inf - inf, 0 * inf),
// which the clamp of quant_code turns into qmin instead of the IEEE code.  A guard for it measured
// slower than run-to-run noise on the row kernel, so the divider stays as is.
struct RecipDiv {
  float s, r;
  __device__ __forceinline__ explicit RecipDiv(float s_) : s(s_), r(dvd(1.0f, s_)) {}
  __device__ __forceinline__ float operator()(float x) const {
    const float q0 = mul(x, r);
    const float rem = __fmaf_rn(-q0, s, x);
    return __fmaf_rn(rem, r, q0);
  }
};

// For fp32 operands, given r = RN(1 / s).  q1 is a faithful quotient (residual-corrected once), and
// the second correction of a faithful quotient with a correctly rounded reciprocal is the correctly
// rounded quotient (Markstein), provided nothing under/overflows: x, s and r with exponents in
// [2^-40, 2^41) keep q and both residuals normal (x = 0 is exact as well).  Anything else takes
// div.rn, kept OUT of line: inlined, its ~10-instruction sequence sat on the dependent chain of
// every GPTQ column step whether or not it was needed.
static __device__ __noinline__ float div_rn_out_of_line(float x, float s) { return dvd(x, s); }

struct MarksteinDiv {
  float s, r;
  bool ok;                 // s and r inside the range guard: a property of the divisor, evaluated once
  __device__ __forceinline__ static bool exp_mid(float v) {
    return (((__float_as_uint(v) >> 23) & 0xffu) - 87u) <= 80u;
  }
  __device__ __forceinline__ MarksteinDiv(float s_, float r_) : s(s_), r(r_), ok(exp_mid(s_) && exp_mid(r_)) {}
  __device__ __forceinline__ explicit MarksteinDiv(float s_) : MarksteinDiv(s_, rcp(s_)) {}
  __device__ __forceinline__ float operator()(float x) const {
    const float q0 = mul(x, r);
    float rem = __fmaf_rn(-q0, s, x);
    const float q1 = __fmaf_rn(rem, r, q0);
    rem = __fmaf_rn(-q1, s, x);
    float q2 = __fmaf_rn(rem, r, q1);
    if (!(ok && (exp_mid(x) || x == 0.f))) q2 = div_rn_out_of_line(x, s);
    return q2;
  }
};
#endif

}  // namespace llmc
