// spqr_row.cuh — the per-row arithmetic of SpQR's column sweep (llmc/compression/quantization/
// spqr.py:172-253), written ONCE for device and host.
//
// Rows of the weight are independent given Hinv and the layer's outlier threshold, and every
// quantity of the reference's weight_transform that involves a row is fp32 elementwise torch
// arithmetic plus sums over <= group_size elements.  This header restates that chain in IEEE fp32
// with one rounding per torch op (no FMA contraction: __f*_rn on the device; compile the host side
// with -ffp-contract=off) and sums in ascending index order.  The CUDA kernel (gptq.cu:
// spqr_inblock_kernel) spreads a row over 16 lanes and runs the lanes_* functions with
// shared-memory strides.  row_block() is the single-thread form of the same arithmetic.  tests/
// build both for the host CPU (the lanes in lock step) and compare them bit for bit with
// oracle/spqr_oracle.py, so the device arithmetic is pinned before it ever runs on a GPU.
#pragma once
#include <cmath>
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define SPQR_HD __host__ __device__ __forceinline__
#else
#define SPQR_HD inline
#endif

namespace spqr {

#if defined(__CUDA_ARCH__)
SPQR_HD float mul(float a, float b) { return __fmul_rn(a, b); }
SPQR_HD float add(float a, float b) { return __fadd_rn(a, b); }
SPQR_HD float sub(float a, float b) { return __fsub_rn(a, b); }
SPQR_HD float dvd(float a, float b) { return __fdiv_rn(a, b); }
#else
SPQR_HD float mul(float a, float b) { return a * b; }
SPQR_HD float add(float a, float b) { return a + b; }
SPQR_HD float sub(float a, float b) { return a - b; }
SPQR_HD float dvd(float a, float b) { return a / b; }
#endif

// One IntegerQuantizer configuration (quant.py:661-678): bit -> [qmin, qmax], symmetric, round_zp.
struct QCfg {
  float qmin, qmax;
  int sym;
  int round_zp;
};

// quant.py:545-559 on a (min, max) pair.
SPQR_HD void qparams(float mn, float mx, const QCfg& c, float& s, float& z) {
  if (c.sym) {
    const float am = fmaxf(fmaxf(fabsf(mx), fabsf(mn)), 1e-5f);
    s = dvd(am, c.qmax);
    z = 0.f;
  } else {
    s = dvd(fmaxf(sub(mx, mn), 1e-5f), sub(c.qmax, c.qmin));
    if (c.round_zp) z = fminf(fmaxf(sub(c.qmin, rintf(dvd(mn, s))), c.qmin), c.qmax);
    else z = sub(c.qmin, dvd(mn, s));
  }
}

// quant.py:699-717: quant + dequant of one value.
SPQR_HD float qdq(float x, float s, float z, const QCfg& c) {
  float q;
  if (c.round_zp) q = add(rintf(dvd(x, s)), z);
  else q = rintf(add(dvd(x, fmaxf(s, 1e-9f)), z));
  q = fminf(fmaxf(q, c.qmin), c.qmax);
  return mul(sub(q, z), s);
}

// spqr.py:337-351: the group's scale (or zero) pushed through the second-level quantizer.  The
// tensor handed to it is [R, 1]; reshape_tensor leaves it alone for per_group / per_channel
// (quant.py:612-632: last dim 1 < group_size), so the statistics are those of ONE value:
// min = max = v.
SPQR_HD float second_level(float v, const QCfg& c) {
  float s, z;
  qparams(v, v, c, s, z);
  return qdq(v, s, z, c);
}

struct Cfg {
  QCfg w;          // the weight quantizer (per_group, group_size = gs)
  QCfg loo;        // spqr.py:56-58: same bit / symmetric, per_channel, round_zp False
  QCfg sc, zc;     // special.scale / special.zero
  int gs;          // group size (16 | 32 | 64 | 128)
  int outliers;    // 1: leave-one-out outlier search for the group statistics (spqr.py:232-241)
  int has_thr;     // threshold != inf: unstructured outlier mask on the column errors (:255-259)
  float thr;
};

// Group statistics -> (scale, zero) after the second level.  g[k * gstride]: the group's current
// weights of this row; hd[k * hstride]: diag(Hinv) of the group's columns.
SPQR_HD void group_qparams(const float* g, int gstride, const float* hd, int hstride, const Cfg& c,
                           float& s_out, float& z_out) {
  const int gs = c.gs;
  float mn = INFINITY, mx = -INFINITY;
  if (!c.outliers) {
    for (int k = 0; k < gs; ++k) { const float v = g[k * gstride]; mn = fminf(mn, v); mx = fmaxf(mx, v); }
  } else {
    // spqr.py:174-192
    float bmn = INFINITY, bmx = -INFINITY;
    for (int k = 0; k < gs; ++k) { const float v = g[k * gstride]; bmn = fminf(bmn, v); bmx = fmaxf(bmx, v); }
    float s, z;
    qparams(bmn, bmx, c.loo, s, z);
    float base = 0.f;
    for (int k = 0; k < gs; ++k) {
      const float v = g[k * gstride];
      const float e = dvd(sub(qdq(v, s, z, c.loo), v), hd[k * hstride]);
      base = add(base, mul(e, e));
    }
    uint32_t flags[4] = {0u, 0u, 0u, 0u};                 // M of spqr.py:235, gs <= 128
    for (int j = 0; j < gs; ++j) {
      float lmn = INFINITY, lmx = -INFINITY;
      for (int k = 0; k < gs; ++k) {
        if (k == j) continue;
        const float v = g[k * gstride];
        lmn = fminf(lmn, v); lmx = fmaxf(lmx, v);
      }
      qparams(lmn, lmx, c.loo, s, z);
      float loo = 0.f;
      for (int k = 0; k < gs; ++k) {
        if (k == j) continue;
        const float v = g[k * gstride];
        const float e = dvd(sub(qdq(v, s, z, c.loo), v), hd[k * hstride]);
        loo = add(loo, mul(e, e));
      }
      if (sub(base, loo) > c.thr) flags[j >> 5] |= 1u << (j & 31);
    }
    // :236-239  mean of the non-outliers, outliers replaced by it
    float num = 0.f, den = 0.f;
    for (int k = 0; k < gs; ++k) {
      const float m = ((flags[k >> 5] >> (k & 31)) & 1u) ? 1.f : 0.f;
      num = add(num, mul(g[k * gstride], sub(1.f, m)));
      den = add(den, sub(1.f, m));
    }
    const float mean = dvd(num, fmaxf(den, 1.f));
    for (int k = 0; k < gs; ++k) {
      const float m = ((flags[k >> 5] >> (k & 31)) & 1u) ? 1.f : 0.f;
      const float v = add(mul(g[k * gstride], sub(1.f, m)), mul(mean, m));
      mn = fminf(mn, v); mx = fmaxf(mx, v);
    }
  }
  float s, z;
  qparams(mn, mx, c.w, s, z);
  s_out = second_level(s, c.sc);
  z_out = second_level(z, c.zc);
}

// One 128-column block of one row (spqr.py:215-268).
//   w[c * ws]           in: the row's weights at block entry; out: tmp (the compensated weights)
//   H(i, j)             = Hb[i * hi + j * hj], the [cnt, cnt] block of Hinv on the diagonal
//   err_out[c * es]     out: Err1
//   mask_out[c * ms]    out: 0 / 1
//   s_out / z_out[g]    out: qparams of the block's cnt / gs groups
// Returns the sum of err^2 (the row's share of Losses).
SPQR_HD float row_block(float* w, int ws, const float* Hb, int hi, int hj, int cnt, const Cfg& c,
                        float* err_out, int es, uint8_t* mask_out, int ms, float* s_out, float* z_out) {
  float loss = 0.f;
  float s = 1.f, z = 0.f;
  for (int col = 0; col < cnt; ++col) {
    if (col % c.gs == 0) {
      group_qparams(w + col * ws, ws, Hb + col * hi + col * hj, hi + hj, c, s, z);
      s_out[col / c.gs] = s;
      z_out[col / c.gs] = z;
    }
    const float wv = w[col * ws];
    const float d = Hb[col * hi + col * hj];
    const float q = qdq(wv, s, z, c.w);
    float err = dvd(sub(wv, q), d);
    uint8_t m = 0;
    if (c.has_thr) {
      m = mul(err, err) > c.thr ? 1 : 0;
      const float mf = m ? 1.f : 0.f;
      const float newq = add(mul(q, sub(1.f, mf)), mul(wv, mf));
      err = dvd(sub(wv, newq), d);
    }
    mask_out[col * ms] = m;
    err_out[col * es] = err;
    loss = add(loss, mul(err, err));
    for (int j = col + 1; j < cnt; ++j)                              // :264-266
      w[j * ws] = sub(w[j * ws], mul(err, Hb[col * hi + j * hj]));
  }
  return loss;
}

// ---- lane-parallel form ----------------------------------------------------------------------------
// The same arithmetic with the work of ONE row spread over NL lanes.  Every value is produced by
// the same operation sequence as in row_block() (a leave-one-out case is evaluated whole by one
// lane; an element of the row receives its rank-1 updates in column order from whichever lane owns
// it), so the results are bit-identical.  Lanes communicate through the row's storage only, with a
// barrier between phases: the CUDA kernel runs phase(lane) on real lanes with __syncwarp() in
// between, the host test runs `for lane: phase(lane)` — the same functions, so the indexing is
// pinned on the CPU as well.

// Phase 1 of a group: lane evaluates the leave-one-out cases j = lane, lane + NL, ... and writes
// flags[j] (0 / 1).  Every lane recomputes the group's base error (gs quantise-dequantise steps).
SPQR_HD void lanes_group_flags(const float* g, int gstride, const float* hd, int hstride, const Cfg& c,
                               int lane, int nl, uint8_t* flags) {
  const int gs = c.gs;
  if (!c.outliers) {
    for (int j = lane; j < gs; j += nl) flags[j] = 0;
    return;
  }
  float bmn = INFINITY, bmx = -INFINITY;
  for (int k = 0; k < gs; ++k) { const float v = g[k * gstride]; bmn = fminf(bmn, v); bmx = fmaxf(bmx, v); }
  float s, z;
  qparams(bmn, bmx, c.loo, s, z);
  float base = 0.f;
  for (int k = 0; k < gs; ++k) {
    const float v = g[k * gstride];
    const float e = dvd(sub(qdq(v, s, z, c.loo), v), hd[k * hstride]);
    base = add(base, mul(e, e));
  }
  for (int j = lane; j < gs; j += nl) {
    float lmn = INFINITY, lmx = -INFINITY;
    for (int k = 0; k < gs; ++k) {
      if (k == j) continue;
      const float v = g[k * gstride];
      lmn = fminf(lmn, v); lmx = fmaxf(lmx, v);
    }
    qparams(lmn, lmx, c.loo, s, z);
    float loo = 0.f;
    for (int k = 0; k < gs; ++k) {
      if (k == j) continue;
      const float v = g[k * gstride];
      const float e = dvd(sub(qdq(v, s, z, c.loo), v), hd[k * hstride]);
      loo = add(loo, mul(e, e));
    }
    flags[j] = sub(base, loo) > c.thr ? 1 : 0;
  }
}

// Phase 2 of a group (every lane, redundantly): statistics with the flagged outliers replaced by the
// mean of the others, weight qparams, second level.
SPQR_HD void lanes_group_qparams(const float* g, int gstride, const uint8_t* flags, const Cfg& c,
                                 float& s_out, float& z_out) {
  const int gs = c.gs;
  float mn = INFINITY, mx = -INFINITY;
  if (!c.outliers) {
    for (int k = 0; k < gs; ++k) { const float v = g[k * gstride]; mn = fminf(mn, v); mx = fmaxf(mx, v); }
  } else {
    float num = 0.f, den = 0.f;
    for (int k = 0; k < gs; ++k) {
      const float m = flags[k] ? 1.f : 0.f;
      num = add(num, mul(g[k * gstride], sub(1.f, m)));
      den = add(den, sub(1.f, m));
    }
    const float mean = dvd(num, fmaxf(den, 1.f));
    for (int k = 0; k < gs; ++k) {
      const float m = flags[k] ? 1.f : 0.f;
      const float v = add(mul(g[k * gstride], sub(1.f, m)), mul(mean, m));
      mn = fminf(mn, v); mx = fmaxf(mx, v);
    }
  }
  float s, z;
  qparams(mn, mx, c.w, s, z);
  s_out = second_level(s, c.sc);
  z_out = second_level(z, c.zc);
}

// Column phase (every lane computes err / mask of column `col` redundantly; the lane then applies
// the rank-1 update to the later columns it owns: col + 1 + lane, + NL, ...).
SPQR_HD float lanes_column(float* w, int ws, const float* Hb, int hi, int hj, int cnt, int col, float s, float z,
                           const Cfg& c, int lane, int nl, uint8_t& m_out) {
  const float wv = w[col * ws];
  const float d = Hb[col * hi + col * hj];
  const float q = qdq(wv, s, z, c.w);
  float err = dvd(sub(wv, q), d);
  uint8_t m = 0;
  if (c.has_thr) {
    m = mul(err, err) > c.thr ? 1 : 0;
    const float mf = m ? 1.f : 0.f;
    const float newq = add(mul(q, sub(1.f, mf)), mul(wv, mf));
    err = dvd(sub(wv, newq), d);
  }
  m_out = m;
  for (int j = col + 1 + lane; j < cnt; j += nl)
    w[j * ws] = sub(w[j * ws], mul(err, Hb[col * hi + j * hj]));
  return err;
}

}  // namespace spqr
