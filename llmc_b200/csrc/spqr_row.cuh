// spqr_row.cuh — the per-row arithmetic of SpQR's column sweep (llmc/compression/quantization/
// spqr.py:172-268), written ONCE for device and host.
//
// Rows of the weight are independent given Hinv and the layer's outlier threshold, and every
// quantity of the reference's weight_transform that involves a row is fp32 elementwise torch
// arithmetic plus sums over <= group_size elements.  This header restates that chain in IEEE fp32
// with one rounding per torch op (the primitives and the quantizer of quant_math.cuh; compile the
// host side with -ffp-contract=off) and sums in ascending index order.  The work of ONE row is
// spread over NL lanes: a leave-one-out case is evaluated whole by one lane, and an element of the
// row receives its rank-1 updates in column order from whichever lane owns it, so every value comes
// from the same operation sequence whatever NL is (NL = 1 is the single-thread form).  Lanes
// communicate through the row's storage only, with a barrier between phases.  The CUDA kernel
// (gptq.cu: spqr_inblock_kernel) runs phase(lane) on 16 real lanes with __syncwarp() in between and
// shared-memory strides; tests/ build the same functions for the host CPU, run
// `for lane: phase(lane)` in lock step and compare them bit for bit with oracle/spqr_oracle.py, so
// the device arithmetic and its indexing are pinned before it ever runs on a GPU.
#pragma once
#include <math.h>
#include <stdint.h>

#include "quant_math.cuh"

namespace llmc {
namespace spqr {

// One IntegerQuantizer configuration (quant.py:661-678): [qmin, qmax], symmetric, round_zp.
struct QCfg {
  float qmin, qmax;
  int sym;
  int round_zp;
};

LLMC_HD void qparams(float mn, float mx, const QCfg& c, float& s, float& z) {
  llmc::qparams<F32Round>(mn, mx, c.sym, c.round_zp, c.qmin, c.qmax, s, z);
}

// quant.py:699-717: quant + dequant of one value.
LLMC_HD float qdq(float x, float s, float z, const QCfg& c) {
  const float q = c.round_zp ? quant_code<F32Round>(x, IeeeDiv{s}, z, c.qmin, c.qmax)
                             : quant_code_zp<F32Round>(x, IeeeDiv{fmaxf(s, 1e-9f)}, z, c.qmin, c.qmax);
  return dequant<F32Round>(q, s, z);
}

// spqr.py:337-351: the group's scale (or zero) pushed through the second-level quantizer.  The
// tensor handed to it is [R, 1]; reshape_tensor leaves it alone for per_group / per_channel
// (quant.py:612-632: last dim 1 < group_size), so the statistics are those of ONE value:
// min = max = v.
LLMC_HD float second_level(float v, const QCfg& c) {
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

// Phase 1 of a group: lane evaluates the leave-one-out cases j = lane, lane + NL, ... and writes
// flags[j] (0 / 1).  Every lane recomputes the group's base error (gs quantise-dequantise steps).
LLMC_HD void lanes_group_flags(const float* g, int gstride, const float* hd, int hstride, const Cfg& c,
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
LLMC_HD void lanes_group_qparams(const float* g, int gstride, const uint8_t* flags, const Cfg& c,
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
LLMC_HD float lanes_column(float* w, int ws, const float* Hb, int hi, int hj, int cnt, int col, float s, float z,
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
}  // namespace llmc
