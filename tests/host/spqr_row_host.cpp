// Host build of llmc_b200/csrc/spqr_row.cuh (and the quant_math.cuh it includes) for
// tests/test_oracle_golden.py: the SAME source the CUDA kernel spqr_inblock_kernel compiles for the
// device, driven row by row on the CPU so that its arithmetic can be compared bit for bit with
// oracle/spqr_oracle.py (and, through it, with the reference-generated goldens).  The lanes_*
// functions the kernel runs are emulated in lock step below; nl = 1 is the single-thread form.
// Build: g++ -O2 -ffp-contract=off -shared -fPIC.
#include <cmath>

#include "spqr_row.cuh"

using namespace llmc;

static spqr::QCfg qcfg(int bit, int sym, int round_zp) {
  spqr::QCfg q{};
  int_range(bit, sym, q.qmin, q.qmax);
  q.sym = sym; q.round_zp = round_zp;
  return q;
}

// Lock-step emulation of the lane-parallel kernel: every phase runs for lane = 0 .. nl-1 before the
// next phase starts (the kernel's __syncwarp()).  Column phases read w[col] BEFORE any lane of that
// phase writes (lanes only write columns > col), as on the device.
extern "C" void spqr_row_block_lanes_host(float* W, const float* Hb, int R, int cnt, int gs, int bit, int sym,
                                          int round_zp, int s_bit, int s_sym, int s_rzp, int z_bit, int z_sym,
                                          int z_rzp, float thr, int simplified, int nl, float* err,
                                          uint8_t* mask, float* S, float* Z, float* loss) {
  spqr::Cfg c{};
  c.w = qcfg(bit, sym, round_zp);
  c.loo = qcfg(bit, sym, 0);
  c.sc = qcfg(s_bit, s_sym, s_rzp);
  c.zc = qcfg(z_bit, z_sym, z_rzp);
  c.gs = gs;
  c.thr = thr;
  c.has_thr = !std::isinf(thr);
  c.outliers = (!simplified && c.has_thr) ? 1 : 0;
  const int ng = (cnt + gs - 1) / gs;
  uint8_t flags[128];
  for (int r = 0; r < R; ++r) {
    float* w = W + static_cast<long>(r) * cnt;
    float l = 0.f, s = 1.f, z = 0.f;
    for (int col = 0; col < cnt; ++col) {
      if (col % gs == 0) {
        for (int lane = 0; lane < nl; ++lane)
          spqr::lanes_group_flags(w + col, 1, Hb + col * cnt + col, cnt + 1, c, lane, nl, flags);
        float s0 = 0.f, z0 = 0.f;
        for (int lane = 0; lane < nl; ++lane) {
          float sl, zl;
          spqr::lanes_group_qparams(w + col, 1, flags, c, sl, zl);
          if (lane == 0) { s0 = sl; z0 = zl; }
        }
        s = s0; z = z0;
        S[static_cast<long>(r) * ng + col / gs] = s;
        Z[static_cast<long>(r) * ng + col / gs] = z;
      }
      float e0 = 0.f;
      uint8_t m0 = 0;
      for (int lane = 0; lane < nl; ++lane) {
        uint8_t m;
        const float e = spqr::lanes_column(w, 1, Hb, cnt, 1, cnt, col, s, z, c, lane, nl, m);
        if (lane == 0) { e0 = e; m0 = m; }
      }
      err[static_cast<long>(r) * cnt + col] = e0;
      mask[static_cast<long>(r) * cnt + col] = m0;
      l = add(l, mul(e0, e0));
    }
    loss[r] = l;
  }
}
