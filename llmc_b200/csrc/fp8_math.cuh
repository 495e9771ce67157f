// fp8_math.cuh — the rounding step of FloatQuantizer with `use_qtorch: True` (quant.py:1061-1072),
// written ONCE for every kernel that quantises onto an e4m3 / e5m2 grid (fp8.cu, gptq.cu).
//
// PARITY UNPINNED: the reference rounds with the third-party `qtorch.quant.float_quantize`
// (SURVEY.md §8c).  It is restated as clamp to +-finfo.max, then IEEE round-to-nearest-even onto
// the e4m3fn / e5m2 grid: the hardware `cvt.rn.satfinite` conversion (oracle/fp8_oracle.py).
#pragma once
#include <cuda_fp8.h>
#include <stdint.h>

namespace llmc {

__device__ __forceinline__ float fp8_round(float v, int e5m2) {
  if (e5m2) {
    const __nv_fp8_storage_t b = __nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E5M2);
    return __half2float(__half(__nv_cvt_fp8_to_halfraw(b, __NV_E5M2)));
  }
  const __nv_fp8_storage_t b = __nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3);
  return __half2float(__half(__nv_cvt_fp8_to_halfraw(b, __NV_E4M3)));
}

__device__ __forceinline__ uint8_t fp8_bits(float v, int e5m2) {
  return static_cast<uint8_t>(__nv_cvt_float_to_fp8(v, __NV_SATFINITE, e5m2 ? __NV_E5M2 : __NV_E4M3));
}

}  // namespace llmc
