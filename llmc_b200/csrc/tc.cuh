// tc.cuh — sm_90a building blocks: mbarrier, TMA (cp.async.bulk.tensor) and warpgroup MMA
// (wgmma.mma_async, fp32 accumulators in registers).  Hand-written inline PTX; descriptor bit
// layouts follow the PTX ISA "asynchronous warpgroup level matrix" chapter.
#pragma once

#include <cuda.h>  // CUtensorMap (types only; the driver entry point is resolved at run time)

#include "common.cuh"

namespace llmc {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ---------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded wait: a protocol bug must trap (kernel error) instead of hanging the GPU.  No printf on
// the timeout path: a function call inside a wgmma loop makes ptxas serialise every wgmma.
__device__ __forceinline__ bool mbar_try_wait(uint32_t addr, uint32_t parity) {
  uint32_t done = 0;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.b32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(done)
      : "r"(addr), "r"(parity)
      : "memory");
  return done != 0;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  if (mbar_try_wait(addr, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  while (!mbar_try_wait(addr, parity)) {
    if (globaltimer_ns() - t0 > 5000000000ull) __trap();  // 5 s: far beyond any legitimate wait
  }
}

// generic-proxy writes to smem -> visible to the async proxy (wgmma / TMA reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- TMA ----------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tile load, completion counted in bytes on `bar`.  c0 = innermost coordinate.
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
        "r"(c1)
      : "memory");
}

// ---- TMA rings ------------------------------------------------------------------------------
// A ring is kStages shared-memory stages that a producer fills and consumers drain, with two
// mbarriers per stage placed after the kernel's ring data: full[s] completes when stage s holds
// its data (TMA transaction bytes, or the producer's arrivals), empty[s] when every consumer has
// released it.  Each role walks the stages in the same order with its own PipeState; the n-th use
// of a stage waits for parity n & 1, and the producer's first pass over the ring waits on the
// parity before that, which a freshly initialised barrier reports complete.

// 1024-byte aligned start of the rings (a 128-byte swizzle atom is 8 rows = 1024 bytes) in the
// kernel's dynamic shared memory.  Offsetting the extern array, instead of rounding its address as
// an integer, keeps the result a pointer the compiler knows to be shared: plain loads and stores
// through it compile to LDS / STS, not generic LD / ST.
__device__ __forceinline__ uint8_t* ring_base(uint8_t* smem_raw) {
  const uint32_t raw = smem_u32(smem_raw);
  return smem_raw + ((0u - raw) & 1023u);
}
// Dynamic shared memory of a kernel whose rings take ring_bytes: the alignment slack above and
// 256 bytes for the barriers (two per stage, at most 16 stages in all).
constexpr int ring_smem_bytes(int ring_bytes) { return ring_bytes + 1024 + 256; }

template <int kStages>
struct PipeState {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void advance() {
    if (++stage == kStages) { stage = 0; phase ^= 1; }
  }
  // the state after i advances from the start
  __device__ __forceinline__ static PipeState at(uint32_t i) {
    return {static_cast<int>(i % kStages), (i / kStages) & 1u};
  }
};

template <int kStages>
struct Ring {
  using State = PipeState<kStages>;
  uint64_t* full;                   // full[kStages], followed by empty[kStages]
  __device__ __forceinline__ explicit Ring(void* bars) : full(static_cast<uint64_t*>(bars)) {}
  __device__ __forceinline__ void* end() const { return full + 2 * kStages; }
  // by one thread, followed by fence_barrier_init and a CTA barrier
  __device__ __forceinline__ void init(uint32_t full_count, uint32_t empty_count) const {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], full_count);
      mbar_init(&full[kStages + s], empty_count);
    }
  }
  __device__ __forceinline__ void wait_full(const State& st) const {
    mbar_wait(&full[st.stage], st.phase);
  }
  __device__ __forceinline__ void wait_empty(const State& st) const {
    mbar_wait(&full[kStages + st.stage], st.phase ^ 1);
  }
  __device__ __forceinline__ void expect_tx(const State& st, uint32_t bytes) const {
    mbar_expect_tx(&full[st.stage], bytes);
  }
  __device__ __forceinline__ void release(int stage) const { mbar_arrive(&full[kStages + stage]); }
};

// ---- wgmma ----------------------------------------------------------------------------------
// Shared-memory matrix descriptor (64 bit):
//   [0,14)  start address >> 4        [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4   [49,52) base offset = 0   [62,64) 1 = SWIZZLE_128B
// K-major, SWIZZLE_128B (rows of 128 B, 8-row 1024-B atoms, as written by TMA):
//   SBO = 1024 (next 8 rows), LBO unused (encoded 1).
// MN-major, SWIZZLE_128B (128-B rows hold 64 MN-contiguous elements of one K index):
//   SBO = 1024 (next 8 K indices), LBO = byte distance between 64-element MN atoms.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes,
                                                   uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3fffu);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3fffu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3fffu) << 32;
  d |= static_cast<uint64_t>(1) << 62;  // SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accumulator reads / writes across an in-flight wgmma.
__device__ __forceinline__ void fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, issued by one warpgroup; trans = operand MN-major.
// Accumulator fragment of thread t (warp w = t / 32 of the group, lane l):
//   d[4 j + 2 i + c] = D[16 w + l / 4 + 8 i][8 j + 2 (l % 4) + c],  j < 16, i, c < 2.
template <int kTransA, int kTransB>
__device__ __forceinline__ void wgmma_m64n128k16_bf16(float (&d)[64], uint64_t adesc, uint64_t bdesc,
                                         uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTransA), "n"(kTransB));
}
template <int kTransA, int kTransB>
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t adesc, uint64_t bdesc,
                                         uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTransA), "n"(kTransB));
}

// D[64 x 128] (+)= A[64 x 32] * B[128 x 32]^T on e4m3 operands, issued by one warpgroup.  8-bit
// operands are read K-major only (no transpose immediates); fragment layout as above.  The Hopper
// tensor core keeps a reduced-precision fp32 accumulator for 8-bit inputs, so long K runs are
// promoted into a full fp32 register sum by the caller (gemm_fp8.cu).
__device__ __forceinline__ void wgmma_m64n128k32_e4m3(float (&d)[64], uint64_t adesc, uint64_t bdesc,
                                                      uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// D[64 x 128] += A[64 x 8] * B[128 x 8]^T on tf32 operands, issued by one warpgroup.  tf32 operands
// are read K-major only (no transpose immediates); fragment layout as above.  Always accumulates:
// the 3xTF32 update (tf32.cu) starts from zeroed accumulators, so an exact-zero sum keeps the
// sign 0.f + ... gives it.
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc));
}

template <bool kBf16, int kTransA, int kTransB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc,
                                                 uint32_t accumulate) {
  if constexpr (kBf16) wgmma_m64n128k16_bf16<kTransA, kTransB>(d, adesc, bdesc, accumulate);
  else wgmma_m64n128k16_f16<kTransA, kTransB>(d, adesc, bdesc, accumulate);
}

// ---- forward GEMMs (gemm.cu, gemm_w4.cu, gemm_fp8.cu) ------------------------------------------
// L2-grouped tile order: the weights are swept in groups of `gn` n-tiles (<= ~32 MB, L2 resident,
// see l2_group_width), all m-tiles per group, n fastest inside the group.  Activations are re-read
// once per group from HBM, weights once; n-fastest over a 14336-row weight would instead stream
// the whole 117 MB weight through L2 once per 132-tile wave.
__device__ __forceinline__ void grouped_tile(int u, int m_tiles, int n_tiles, int gn, int& m_blk,
                                             int& n_blk) {
  const int per_group = gn * m_tiles;
  const int g = u / per_group;
  const int rem = u - g * per_group;
  const int gsz = min(gn, n_tiles - g * gn);
  m_blk = rem / gsz;
  n_blk = g * gn + (rem - m_blk * gsz);
}

// Stores the 16-bit pair pk (pack_pair) of columns col, col + 1 at o = &Y[row][col], the second
// element only if `pair`: one 32-bit word when ld is even (o is then 4-byte aligned), element by
// element otherwise.
__device__ __forceinline__ void store_pair16(uint16_t* o, uint32_t pk, bool pair, int64_t ld) {
  if (pair && (ld & 1) == 0) *reinterpret_cast<uint32_t*>(o) = pk;
  else {
    o[0] = static_cast<uint16_t>(pk & 0xffffu);
    if (pair) o[1] = static_cast<uint16_t>(pk >> 16);
  }
}

// Stores this thread's part of an m64n128 accumulator fragment (layout at wgmma_m64n128k16_bf16)
// whose element (0, 0) is Y[row0][col0] of the fp32 matrix Y[M, N] with row stride ld.  Column
// pairs are stored as one 8-byte word when ld is even, element by element otherwise.
__device__ __forceinline__ void store_f32_m64n128(const float (&acc)[64], int64_t row0, int64_t col0,
                                                  int64_t M, int64_t N, int64_t ld, float* out) {
  const int tid = threadIdx.x & 127, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int64_t col = col0 + 8 * j + 2 * (lane & 3);
    if (col >= N) continue;
    const bool pair = col + 1 < N;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int64_t row = row0 + (tid >> 5) * 16 + (lane >> 2) + 8 * i;
      if (row >= M) continue;
      const float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
      float* o = out + row * ld + col;
      if (pair && (ld & 1) == 0) *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
      else {
        o[0] = v0;
        if (pair) o[1] = v1;
      }
    }
  }
}

// The F.linear epilogue: stores this thread's part of an m64n128 accumulator fragment whose
// element (0, 0) is Y[row0][col0] of the DT matrix Y[M, N] with row stride ld.  The bias (DT, may
// be null) is added in fp32 before the single rounding, as F.linear does.
template <int DT>
__device__ __forceinline__ void store_linear_m64n128(const float (&acc)[64], int64_t row0,
                                                     int64_t col0, int64_t M, int64_t N, int64_t ld,
                                                     const void* bias, void* out) {
  const int tid = threadIdx.x & 127, lane = threadIdx.x & 31;
  const uint16_t* bs = static_cast<const uint16_t*>(bias);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int64_t col = col0 + 8 * j + 2 * (lane & 3);
    if (col >= N) continue;
    const bool pair = col + 1 < N;
    float b0 = 0.f, b1 = 0.f;                    // loaded once per column pair
    if (bs != nullptr) {
      b0 = widen16<DT>(bs[col]);
      if (pair) b1 = widen16<DT>(bs[col + 1]);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int64_t row = row0 + (tid >> 5) * 16 + (lane >> 2) + 8 * i;
      if (row >= M) continue;
      float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
      if (bs != nullptr) { v0 += b0; v1 += b1; }
      store_pair16(static_cast<uint16_t*>(out) + row * ld + col, pack_pair<DT>(v0, v1), pair, ld);
    }
  }
}

}  // namespace tc

// ---- host helpers shared across translation units ---------------------------------------------
// gemm.cu: tensor-map encoding through the driver entry point.  rows x cols matrix of elem_bytes
// elements, row stride ld_elems; box = box_cols (inner) x box_rows.  A swizzled box row must be
// exactly the swizzle span (128-byte swizzle: box_cols * elem_bytes == 128).
int encode_tmap_2d(CUtensorMap* out, const void* base, CUtensorMapDataType dtype, uint32_t elem_bytes,
                   uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows,
                   uint32_t box_cols, CUtensorMapSwizzle swizzle);

// Width in n-tiles of a group of tc::grouped_tile: as many n-tiles of weights as 32 MB of L2
// holds, given the bytes one n-tile takes (divisor > 0), and at least one, at most n_tiles.
inline int l2_group_width(int64_t divisor, int n_tiles) {
  int64_t gn = (32ll << 20) / divisor;
  if (gn < 1) gn = 1;
  if (gn > n_tiles) gn = n_tiles;
  return static_cast<int>(gn);
}

// tf32.cu: 3xTF32 rank-K updates (see there) and the tf32 split hi = tf32(x), lo = tf32(x - hi).
// tf32_split(x) is that split of one element (.x = hi, .y = lo), tf32 rounding to nearest with
// ties away from zero (cvt.rna); hi + lo carries x to ~2^-22 relative.  The 3xTF32 update's error
// bound and the oracle's tf32_split assume exactly this format.
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ float2 tf32_split(float x) {
  const float hi = tf32_rna(x);
  return make_float2(hi, tf32_rna(x - hi));
}
// A GEMM operand held as its tf32 split, K-major: element (i, k) at [i * ld + k]; i indexes M
// (operand A) or N (operand B).
struct SplitOperand {
  const float* hi;
  const float* lo;
  int64_t ld;
};
// An fp32 matrix held as its tf32 split with row stride ld.  at: the K-major operand whose element
// (i, k) is the matrix element (row + i, col + k).
struct SplitMatrix {
  float* hi;
  float* lo;
  int64_t ld;
  SplitOperand at(int64_t row, int64_t col) const {
    return {hi + row * ld + col, lo + row * ld + col, ld};
  }
};
// C[i][j] -= sum_k A(i, k) B(j, k) for i < M, j < N, k < K; C has row stride ldc.  The optional
// parts default to off and are set by the chained setters, so one update reads as one statement:
//   tf32x3_update(Tf32x3Update{A, B, c, ldc, M, N, K}.overwrite().split_into(S, row, col), stream)
struct Tf32x3Update {
  SplitOperand a, b;
  float* c;
  int64_t ldc, M, N, K;
  bool assign = false;              // C = A B^T instead of C -= A B^T
  bool lower = false;               // only the tiles that touch the lower triangle (col <= row),
  int64_t row_off = 0, col_off = 0; //   C[0][0] being element (row_off, col_off) of the matrix
  SplitMatrix c_split{};            // tf32 split of the result (ld == ldc) where C's row <
  int64_t split_rows = INT64_MAX;   //   split_rows or column < split_cols; hi == nullptr: none
  int64_t split_cols = INT64_MAX;
  bool one_tile_per_cta = false;    // grid = tile count (see tf32x3_update)
  bool transposed = false;          // C holds the transpose of the updated matrix (see transpose())

  Tf32x3Update& overwrite() { assign = true; return *this; }
  // C^T -= B A^T written as C -= A B^T: the cross terms are issued as A_hi*B_lo, then A_lo*B_hi,
  // the order C^T's own update would issue them in, so either form gives the same bits.
  Tf32x3Update& transpose() { transposed = true; return *this; }
  Tf32x3Update& lower_tiles(int64_t row0, int64_t col0) {
    lower = true; row_off = row0; col_off = col0; return *this;
  }
  // the split goes to s at (row, col) onward, everywhere unless narrowed by split_first_*
  Tf32x3Update& split_into(const SplitMatrix& s, int64_t row, int64_t col) {
    c_split = {s.hi + row * s.ld + col, s.lo + row * s.ld + col, s.ld};
    return *this;
  }
  Tf32x3Update& split_first_rows(int64_t rows) { split_rows = rows; split_cols = 0; return *this; }
  Tf32x3Update& split_first_cols(int64_t cols) { split_rows = 0; split_cols = cols; return *this; }
  Tf32x3Update& tile_per_cta() { one_tile_per_cta = true; return *this; }
};
int tf32x3_update(const Tf32x3Update& u, cudaStream_t st);
int split_tf32(const float* x, int64_t rows, int64_t cols, int64_t ld, float* hi, float* lo,
               int64_t ld_out, cudaStream_t st);
// the split of x^T: hi/lo[c * ld_out + r] for x[r * ld + c]
int split_tf32_transposed(const float* x, int64_t rows, int64_t cols, int64_t ld, float* hi, float* lo,
                          int64_t ld_out, cudaStream_t st);

}  // namespace llmc
