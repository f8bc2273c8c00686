// tc_common.cuh — Hopper warpgroup MMA (wgmma) helpers and operand conversions (sm_90a inline PTX).
//
// Encodings follow the PTX ISA "wgmma" shared-memory matrix descriptor. Every operand image in
// this project is K-major without swizzle ("interleave"): core matrices of 8 rows x 16 bytes
// (128 contiguous bytes, row r at +16*r).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstring>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma_ops.cuh"

namespace sonet {
namespace tc {

// ---- descriptors ---------------------------------------------------------------------------------
// Shared-memory matrix descriptor, K-major, no swizzle:
//   LBO = byte distance between the two core matrices adjacent along K (bits 16..29, >>4)
//   SBO = byte distance between 8-row groups along M/N            (bits 32..45, >>4)
// layout type (bits 62..63) = 0. Advancing the start address by n bytes is desc + (n >> 4).
__host__ __device__ constexpr uint64_t smem_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4) |
         (static_cast<uint64_t>((lbo >> 4) & 0x3FFFu) << 16) |
         (static_cast<uint64_t>((sbo >> 4) & 0x3FFFu) << 32);
}

// ---- wgmma ordering ------------------------------------------------------------------------------
// fence before the first wgmma that reads accumulator registers written by ordinary instructions
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
// wait until at most N committed groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// shared-memory writes of ordinary instructions become visible to wgmma / TMA (the async proxy)
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// named barrier over `count` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
// per-thread register budget of the executing warpgroup (all its warps must execute it)
template <int N>
__device__ __forceinline__ void regs_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void regs_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// ---- conversions -----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo_elem, float hi_elem) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
  return r;
}
// fp16 hi/lo split (22 significant bits, vs 16 for bf16): x*w ~= hi(x)*hi(w) + lo(x)*hi(w) +
// hi(x)*lo(w). Weights are pre-scaled by one power of two per matrix (max |s*w| in [256,512)).
// Error envelope of one GEMM output y = sum_k w_k x_k, measured on an H100 80GB HBM3
// (tests/test_gpu_tc_envelope.py, helpers.TC_R / TC_F):
//   |err| <= 4e-6 * sum_k |w_k x_k| + 2^-24 * (sum_k |w_k| + sum_k |x_k| / s)
// The relative term measured up to 1.6e-6 (strict fp32 cuBLAS: 3.2e-7). The second is the floor
// of the split: below |x| ~ 2^-3 lo(x) is an fp16 subnormal, so each activation carries up to
// 2^-25 of ABSOLUTE error however small it is (likewise each weight, 2^-25 / s). A layer whose
// inputs all sit near 2^-14 therefore loses ~1e-4 of its output's precision (the fused first
// PointResNet scaled by 2^-14 end to end: 1.8e-4), and a weight row 10^6 below its matrix's
// largest one leans on the weight-side floor. Range: hi and lo each saturate at 65504, so an
// activation with |x| >= 131008 acts as +-131008, and between 65504 and 131008 the dropped
// lo(x)*lo(w) term costs up to 2^-12 of that product.
// Two floats -> packed fp16 pair (lo = low half = lower K index) with saturation to the largest
// finite fp16 (one F2FP.SATFINITE, where clamps in front of a plain conversion cost more). NaN
// stays NaN.
__device__ __forceinline__ uint32_t pack_f16x2_sat(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// hi and lo words of the pair (a, b)
__device__ __forceinline__ void split2_f16(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = pack_f16x2_sat(a, b);
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  lo = pack_f16x2_sat(a - hf.x, b - hf.y);
}

// Spin on the barrier phase; a protocol bug traps (instead of hanging the GPU) after 2^24 failed
// try_waits.
// The whole loop is ONE asm statement so that values live across it stay in the uniform datapath.
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* bar, uint32_t parity, int tag) {
  (void)tag;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      ".reg .u32 c;\n"
      "mov.u32 c, 0;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "add.u32 c, c, 1;\n"
      "setp.lt.u32 p, c, 0x1000000;\n"
      "@p bra WAIT_%=;\n"
      "trap;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

// Same for waiters that are never latency-critical (a TMA producer running slots ahead): back off
// between polls so the spin does not take issue slots from the warps sharing the sub-partition.
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity, int tag) {
  uint32_t done = 0;
#pragma unroll 1
  for (uint32_t it = 0; it < (1u << 22); ++it) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) return;
    __nanosleep(100);
  }
  (void)tag;
  // no call here (not even printf): a call inside a kernel that issues wgmma makes ptxas
  // serialize every wgmma of the kernel
  asm volatile("trap;");
}

}  // namespace tc

// ---- host-side packing -------------------------------------------------------------------------------
// fp16 hi/lo images of scale * W[rows r0..r0+nr) x [k0..k0+kt) (row stride ld), K-major no-swizzle:
// element (r,k) at (r/8)*SBO + (k/8)*128 + (r%8)*16 + (k%8)*2 with SBO = kt*16.
inline void pack_tile(const float* W, float scale, int ld, int r0, int nr, int k0, int kt,
                      unsigned char* hi, unsigned char* lo) {
  const uint32_t sbo = static_cast<uint32_t>(kt) * 16;
  for (int r = 0; r < nr; ++r)
    for (int k = 0; k < kt; ++k) {
      const float w = W[static_cast<size_t>(r0 + r) * ld + k0 + k] * scale;  // exact (power of 2)
      const __half h = __float2half_rn(w);
      const __half l = __float2half_rn(w - __half2float(h));
      const uint32_t off = (r >> 3) * sbo + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2;
      std::memcpy(hi + off, &h, 2);
      std::memcpy(lo + off, &l, 2);
    }
}
// power of two that brings max|W| into [256, 512): keeps the lo parts normal fp16 numbers and the
// hi parts far from the 65504 overflow; undone exactly by the epilogue's multiply.
inline float pow2_scale(const float* W, size_t n) {
  float m = 0.f;
  for (size_t i = 0; i < n; ++i) m = std::max(m, std::fabs(W[i]));
  if (!(m > 0.f) || !std::isfinite(m)) return 1.f;
  int e;
  std::frexp(m, &e);  // m = f * 2^e, f in [0.5, 1)
  return std::ldexp(1.f, 9 - e);
}

}  // namespace sonet
