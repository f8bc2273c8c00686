// tc_common.cuh — Hopper warpgroup MMA (wgmma) helpers and operand conversions (sm_90a inline PTX).
//
// Encodings follow the PTX ISA "wgmma" shared-memory matrix descriptor. Every operand image in
// this project is K-major without swizzle ("interleave"): core matrices of 8 rows x 16 bytes
// (128 contiguous bytes, row r at +16*r).
#pragma once
#include <algorithm>
#include <cfloat>
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
// The A-operand words of one product count: NPROD = 3 is split2_f16; NPROD = 1 (the opt-in fp16
// mode, x*w ~= hi(x)*hi(w)) writes only the hi word, the same bits split2_f16 writes, and leaves
// lo untouched. In that mode the kernels issue one wgmma per K step and read only the hi image of
// each weight stage: |err| ~ 2^-11 * sum_k |w_k x_k| instead of the split's 4e-6.
template <int NPROD>
__device__ __forceinline__ void split_words(float a, float b, uint32_t& hi, uint32_t& lo) {
  static_assert(NPROD == 1 || NPROD == 3, "one or three fp16 products");
  if constexpr (NPROD == 3)
    split2_f16(a, b, hi, lo);
  else
    hi = pack_f16x2_sat(a, b);
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

// ---- weight blobs ----------------------------------------------------------------------------------
// Every kernel reads its weights (the B operand) from blobs packed by the host or, in train mode, by
// the device; both packers use the definitions below.
//
// Byte offset of element (r, k) in one fp16 image with K extent kt, K-major without swizzle:
// SBO = kt * 16, LBO = 128.
__host__ __device__ inline uint32_t img_off(int r, int k, int kt) {
  return static_cast<uint32_t>((r >> 3) * kt * 16 + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2);
}
// Writes the hi/lo split of one pre-scaled weight, h = rn16(w), l = rn16(w - h). Unlike the
// activations' split2_f16 it does not saturate: a pre-scaled weight is below 512.
__host__ __device__ inline void put_weight(unsigned char* hi, unsigned char* lo, float w) {
  const __half h = __float2half_rn(w);
  const __half l = __float2half_rn(w - __half2float(h));
  *reinterpret_cast<__half*>(hi) = h;
  *reinterpret_cast<__half*>(lo) = l;
}
// The pre-scale of a matrix with max|W| = absmax: the power of two that brings max|W| into
// [256, 512), so the lo parts stay normal fp16 numbers and the hi parts far from the 65504
// overflow; the epilogue's multiply undoes it exactly. 1 for an all-zero or non-finite matrix.
// The exponent is capped at max_exp, by default 126 so that 1/scale stays a normal float: uncapped,
// absmax < 2^-119 would give 2^128 = inf (and 1/scale = 0). Every absmax >= 2^-118 is below the cap.
__host__ __device__ inline float pow2_scale(float absmax, int max_exp = 126) {
  if (!(absmax > 0.f && absmax <= FLT_MAX)) return 1.f;
  int e;
  frexpf(absmax, &e);  // absmax = f * 2^e, f in [0.5, 1)
  return ldexpf(1.f, min(9 - e, max_exp));
}

// The generic layer's blob (csrc/pointwise_tc.cu) of a logical [N x K] matrix. N is padded to 64
// and cut into n-tiles of up to 256 rows; K is padded to 16 and cut into 64-k chunks. A chunk is
// two [nw x 32] stages (k 0..31, then 32..63), each a hi image then a lo image, where nw is the
// tile's width. Tiles, chunks and stages follow each other without gaps; padding is zero.
namespace wblob {
constexpr int NT = 256, KCH = 64, WK = 32;
__host__ __device__ inline int npad(int N) { return (N + 63) / 64 * 64; }
__host__ __device__ inline int kchunks(long long K) {
  return static_cast<int>(((K + 15) / 16 * 16 + KCH - 1) / KCH);
}
__host__ __device__ inline long long bytes(int N, long long K) {
  return static_cast<long long>(npad(N)) * kchunks(K) * KCH * 4;
}
// rows of n-tile nt
__host__ __device__ inline int tile_width(int N, int nt) { return min(NT, npad(N) - nt * NT); }
// stage hh of chunk kc of n-tile nt; kch = kchunks(K)
__host__ __device__ inline long long stage_off(int N, int kch, int nt, int kc, int hh) {
  return static_cast<long long>(nt) * NT * kch * KCH * 4 +
         (static_cast<long long>(kc) * 2 + hh) * tile_width(N, nt) * WK * 4;
}
// hi and lo images of element (n, k)
__host__ __device__ inline void elem_off(int N, int kch, int n, int k, long long& hi, long long& lo) {
  const int nt = n / NT;
  hi = stage_off(N, kch, nt, k / KCH, (k / WK) & 1) + img_off(n - nt * NT, k % WK, WK);
  lo = hi + tile_width(N, nt) * WK * 2;
}
}  // namespace wblob
}  // namespace tc

// ---- host-side packing -------------------------------------------------------------------------------
// hi/lo images of scale * W[rows r0..r0+nr) x [k0..k0+kt) (row stride ld) with K extent kt
inline void pack_tile(const float* W, float scale, int ld, int r0, int nr, int k0, int kt,
                      unsigned char* hi, unsigned char* lo) {
  for (int r = 0; r < nr; ++r)
    for (int k = 0; k < kt; ++k) {
      const uint32_t off = tc::img_off(r, k, kt);
      tc::put_weight(hi + off, lo + off, W[static_cast<size_t>(r0 + r) * ld + k0 + k] * scale);
    }
}
// tc::pow2_scale of the n floats at W
inline float pow2_scale(const float* W, size_t n) {
  float m = 0.f;
  for (size_t i = 0; i < n; ++i) m = std::max(m, std::fabs(W[i]));
  return tc::pow2_scale(m);
}

}  // namespace sonet
