// common.cuh — shared helpers for libsonet_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/sonet_b200.h"

namespace sonet {

// thread-local error string, set by SONET_FAIL / check_launch
void set_error(const char* fmt, ...);

#define SONET_FAIL(code, ...)        \
  do {                               \
    ::sonet::set_error(__VA_ARGS__); \
    return (code);                   \
  } while (0)

#define SONET_REQUIRE(cond, ...)                         \
  do {                                                   \
    if (!(cond)) SONET_FAIL(SONET_ERR_BAD_ARG, __VA_ARGS__); \
  } while (0)

// to be called right after a kernel launch; does not synchronise.
int check_launch(const char* what);

inline cudaStream_t as_stream(sonet_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

int sm_count();           // cached multiprocessor count of the current device
int max_smem_optin();     // cached max opt-in dynamic shared memory per block

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Activation code argument (SONET_ACT_*): validated before any CUDA call.
#define SONET_REQUIRE_ACT(act, what)                                                       \
  SONET_REQUIRE((act) == SONET_ACT_NONE || (act) == SONET_ACT_RELU || (act) == SONET_ACT_ELU, \
                "%s: activation code %d is not SONET_ACT_NONE (0), _RELU (1) or _ELU (2)", what, \
                static_cast<int>(act))

// ---- activations ------------------------------------------------------------------------------
// ELU with alpha = 1 (nn.ELU(alpha=1.0), models/layers.py:136-137), in fp32 in every mode. expm1f,
// not __expf(x) - 1: near 0 the difference loses the relative precision of the small result.
__device__ __forceinline__ float elu1(float v) { return v > 0.f ? v : expm1f(v); }
// The compile-time activation of the kernels that hard-code it (ACT = SONET_ACT_RELU or _ELU).
template <int ACT>
__device__ __forceinline__ float act_fn(float v) {
  if constexpr (ACT == SONET_ACT_ELU) return elu1(v);
  else if constexpr (ACT == SONET_ACT_RELU) return fmaxf(v, 0.f);
  else return v;
}

// ---- device helpers ---------------------------------------------------------------------------
// Running per-node maxima of the fused pool (csrc/pointmlp_tc.cu) are order-preserving int keys.
constexpr int POOL_KEY_INIT = static_cast<int>(0x80000000u);  // below the key of every float
// key -> value with the reference's semantics: the max must be > -1000 (index_max.cpp:80-81,103),
// otherwise the node gathers the feature of stacked copy 0 (models/networks.py:185).
__device__ __forceinline__ float pool_key_value(int key, float p0v) {
  const int bits = key ^ ((key >> 31) & 0x7fffffff);
  const float v = __int_as_float(bits);
  return (key != POOL_KEY_INIT && v > -1000.0f) ? v : p0v;
}
__device__ __forceinline__ float4 ldg_stream_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ float ldg_stream_f1(const float* p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}

// ---- fp32 pairs: IEEE round-to-nearest per half ---------------------------------------------------
// sm_90 has no packed fp32x2 instructions; each half is one explicitly rounded scalar op. __fadd_rn /
// __fmul_rn are never contracted into an FMA, which keeps (dx*dx + dy*dy) + dz*dz rounded like the
// reference and with it the bit-exact distance parity the arg-min kernels rely on.
__device__ __forceinline__ float2 add2_rn(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 mul2_rn(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 sqsum3_rn(float2 dx, float2 dy, float2 dz) {
  const float2 xx = mul2_rn(dx, dx), yy = mul2_rn(dy, dy), zz = mul2_rn(dz, dz);
  return make_float2(__fadd_rn(__fadd_rn(xx.x, yy.x), zz.x), __fadd_rn(__fadd_rn(xx.y, yy.y), zz.y));
}

// ---- the SOM assignment: each point's KK nearest nodes in registers -------------------------------
// The one rule of every kernel that assigns points to SOM nodes (som.cu, som_ragged.cu,
// seg_points.cu), which is why their indices agree bit for bit. The distance is ((dx*dx + dy*dy) +
// dz*dz) rounded op by op, no FMA (som_dist_rn; som.cu's packed pairs round each half the same way).
// The slots start at (+inf, -1) and take the nodes in ascending index order; a distance enters only
// when it is strictly below the last slot's, so on an exact tie the lower node index stays ahead,
// and a finite distance always enters while +inf and NaN never do. Slots still empty after the last
// node are filled by topk_fill_nonfinite.

// p + (-n) == p - n bit for bit: the arithmetic of som_assign_kernel's negated packed nodes.
__device__ __forceinline__ float som_dist_rn(float px, float py, float pz, float nx, float ny, float nz) {
  const float dx = __fadd_rn(px, -nx), dy = __fadd_rn(py, -ny), dz = __fadd_rn(pz, -nz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

template <int KK>
__device__ __forceinline__ void topk_reset(float (&bd)[KK], int (&bi)[KK]) {
#pragma unroll
  for (int s = 0; s < KK; ++s) {
    bd[s] = __int_as_float(0x7f800000);  // +inf
    bi[s] = -1;                          // empty (topk_fill_nonfinite)
  }
}

template <int KK>
__device__ __forceinline__ void topk_insert(float (&bd)[KK], int (&bi)[KK], float d, int m) {
  if (d < bd[KK - 1]) {  // strict: on exact ties the earlier (lower) node index stays
    bd[KK - 1] = d;
    bi[KK - 1] = m;
#pragma unroll
    for (int s = KK - 1; s > 0; --s) {
      if (bd[s] < bd[s - 1]) {
        const float td = bd[s];
        bd[s] = bd[s - 1];
        bd[s - 1] = td;
        const int ti = bi[s];
        bi[s] = bi[s - 1];
        bi[s - 1] = ti;
      }
    }
  }
}

// A point with fewer than KK nodes at a finite distance (a coordinate whose square overflows for
// some nodes, or a point that is not finite) leaves slots at -1. This fills them with the nodes at
// +inf, then the NaN ones, each in ascending index order, so that the KK nodes stay distinct and keep
// the order (distance, index) with NaN last: a NaN point gets nodes 0..KK-1. dist(m) must give the
// insertion loop's value for node m. Run only when bi[KK-1] < 0, which a finite point with KK finite
// distances never reaches.
template <int KK, typename Dist>
__device__ __forceinline__ void topk_fill_nonfinite(float (&bd)[KK], int (&bi)[KK], int M, Dist dist) {
  int filled = 0;
#pragma unroll
  for (int s = 0; s < KK; ++s) filled += bi[s] >= 0;
  for (int pass = 0; pass < 2; ++pass) {
    for (int m = 0; m < M && filled < KK; ++m) {
      const float d = dist(m);
      if (pass == 0 ? d == __int_as_float(0x7f800000) : d != d) {
#pragma unroll
        for (int s = 0; s < KK; ++s)   // register slots: no dynamic index
          if (s == filled) {
            bd[s] = d;
            bi[s] = m;
          }
        ++filled;
      }
    }
  }
}

// The KK nearest of M nodes, dist(m) the distance of node m (som_dist_rn).
template <int KK, typename Dist>
__device__ __forceinline__ void som_topk(int M, Dist dist, float (&bd)[KK], int (&bi)[KK]) {
  topk_reset(bd, bi);
  for (int m = 0; m < M; ++m) topk_insert(bd, bi, dist(m), m);
  if (bi[KK - 1] < 0) topk_fill_nonfinite(bd, bi, M, dist);
}

// ---- ragged clouds ----------------------------------------------------------------------------------
// Cloud b of a ragged batch of T rows is rows offsets[b] .. offsets[b+1]. Every offset is clamped
// into [0, T] and a decreasing pair is an empty cloud, so that no offsets array makes a kernel read
// or write out of range.
template <typename Off>
__device__ __forceinline__ long long ragged_offset(const Off* offsets, int b, long long T) {
  const long long o = __ldg(offsets + b);
  return o < 0 ? 0 : (o > T ? T : o);
}

// rows [lo, hi) of cloud b, hi >= lo
template <typename Off>
__device__ __forceinline__ void ragged_range(const Off* offsets, int b, long long T, long long& lo,
                                             long long& hi) {
  lo = ragged_offset(offsets, b, T);
  const long long e = __ldg(offsets + b + 1);
  hi = e < lo ? lo : (e > T ? T : e);
}

// The cloud of row g: the last b in [0, B) whose clamped offset is <= g (0 when there is none), and
// its rows [lo, hi); g lies in no cloud unless lo <= g < hi. For a row g in [0, T), a clamped offset
// is <= g exactly when the raw one is, so the search picks the cloud an unclamped search over the
// raw offsets would, for any offsets array.
template <typename Off>
__device__ __forceinline__ int ragged_find(const Off* offsets, int B, long long T, long long g,
                                           long long& lo, long long& hi) {
  int a = 0, z = B - 1;
  while (a < z) {
    const int mid = (a + z + 1) >> 1;
    if (ragged_offset(offsets, mid, T) <= g) a = mid;
    else z = mid - 1;
  }
  ragged_range(offsets, a, T, lo, hi);
  return a;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier / bulk-copy (TMA 1-D) wrappers ------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D bulk async copy global -> shared (TMA unit, SASS UBLKCP); size multiple of 16, 16B aligned.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

}  // namespace sonet
