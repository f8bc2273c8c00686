// tc_probe.cu — diagnostic kernel: one 128 x N x K bf16 GEMM on Hopper wgmma with A from shared
// memory (SS) or from registers (RS), fp32 accumulate in registers. Used by
// tests/test_gpu_tcgen05.py to pin the shared-memory descriptor encoding (LBO/SBO roles) and the
// K-major no-swizzle operand layout that the point-MLP kernels rely on. Not on the product path.
#include "tc_common.cuh"

namespace sonet {

__device__ __forceinline__ uint32_t canon_off(int r, int k, uint32_t lbo, uint32_t sbo) {
  // K-major, no swizzle: 8x16B core matrices; k/8 chunks strided by LBO, r/8 groups by SBO
  return (r >> 3) * sbo + (k >> 3) * lbo + (r & 7) * 16 + (k & 7) * 2;
}

template <int N>
__device__ __forceinline__ void probe_mma(float (&acc)[N / 2], uint64_t adesc, const uint32_t (&a)[4],
                                          uint64_t bdesc, int mode) {
  if constexpr (N == 16) {
    if (mode == 0) tc::wgmma_bf16_n16(acc, adesc, bdesc, 1); else tc::wgmma_bf16_rs_n16(acc, a, bdesc, 1);
  } else if constexpr (N == 32) {
    if (mode == 0) tc::wgmma_bf16_n32(acc, adesc, bdesc, 1); else tc::wgmma_bf16_rs_n32(acc, a, bdesc, 1);
  } else if constexpr (N == 64) {
    if (mode == 0) tc::wgmma_bf16_n64(acc, adesc, bdesc, 1); else tc::wgmma_bf16_rs_n64(acc, a, bdesc, 1);
  } else {
    if (mode == 0) tc::wgmma_bf16_n128(acc, adesc, bdesc, 1); else tc::wgmma_bf16_rs_n128(acc, a, bdesc, 1);
  }
}

template <int N>
__global__ void __launch_bounds__(128, 1)
    tc_probe_kernel(const float* __restrict__ A, const float* __restrict__ Bm, int K, int mode,
                    uint32_t lbo_a, uint32_t sbo_a, uint32_t lbo_b, uint32_t sbo_b,
                    int swap_fields, float* __restrict__ D) {
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* a_img = smem;
  unsigned char* b_img = smem + 128 * K * 2;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  for (int i = tid; i < 128 * K; i += 128) {
    const int r = i / K, k = i % K;
    *reinterpret_cast<__nv_bfloat16*>(a_img + canon_off(r, k, lbo_a, sbo_a)) =
        __float2bfloat16_rn(A[i]);
  }
  for (int i = tid; i < N * K; i += 128) {
    const int r = i / K, k = i % K;
    *reinterpret_cast<__nv_bfloat16*>(b_img + canon_off(r, k, lbo_b, sbo_b)) =
        __float2bfloat16_rn(Bm[i]);
  }
  tc::fence_proxy_async();
  __syncthreads();

  // accumulator / register-A fragment: rows g and g + 8 (g = 16*warp + lane/4), k / n pairs at
  // 2*(lane%4)
  const int g = 16 * warp + (lane >> 2), c2 = 2 * (lane & 3);
  for (int h = 0; h < 2; ++h) {   // two M=64 halves of the 128-row tile
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    tc::wg_fence();
    for (int ks = 0; ks < K / 16; ++ks) {
      // one K step = 16 bf16 = two 16-byte core matrices along K
      const uint32_t a_addr = smem_u32(a_img) + 8 * h * sbo_a + 2 * ks * lbo_a;
      const uint32_t b_addr = smem_u32(b_img) + 2 * ks * lbo_b;
      const uint64_t adesc = swap_fields ? tc::smem_desc(a_addr, sbo_a, lbo_a)
                                         : tc::smem_desc(a_addr, lbo_a, sbo_a);
      const uint64_t bdesc = swap_fields ? tc::smem_desc(b_addr, sbo_b, lbo_b)
                                         : tc::smem_desc(b_addr, lbo_b, sbo_b);
      uint32_t a[4] = {0, 0, 0, 0};
      if (mode == 1) {
        const float* r0 = A + static_cast<size_t>(64 * h + g) * K + 16 * ks + c2;
        const float* r1 = r0 + 8 * K;
        a[0] = tc::pack_bf16x2(r0[0], r0[1]);
        a[1] = tc::pack_bf16x2(r1[0], r1[1]);
        a[2] = tc::pack_bf16x2(r0[8], r0[9]);
        a[3] = tc::pack_bf16x2(r1[8], r1[9]);
      }
      probe_mma<N>(acc, adesc, a, bdesc, mode);
    }
    tc::wg_commit();
    tc::wg_wait<0>();
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        D[static_cast<size_t>(64 * h + g + 8 * (e >> 1)) * N + 8 * j + c2 + (e & 1)] = acc[4 * j + e];
  }
}

}  // namespace sonet

extern "C" int sonet_debug_tc_probe(const float* A, const float* Bm, int N, int K, int mode,
                                    int layout, int swap_fields, float* D, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(N == 16 || N == 32 || N == 64 || N == 128, "tc_probe: N must be 16, 32, 64 or 128");
  SONET_REQUIRE(K >= 16 && K <= 256 && K % 32 == 0, "tc_probe: K must be a multiple of 32 in [32,256]");
  SONET_REQUIRE(mode == 0 || mode == 1, "tc_probe: mode must be 0 (A in shared memory) or 1 (registers)");
  SONET_REQUIRE(A && Bm && D, "tc_probe: null pointer");
  uint32_t lbo_a, sbo_a, lbo_b, sbo_b;
  if (layout == 0) {  // K chunks adjacent (128 B apart), 8-row groups K*16 B apart
    lbo_a = lbo_b = 128;
    sbo_a = sbo_b = static_cast<uint32_t>(K) * 16;
  } else {            // 8-row groups adjacent, K chunks rows*16 B apart
    sbo_a = sbo_b = 128;
    lbo_a = 128 * 16;
    lbo_b = static_cast<uint32_t>(N) * 16;
  }
  const size_t smem = static_cast<size_t>(128 + N) * K * 2;
  auto kern = N == 16 ? tc_probe_kernel<16> : N == 32 ? tc_probe_kernel<32>
            : N == 64 ? tc_probe_kernel<64> : tc_probe_kernel<128>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  kern<<<1, 128, smem, as_stream(stream)>>>(A, Bm, K, mode, lbo_a, sbo_a, lbo_b, sbo_b, swap_fields, D);
  return check_launch("tc_probe");
}

// ---- MMA rate microbenchmark: `iters` back-to-back M=64 x N x 16 fp16 wgmmas of one warpgroup, B in
// shared memory, A in shared memory (RS = false) or in registers (RS = true) ----------------------
namespace sonet {
template <int N, bool RS>
__global__ void __launch_bounds__(128, 1)
    tc_rate_kernel(uint32_t sbo, int iters, long long* __restrict__ cycles) {
  extern __shared__ __align__(1024) unsigned char smem[];
  for (int i = threadIdx.x; i < 48 * 1024 / 4; i += 128) reinterpret_cast<uint32_t*>(smem)[i] = 0x3c003c00u;
  tc::fence_proxy_async();
  __syncthreads();
  const uint32_t a_addr = smem_u32(smem), b_addr = smem_u32(smem) + 16384;
  const uint64_t ad = tc::smem_desc(a_addr, 128, sbo), bd = tc::smem_desc(b_addr, 128, sbo);
  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  const uint32_t a[4] = {0x3c003c00u, 0x3c003c00u, 0x3c003c00u, 0x3c003c00u};   // fp16 1.0 pairs
  const long long t0 = clock64();
  tc::wg_fence();
  for (int i = 0; i < iters; ++i) {
    if constexpr (RS && N == 96) tc::wgmma_f16_rs_n96(acc, a, bd + (i & 3) * 16, 1);
    else if constexpr (RS && N == 128) tc::wgmma_f16_rs_n128(acc, a, bd + (i & 3) * 16, 1);
    else if constexpr (RS) tc::wgmma_f16_rs_n256(acc, a, bd + (i & 3) * 16, 1);
    else if constexpr (N == 64) tc::wgmma_f16_n64(acc, ad + (i & 3) * 16, bd + (i & 3) * 16, 1);
    else if constexpr (N == 96) tc::wgmma_f16_n96(acc, ad + (i & 3) * 16, bd + (i & 3) * 16, 1);
    else if constexpr (N == 128) tc::wgmma_f16_n128(acc, ad + (i & 3) * 16, bd + (i & 3) * 16, 1);
    else tc::wgmma_f16_n256(acc, ad + (i & 3) * 16, bd + (i & 3) * 16, 1);
  }
  tc::wg_commit();
  tc::wg_wait<0>();
  const long long t1 = clock64();
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) s += acc[i];
  if (threadIdx.x == 0) {
    cycles[0] = t1 - t0;
    if (s == 12345.f) cycles[1] = 0;   // keeps the accumulators live
  }
}
}  // namespace sonet

extern "C" int sonet_debug_tc_mma_rate(int mode, int N, int sbo, int iters, long long* cycles,
                                       sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(cycles && ((mode == 0 && (N == 64 || N == 96 || N == 128 || N == 256)) ||
                           (mode == 1 && (N == 96 || N == 128 || N == 256))),
                "tc_mma_rate: mode 0 with N in {64, 96, 128, 256} or mode 1 with N in {96, 128, 256}");
  auto kern = mode == 1 ? (N == 96 ? tc_rate_kernel<96, true> : N == 128 ? tc_rate_kernel<128, true>
                                                                       : tc_rate_kernel<256, true>)
            : N == 64 ? tc_rate_kernel<64, false> : N == 96 ? tc_rate_kernel<96, false>
            : N == 128 ? tc_rate_kernel<128, false> : tc_rate_kernel<256, false>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
  kern<<<1, 128, 64 * 1024, as_stream(stream)>>>(static_cast<uint32_t>(sbo), iters, cycles);
  return check_launch("tc_mma_rate");
}
