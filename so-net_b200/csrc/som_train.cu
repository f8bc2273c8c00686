// som_train.cu — batch-SOM training (SURVEY.md §8f-4) for sm_90a.
//
// Replaces BatchSOM.batch_update / BatchSOM.optimize (util/som.py:295-366): T assign-and-update
// iterations per cloud. The reference materialises diff[B,3,N,M], a float one-hot mask [B,N,M] and
// a [B,3,N,M] masked product per iteration (2.6 GB of temporaries at B=64, N=5000) and launches
// ~25 ATen kernels per iteration; here one persistent CTA per cloud keeps the cloud, the nodes and
// the assignment in shared memory for all T iterations: HBM traffic is 12 B/point in and 12 B/node
// out per cloud, once.
//
// Per iteration (numerics follow the reference line by line):
//   1. assignment (util/som.py:301-309): d = ((x-n)**2).sum(1) evaluated as (dx*dx+dy*dy)+dz*dz
//      with separate roundings (no FMA) — bit-equal distances; torch.min -> first minimal index
//      (strict '<' over ascending node index).
//      Nodes are kept negated and packed two per register pair (add2_rn / mul2_rn, common.cuh).
//   2. per-node statistics (:313-321): count and coordinate sums. The reference's torch.sum is a
//      cascade summation (error ~1 ulp); sums here are accumulated in fp64 in a FIXED order and
//      rounded once to fp32 — measured: a plain fp32 accumulation drifts by 1e-7 per sum, which
//      flips assignments and moves nodes by up to 3e-2 after 80 iterations, the fp64 form agrees
//      with the reference to 1.2e-7. mean = sum / (count + 1e-5f) in fp32.
//   3. node update (:325-347): delta[c][j] = sum_m ((mean[c][m] - node[c][j]) * occupied[m])
//      * W_t[m][j] * lr_t, products rounded to fp32 in the reference's order, summed over m
//      (fp64 TwoSum accumulate, one fp32 rounding of the exact sum: exact_sum_to_float); node +=
//      delta.
// W_t (the neighbourhood weighting matrix of get_weighting_matrix, :232-235) and lr_t are inputs:
// the host computes the schedule with the reference's own expressions.
//
// Determinism: every reduction has a fixed order -> results are bit-reproducible and independent
// of the batch composition (shard invariance).
#include <algorithm>

#include "common.cuh"

namespace sonet {

constexpr int ST_THREADS = 1024;
constexpr int ST_WARPS = ST_THREADS / 32;
constexpr int ST_MAX_M = 256;

// fp32 nearest to hi + lo (an fp64 TwoSum accumulation: hi the running sum, lo its exact rounding
// errors). A plain (float)hi rounds twice: when two comparable terms sum exactly onto an fp32
// midpoint and a far smaller neighbourhood-tail term (W ~ 1e-21) decides the side, fp64 has
// dropped that term and ties-to-even may pick the wrong side. Rounding hi + lo to odd in fp64
// first keeps the sticky information, and odd-then-nearest with 53 >= 24 + 2 bits is one rounding.
__device__ __forceinline__ float exact_sum_to_float(double hi, double lo) {
  const double s = hi + lo, bb = s - hi;
  const double e = (hi - (s - bb)) + (lo - bb);           // s + e == hi + lo
  double r = s;
  if (e != 0.0 && (__double_as_longlong(s) & 1) == 0)   // inexact and even: step toward the rest
    r = nextafter(s, e > 0.0 ? HUGE_VAL : -HUGE_VAL);
  return __double2float_rn(r);
}

// smem: nodes as float4 [M] | mean float [3][M] + occupied [M] | W_t [M][M] (optional) |
//       x [3][N] (optional) | idx u8 [N]
__global__ void __launch_bounds__(ST_THREADS, 1)
    som_train_kernel(const float* __restrict__ x, const float* __restrict__ node_init,
                     int node_init_batched, const float* __restrict__ weights,
                     const float* __restrict__ lr, int T, int N, int M, int x_in_smem, int w_in_smem,
                     float* __restrict__ node_out, int32_t* __restrict__ idx_out) {
  extern __shared__ __align__(16) unsigned char st_smem[];
  float4* snode = reinterpret_cast<float4*>(st_smem);                  // [M]
  float* smean = reinterpret_cast<float*>(snode + M);                  // [3][M]
  float* socc = smean + 3 * M;                                         // [M]
  float2* spk = reinterpret_cast<float2*>(socc + M);                   // [3][MP] negated node pairs
  const int MP = (M + 1) >> 1;
  float* sw = reinterpret_cast<float*>(spk + 3 * MP);                  // [M][M] when w_in_smem
  float* sx = sw + (w_in_smem ? M * M : 0);                            // [3][N] when x_in_smem
  unsigned char* sidx =
      reinterpret_cast<unsigned char*>(sx + (x_in_smem ? 3 * static_cast<size_t>(N) : 0));

  const int b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* xg = x + static_cast<size_t>(b) * 3 * N;
  const float* ni = node_init + (node_init_batched ? static_cast<size_t>(b) * 3 * M : 0);
  for (int m = tid; m < M; m += ST_THREADS) snode[m] = make_float4(ni[m], ni[M + m], ni[2 * M + m], 0.f);
  // packed, negated copies of the nodes for the assignment (p - n == p + (-n) bit for bit; add2_rn /
  // mul2_rn round each half like the scalar ops, sums stay scalar — common.cuh); odd M: the last
  // pair repeats its node and the duplicate is skipped
  auto pack_nodes = [&]() {
    for (int m2 = tid; m2 < MP; m2 += ST_THREADS) {
      const float4 a = snode[2 * m2], b2 = snode[min(2 * m2 + 1, M - 1)];
      spk[m2] = make_float2(-a.x, -b2.x);
      spk[MP + m2] = make_float2(-a.y, -b2.y);
      spk[2 * MP + m2] = make_float2(-a.z, -b2.z);
    }
  };
  __syncthreads();
  pack_nodes();
  if (x_in_smem)
    for (int i = tid; i < 3 * N; i += ST_THREADS) sx[i] = xg[i];
  const float* xs = x_in_smem ? sx : xg;
  __syncthreads();

  // ---- 1. assignment of every point to its nearest node (sidx) ---------------------------------
  auto assign = [&]() {
    for (int n0 = tid; n0 < N; n0 += 2 * ST_THREADS) {
      const int n1 = n0 + ST_THREADS;
      const bool two = n1 < N;
      const float ax = xs[n0], ay = xs[N + n0], az = xs[2 * N + n0];
      const float bx = two ? xs[n1] : 0.f, by = two ? xs[N + n1] : 0.f,
                  bz = two ? xs[2 * N + n1] : 0.f;
      const float2 ax2 = make_float2(ax, ax), ay2 = make_float2(ay, ay), az2 = make_float2(az, az);
      const float2 bx2 = make_float2(bx, bx), by2 = make_float2(by, by), bz2 = make_float2(bz, bz);
      float da = __int_as_float(0x7f800000), db = da;
      int ia = 0, ib = 0;
#pragma unroll 2
      for (int m2 = 0; m2 < MP; ++m2) {
        const float2 qx = spk[m2], qy = spk[MP + m2], qz = spk[2 * MP + m2];
        const bool odd = 2 * m2 + 1 < M;
        float2 d = sqsum3_rn(add2_rn(ax2, qx), add2_rn(ay2, qy), add2_rn(az2, qz));
        if (d.x < da) { da = d.x; ia = 2 * m2; }
        if (odd && d.y < da) { da = d.y; ia = 2 * m2 + 1; }
        d = sqsum3_rn(add2_rn(bx2, qx), add2_rn(by2, qy), add2_rn(bz2, qz));
        if (d.x < db) { db = d.x; ib = 2 * m2; }
        if (odd && d.y < db) { db = d.y; ib = 2 * m2 + 1; }
      }
      sidx[n0] = static_cast<unsigned char>(ia);
      if (two) sidx[n1] = static_cast<unsigned char>(ib);
    }
  };

  for (int t = 0; t < T; ++t) {
    // this iteration's neighbourhood weights: issued now, consumed in step 3 — the 64 dependent-
    // latency L2 reads per thread of the first version cost more than the assignment
    if (w_in_smem) {
      const float* Wg = weights + static_cast<size_t>(t) * M * M;
      for (int i = tid; i < M * M; i += ST_THREADS) sw[i] = __ldg(Wg + i);
    }
    assign();
    __syncthreads();

    // ---- 2. per-node count / sums: warp per node, lanes stride the points, fixed order. The
    // assignment bytes are scanned four at a time (one 32-bit shared load + a SIMD byte compare:
    // 94 % of the words hold no point of the node and cost four instructions) ----
    for (int m = warp; m < M; m += ST_WARPS) {
      double s0 = 0.0, s1 = 0.0, s2 = 0.0;
      int cnt = 0;
      const uint32_t pat = static_cast<uint32_t>(m) * 0x01010101u;
      const uint32_t* sidx4 = reinterpret_cast<const uint32_t*>(sidx);
      const int nq = N >> 2;
      for (int q = lane; q < nq; q += 32) {
        uint32_t eq = __vcmpeq4(sidx4[q], pat);            // 0xff in every matching byte
        while (eq != 0) {
          const int byte = (__ffs(eq) - 1) >> 3;           // ascending point order inside the word
          const int n = 4 * q + byte;
          s0 += static_cast<double>(xs[n]);
          s1 += static_cast<double>(xs[N + n]);
          s2 += static_cast<double>(xs[2 * N + n]);
          ++cnt;
          eq &= ~(0xffu << (8 * byte));
        }
      }
      for (int n = 4 * nq + lane; n < N; n += 32) {          // tail (N % 4 points)
        if (sidx[n] == m) {
          s0 += static_cast<double>(xs[n]);
          s1 += static_cast<double>(xs[N + n]);
          s2 += static_cast<double>(xs[2 * N + n]);
          ++cnt;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      }
      if (lane == 0) {
        // mask_row_sum = sum(mask) + 0.00001 (fp32), mean = masked_sum / mask_row_sum (:313-321)
        const float den = __fadd_rn(static_cast<float>(cnt), 0.00001f);
        smean[m] = __fdiv_rn(static_cast<float>(s0), den);
        smean[M + m] = __fdiv_rn(static_cast<float>(s1), den);
        smean[2 * M + m] = __fdiv_rn(static_cast<float>(s2), den);
        socc[m] = cnt > 0 ? 1.f : 0.f;
      }
    }
    __syncthreads();

    // ---- 3. node update: thread per (c, j) ----------------------------------------------------
    const float* W = w_in_smem ? sw : weights + static_cast<size_t>(t) * M * M;   // W[m][j]
    const float lrt = __ldg(lr + t);
    float newv = 0.f;
    const bool upd = tid < 3 * M;
    if (upd) {
      const int c = tid / M, j = tid - c * M;
      const float4 q = snode[j];
      const float nj = c == 0 ? q.x : (c == 1 ? q.y : q.z);
      double hi = 0.0, lo = 0.0;
      for (int m = 0; m < M; ++m) {
        const float diff = __fmul_rn(__fsub_rn(smean[c * M + m], nj), socc[m]);
        const double term =
            static_cast<double>(__fmul_rn(__fmul_rn(diff, W[static_cast<size_t>(m) * M + j]), lrt));
        const double s = hi + term, bb = s - hi;
        lo += (hi - (s - bb)) + (term - bb);
        hi = s;
      }
      newv = __fadd_rn(nj, exact_sum_to_float(hi, lo));
    }
    __syncthreads();   // every thread has read the old nodes
    if (upd) {
      const int c = tid / M, j = tid - c * M;
      float* p = reinterpret_cast<float*>(snode + j);
      p[c] = newv;
    }
    __syncthreads();
    pack_nodes();
    __syncthreads();
  }

  float* no = node_out + static_cast<size_t>(b) * 3 * M;
  for (int i = tid; i < 3 * M; i += ST_THREADS) {
    const int c = i / M, j = i - c * M;
    no[i] = reinterpret_cast<const float*>(snode + j)[c];
  }
  if (idx_out != nullptr) {
    // assignment of the LAST iteration (w.r.t. the nodes before its update); with T = 0 the
    // assignment against the initial nodes, by the same arithmetic as iteration 1
    if (T == 0) {
      assign();
      __syncthreads();
    }
    for (int n = tid; n < N; n += ST_THREADS) idx_out[static_cast<size_t>(b) * N + n] = sidx[n];
  }
}

}  // namespace sonet

extern "C" int sonet_som_train(const float* x, const float* node_init, int node_init_batched,
                               const float* weights, const float* lr, int T, int B, int N, int M,
                               float* node_out, int32_t* last_idx, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && N >= 0 && T >= 0, "som_train: negative dimension");
  SONET_REQUIRE(M >= 1 && M <= ST_MAX_M, "som_train: M=%d out of range [1,%d]", M, ST_MAX_M);
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(x && node_init && node_out && (T == 0 || (weights && lr)), "som_train: null pointer");
  const int w_in_smem = (static_cast<size_t>(M) * M * sizeof(float) <= 64 * 1024) ? 1 : 0;
  const size_t fixed = sizeof(float4) * M + sizeof(float) * 4 * M + sizeof(float2) * 3 * ((M + 1) / 2) +
                       (w_in_smem ? sizeof(float) * M * M : 0);
  const size_t with_x = fixed + sizeof(float) * 3 * static_cast<size_t>(N) + static_cast<size_t>(N) + 16;
  const size_t without_x = fixed + static_cast<size_t>(N) + 16;
  const size_t cap = static_cast<size_t>(max_smem_optin());
  const int x_in_smem = with_x <= cap ? 1 : 0;
  const size_t smem = x_in_smem ? with_x : without_x;
  SONET_REQUIRE(smem <= cap, "som_train: N=%d does not fit the per-CTA assignment table (%zu > %zu B)",
                N, smem, cap);
  cudaFuncSetAttribute(som_train_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       static_cast<int>(smem));
  som_train_kernel<<<B, ST_THREADS, smem, as_stream(stream)>>>(
      x, node_init, node_init_batched, weights, lr, T, N, M, x_in_smem, w_in_smem, node_out, last_idx);
  return check_launch("som_train");
}
