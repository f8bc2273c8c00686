// som.cu — SOM node <-> point assignment for sm_90a.
//
// Replaces BatchSOM.query_topk (util/som.py:237-269) and the dense-mask arithmetic that
// Encoder.forward builds on top of it (models/networks.py:127-143, 168-172). The reference
// materialises diff[B,3,N,M], dist[B,N,M], a [B,N,M,k] compare and two [B,3,kN,M] products
// (~2 GB at B=64,N=5000); here the assignment is 12 B in + 4k B out per point and the cluster
// statistics are reduced straight from the indices.
//
//  som_assign_kernel   thread per point: the nodes in smem (broadcast reads), two distances per step
//                      from packed pairs, the SOM assignment rule of common.cuh (som_topk).
//  som_stats_kernel    CTA per (cloud, node): counts and coordinate sums in a fixed order
//                      (strided per-thread partials + fixed tree) -> bit-reproducible and
//                      independent of batch sharding; cluster_mean = sum / (count + 1e-5f).
//  som_mask_kernel     optional dense one-hot mask [B,kN,M] int32 (the API of query_topk):
//                      pure 16-byte streaming stores.
//  som_decenter_kernel centers / x_decentered / x_augmented (networks.py:168-172).
#include <algorithm>

#include "common.cuh"

namespace sonet {

constexpr int SOM_MAX_M = 256;
constexpr int SOM_MAX_K = 4;

template <int KK>
__global__ void __launch_bounds__(256)
    som_assign_kernel(const float* __restrict__ x, const float* __restrict__ node, int N, int M,
                      int32_t* __restrict__ idx32, int64_t* __restrict__ idx64,
                      int32_t* __restrict__ row_flag, int32_t* __restrict__ mask) {
  // nodes NEGATED and packed two per register pair: p - n == p + (-n) bit for bit, and the packed
  // add/mul round each half like the scalar ops (sums stay scalar: common.cuh)
  __shared__ float2 snx[SOM_MAX_M / 2], sny[SOM_MAX_M / 2], snz[SOM_MAX_M / 2];
  const int b = blockIdx.y;
  const float* nb = node + static_cast<size_t>(b) * 3 * M;
  const int MP = (M + 1) >> 1;
  for (int m2 = threadIdx.x; m2 < MP; m2 += blockDim.x) {
    const int m0 = 2 * m2, m1 = min(2 * m2 + 1, M - 1);   // odd M: the last pair repeats its node
    snx[m2] = make_float2(-nb[m0], -nb[m1]);
    sny[m2] = make_float2(-nb[M + m0], -nb[M + m1]);
    snz[m2] = make_float2(-nb[2 * M + m0], -nb[2 * M + m1]);
  }
  __syncthreads();

  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = n < N;
  if (!live && mask == nullptr) return;   // (with a fused mask the whole warp stays for the shuffles)
  const float* xb = x + static_cast<size_t>(b) * 3 * N;
  const int nl = live ? n : 0;
  const float px = xb[nl], py = xb[N + nl], pz = xb[2 * N + nl];
  const float2 px2 = make_float2(px, px), py2 = make_float2(py, py), pz2 = make_float2(pz, pz);

  // som_topk's rule (common.cuh), with the distances of two nodes per step
  float bd[KK];
  int bi[KK];
  topk_reset(bd, bi);
#pragma unroll 2
  for (int m2 = 0; m2 < MP; ++m2) {
    const float2 d = sqsum3_rn(add2_rn(px2, snx[m2]), add2_rn(py2, sny[m2]), add2_rn(pz2, snz[m2]));
    topk_insert(bd, bi, d.x, 2 * m2);
    if (2 * m2 + 1 < M) topk_insert(bd, bi, d.y, 2 * m2 + 1);
  }
  if (bi[KK - 1] < 0) {
    topk_fill_nonfinite(bd, bi, M, [&](int m) {
      const float2 nx = snx[m >> 1], ny = sny[m >> 1], nz = snz[m >> 1];
      return som_dist_rn(px, py, pz, -((m & 1) ? nx.y : nx.x), -((m & 1) ? ny.y : ny.x),
                         -((m & 1) ? nz.y : nz.x));
    });
  }
  if (mask != nullptr) {
    // Fused dense one-hot mask (util/som.py:255-265), M % 32 == 0: the warp writes the KK rows of
    // each of its 32 points cooperatively — every lane M/32 consecutive ints of a row, so a row
    // (M*4 bytes) is one coalesced store instruction; the index comes from the owning lane by
    // shuffle. 4 B/point read, 4*M*KK B/point written: pure HBM streaming.
    const int lane = threadIdx.x & 31;
    const int n_base = n - lane;                  // first point of this warp
    const size_t mrow0 = static_cast<size_t>(b) * KK * N;
    if (M == 64 && (reinterpret_cast<uintptr_t>(mask) & 15u) == 0) {
      // M = 64: a mask row is 256 B = 16 lanes x 16 B -> one warp store instruction writes TWO
      // rows (lanes 0-15 the row of point r, lanes 16-31 the row of point r+1) as 128-bit streaming
      // stores (r01: 8-byte stores, 59 % of the HBM copy peak; the store width was the limiter)
      const int half = lane >> 4, q = lane & 15;  // which of the two rows; which 4 nodes of it
      for (int r = 0; r < 32; r += 2) {
        if (n_base + r >= N) break;               // warp-uniform
#pragma unroll
        for (int s = 0; s < KK; ++s) {
          const int id = __shfl_sync(0xffffffffu, bi[s], r + half) - 4 * q;
          if (n_base + r + half < N) {
            int4* dst = reinterpret_cast<int4*>(
                mask + (mrow0 + static_cast<size_t>(s) * N + n_base + r + half) * 64) + q;
            __stcs(dst, make_int4(id == 0, id == 1, id == 2, id == 3));
          }
        }
      }
    } else {
      const int per = M >> 5;                       // ints per lane and row
      for (int r = 0; r < 32; ++r) {
        if (n_base + r >= N) break;                 // warp-uniform
#pragma unroll
        for (int s = 0; s < KK; ++s) {
          const int id = __shfl_sync(0xffffffffu, bi[s], r);
          int32_t* dst = mask + (mrow0 + static_cast<size_t>(s) * N + n_base + r) * M + lane * per;
          if (per == 2) {
            __stcs(reinterpret_cast<int2*>(dst), make_int2(id == 2 * lane, id == 2 * lane + 1));
          } else {
            for (int e = 0; e < per; ++e) dst[e] = (id == lane * per + e) ? 1 : 0;
          }
        }
      }
    }
  }
  if (!live) return;
  const size_t o = static_cast<size_t>(b) * KK * N + n;
#pragma unroll
  for (int s = 0; s < KK; ++s) {
    idx32[o + static_cast<size_t>(s) * N] = bi[s];
    if (idx64 != nullptr) idx64[o + static_cast<size_t>(s) * N] = bi[s];
    // occupancy flag (mask_row_max) without the statistics pass: every writer stores the same 1
    if (row_flag != nullptr) row_flag[static_cast<size_t>(b) * M + bi[s]] = 1;
  }
}

constexpr int STATS_THREADS = 256;

__global__ void __launch_bounds__(STATS_THREADS)
    som_stats_kernel(const float* __restrict__ x, const int32_t* __restrict__ idx32, int N, int M,
                     int k, int32_t* __restrict__ count, int32_t* __restrict__ row_max,
                     float* __restrict__ cluster_mean) {
  const int m = blockIdx.x, b = blockIdx.y;
  const int kN = k * N;
  const int32_t* ib = idx32 + static_cast<size_t>(b) * kN;
  const float* xb = x + static_cast<size_t>(b) * 3 * N;
  float sx = 0.f, sy = 0.f, sz = 0.f;
  int cnt = 0;
  // the stacked point order j = s*N + n is the reference's x_stack order (networks.py:132-137).
  // Per-thread order is fixed (depends only on N), so the sums are bit-reproducible.
  auto take = [&](int j) {
    int n = j;
    while (n >= N) n -= N;
    sx += xb[n];
    sy += xb[N + n];
    sz += xb[2 * N + n];
    ++cnt;
  };
  if ((kN & 3) == 0 && (reinterpret_cast<uintptr_t>(ib) & 15u) == 0) {
    // 128-bit index loads, 2 in flight per thread: the scan is latency-bound, not bandwidth-bound
    const int4* ib4 = reinterpret_cast<const int4*>(ib);
    const int nq = kN >> 2;
    for (int q0 = threadIdx.x; q0 < nq; q0 += 2 * STATS_THREADS) {
      const int q1 = q0 + STATS_THREADS;
      const int4 a = __ldg(ib4 + q0);
      const int4 c = (q1 < nq) ? __ldg(ib4 + q1) : make_int4(-1, -1, -1, -1);
      if (a.x == m) take(4 * q0);
      if (a.y == m) take(4 * q0 + 1);
      if (a.z == m) take(4 * q0 + 2);
      if (a.w == m) take(4 * q0 + 3);
      if (c.x == m) take(4 * q1);
      if (c.y == m) take(4 * q1 + 1);
      if (c.z == m) take(4 * q1 + 2);
      if (c.w == m) take(4 * q1 + 3);
    }
  } else {
    for (int j = threadIdx.x; j < kN; j += STATS_THREADS)
      if (ib[j] == m) take(j);
  }
  __shared__ float rs[3][STATS_THREADS];
  __shared__ int rc[STATS_THREADS];
  rs[0][threadIdx.x] = sx;
  rs[1][threadIdx.x] = sy;
  rs[2][threadIdx.x] = sz;
  rc[threadIdx.x] = cnt;
  __syncthreads();
  for (int w = STATS_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      rs[0][threadIdx.x] += rs[0][threadIdx.x + w];
      rs[1][threadIdx.x] += rs[1][threadIdx.x + w];
      rs[2][threadIdx.x] += rs[2][threadIdx.x + w];
      rc[threadIdx.x] += rc[threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int c = rc[0];
    count[static_cast<size_t>(b) * M + m] = c;
    row_max[static_cast<size_t>(b) * M + m] = c > 0 ? 1 : 0;
    const float den = __fadd_rn(static_cast<float>(c), 1e-5f);
    float* cm = cluster_mean + static_cast<size_t>(b) * 3 * M;
    cm[m] = __fdiv_rn(rs[0][0], den);
    cm[M + m] = __fdiv_rn(rs[1][0], den);
    cm[2 * M + m] = __fdiv_rn(rs[2][0], den);
  }
}

// mask[b, j, m] = (idx[b,j] == m): one thread writes 4 consecutive m as an int4.
__global__ void __launch_bounds__(256)
    som_mask_kernel(const int32_t* __restrict__ idx32, long long rows, int M,
                    int32_t* __restrict__ mask) {
  const int quads = M >> 2;  // M % 4 == 0 on this path
  const long long total = rows * quads;
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = t / quads;
    const int q = static_cast<int>(t - r * quads);
    const int id = __ldg(idx32 + r) - (q << 2);
    int4 v = make_int4(id == 0, id == 1, id == 2, id == 3);
    __stcs(reinterpret_cast<int4*>(mask + r * M) + q, v);
  }
}
__global__ void __launch_bounds__(256)
    som_mask_scalar_kernel(const int32_t* __restrict__ idx32, long long rows, int M,
                           int32_t* __restrict__ mask) {
  const long long total = rows * M;
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = t / M;
    mask[t] = (__ldg(idx32 + r) == static_cast<int>(t - r * M)) ? 1 : 0;
  }
}

__global__ void __launch_bounds__(256)
    som_decenter_kernel(const float* __restrict__ x, const float* __restrict__ sn,
                        const float* __restrict__ cluster_mean, const int32_t* __restrict__ idx32,
                        int N, int M, int k, float* __restrict__ centers,
                        float* __restrict__ x_aug) {
  extern __shared__ float scm[];  // [3][M]
  const int b = blockIdx.y;
  const float* cm = cluster_mean + static_cast<size_t>(b) * 3 * M;
  for (int i = threadIdx.x; i < 3 * M; i += blockDim.x) scm[i] = cm[i];
  __syncthreads();
  const int kN = k * N;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= kN) return;
  int n = j;
  while (n >= N) n -= N;
  int id = idx32[static_cast<size_t>(b) * kN + j];
  id = min(max(id, 0), M - 1);
  const float* xb = x + static_cast<size_t>(b) * 3 * N;
  const int CA = sn ? 6 : 3;
  float* ab = x_aug + static_cast<size_t>(b) * CA * kN;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float ctr = scm[c * M + id];
    if (centers) centers[(static_cast<size_t>(b) * 3 + c) * kN + j] = ctr;
    ab[static_cast<size_t>(c) * kN + j] = __fsub_rn(xb[c * N + n], ctr);
  }
  if (sn) {
    const float* sb = sn + static_cast<size_t>(b) * 3 * N;
#pragma unroll
    for (int c = 0; c < 3; ++c) ab[static_cast<size_t>(3 + c) * kN + j] = sb[c * N + n];
  }
}

}  // namespace sonet

static int som_assign_impl(const float* x, const float* node, int B, int N, int M, int k,
                           int32_t* min_idx_i32, int64_t* min_idx_i64, int32_t* count,
                           int32_t* row_max, float* cluster_mean, int32_t* fused_mask,
                           sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && N >= 0, "som_assign: negative dimension");
  SONET_REQUIRE(M >= 1 && M <= SOM_MAX_M, "som_assign: M=%d out of range [1,%d]", M, SOM_MAX_M);
  SONET_REQUIRE(k >= 1 && k <= SOM_MAX_K && k <= M,
                "som_assign: k=%d out of range [1,%d] (and k <= M=%d)", k, SOM_MAX_K, M);
  SONET_REQUIRE(B <= 65535, "som_assign: B=%d exceeds grid limit", B);
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(x && node && min_idx_i32, "som_assign: null pointer");
  SONET_REQUIRE((count && row_max && cluster_mean) || (!count && !cluster_mean),
                "som_assign: count and cluster_mean go together (row_max alone is allowed)");
  cudaStream_t st = as_stream(stream);
  // row_max without statistics (the query_topk API): flags written by the assignment kernel itself
  int32_t* row_flag = (row_max && !count) ? row_max : nullptr;
  if (row_flag) cudaMemsetAsync(row_flag, 0, sizeof(int32_t) * static_cast<size_t>(B) * M, st);
  if (N > 0) {
    dim3 grid((N + 255) / 256, B);
    switch (k) {
      case 1: som_assign_kernel<1><<<grid, 256, 0, st>>>(x, node, N, M, min_idx_i32, min_idx_i64, row_flag, fused_mask); break;
      case 2: som_assign_kernel<2><<<grid, 256, 0, st>>>(x, node, N, M, min_idx_i32, min_idx_i64, row_flag, fused_mask); break;
      case 3: som_assign_kernel<3><<<grid, 256, 0, st>>>(x, node, N, M, min_idx_i32, min_idx_i64, row_flag, fused_mask); break;
      default: som_assign_kernel<4><<<grid, 256, 0, st>>>(x, node, N, M, min_idx_i32, min_idx_i64, row_flag, fused_mask); break;
    }
    int rc = check_launch("som_assign");
    if (rc) return rc;
  }
  if (count) {
    som_stats_kernel<<<dim3(M, B), STATS_THREADS, 0, st>>>(x, min_idx_i32, N, M, k, count, row_max,
                                                          cluster_mean);
    return check_launch("som_stats");
  }
  return SONET_OK;
}

extern "C" int sonet_som_assign(const float* x, const float* node, int B, int N, int M, int k,
                                int32_t* min_idx_i32, int64_t* min_idx_i64, int32_t* count,
                                int32_t* row_max, float* cluster_mean, sonet_stream_t stream) {
  return som_assign_impl(x, node, B, N, M, k, min_idx_i32, min_idx_i64, count, row_max, cluster_mean,
                         nullptr, stream);
}

extern "C" int sonet_som_query_topk(const float* x, const float* node, int B, int N, int M, int k,
                                    int32_t* mask, int32_t* row_max, int64_t* min_idx_i64,
                                    int32_t* min_idx_i32, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(mask && row_max && min_idx_i32, "som_query_topk: null pointer");
  if (M % 32 != 0 || (M / 32 == 2 && (reinterpret_cast<uintptr_t>(mask) & 7u))) {
    int rc = som_assign_impl(x, node, B, N, M, k, min_idx_i32, min_idx_i64, nullptr, row_max, nullptr,
                             nullptr, stream);
    return rc ? rc : sonet_som_mask(min_idx_i32, B, k * N, M, mask, stream);
  }
  return som_assign_impl(x, node, B, N, M, k, min_idx_i32, min_idx_i64, nullptr, row_max, nullptr,
                         mask, stream);
}

extern "C" int sonet_som_mask(const int32_t* min_idx_i32, int B, int kN, int M, int32_t* mask,
                              sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && kN >= 0 && M >= 1, "som_mask: bad dimension");
  const long long rows = static_cast<long long>(B) * kN;
  if (rows == 0) return SONET_OK;
  SONET_REQUIRE(min_idx_i32 && mask, "som_mask: null pointer");
  cudaStream_t st = as_stream(stream);
  const int sms = sm_count();
  if (M % 4 == 0 && aligned16(mask)) {
    const long long total = rows * (M >> 2);
    const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, 16LL * sms));
    som_mask_kernel<<<grid, 256, 0, st>>>(min_idx_i32, rows, M, mask);
  } else {
    const long long total = rows * M;
    const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, 16LL * sms));
    som_mask_scalar_kernel<<<grid, 256, 0, st>>>(min_idx_i32, rows, M, mask);
  }
  return check_launch("som_mask");
}

extern "C" int sonet_som_decenter(const float* x, const float* sn, const float* cluster_mean,
                                  const int32_t* min_idx_i32, int B, int N, int M, int k,
                                  float* centers, float* x_aug, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && N >= 0 && M >= 1 && k >= 1, "som_decenter: bad dimension");
  SONET_REQUIRE(B <= 65535, "som_decenter: B=%d exceeds grid limit", B);
  if (B == 0 || N == 0) return SONET_OK;
  SONET_REQUIRE(x && cluster_mean && min_idx_i32 && x_aug, "som_decenter: null pointer");
  const int kN = k * N;
  dim3 grid((kN + 255) / 256, B);
  som_decenter_kernel<<<grid, 256, 3 * M * sizeof(float), as_stream(stream)>>>(
      x, sn, cluster_mean, min_idx_i32, N, M, k, centers, x_aug);
  return check_launch("som_decenter");
}
