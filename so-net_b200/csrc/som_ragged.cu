// som_ragged.cu — the encoder's stage before the first per-node max over RAGGED clouds
// (networks.Encoder.forward_ragged): every point of each cloud, whatever its size, in one batch.
//
// points [T,6] f32 (xyz | normal); cloud b owns rows offsets[b] .. offsets[b+1] (P_b points). Its k
// stacked copies are the columns k*offsets[b] + s*P_b + n (copy s of point n: the reference's x_stack
// order at N = P_b, models/networks.py:132-137), so the copies of the batch fill k*T columns with each
// cloud's block where the dense [B,k*N] layout would put it at N = P_b.
//
//   som_assign_ragged_kernel        thread per point: its cloud by binary search over offsets, then the
//                                   k nearest of the cloud's M nodes by the SOM assignment rule of
//                                   common.cuh (som_topk, sonet_som_assign's bits). count [B,M] by
//                                   integer atomics, row_max [B,M] = count > 0.
//   som_group_ragged_kernel         CTA per cloud, any size: stable counting sort of the cloud's copies
//                                   by node through global memory (warp-private histograms over
//                                   warp-contiguous ranges, ballot ranks), then per-node sums in
//                                   som_group_kernel's order (csrc/som_sort.cu: a node's copies in
//                                   ascending stacked order, lane l sums copies l, l+32, ... in groups
//                                   of four rows, xor butterfly 16, 8, 4, 2, 1), cluster_mean =
//                                   sum / (count + 1e-5), then the decentred copies in sorted order.
//                                   A cloud's cluster means are the dense group route's bits at
//                                   N = P_b, also for clouds too large for that kernel's shared memory.
//   som_decenter_ragged_kernel      the decentred copies in stacked order (the unfused route's input).
//
// Offsets are clamped as common.cuh's ragged_range states, so that no input reads or writes out of
// range; the Python caller refuses such offsets before any launch. Offsets that decrease can leave
// two clouds' clamped ranges overlapping: their CTAs in som_group_ragged_kernel then share columns of
// node_sorted, which holds each CTA's packed sort entries, and one CTA can read the other's entries
// or flat ids there. Every entry is read back clamped to the CTA's own points and nodes, so such
// columns hold unspecified values but no access leaves the cloud's rows.
#include <algorithm>

#include "common.cuh"

namespace sonet {

constexpr int RAG_MAX_M = 256;
constexpr int RAG_MAX_K = 4;
constexpr int RAG_THREADS = 256;
constexpr int RGROUP_THREADS = 1024, RGROUP_WARPS = RGROUP_THREADS / 32;

template <int KK>
__global__ void __launch_bounds__(RAG_THREADS)
    som_assign_ragged_kernel(const float* __restrict__ points, long long T,
                             const long long* __restrict__ offsets, int B,
                             const float* __restrict__ node, int M, int32_t* __restrict__ min_idx,
                             int32_t* __restrict__ count, int32_t* __restrict__ row_max) {
  const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g >= T) return;
  long long lo, hi;
  const int b = ragged_find(offsets, B, T, g, lo, hi);
  if (g < lo || g >= hi) return;
  const long long P = hi - lo, n = g - lo;
  const float* p = points + static_cast<size_t>(g) * 6;
  const float px = p[0], py = p[1], pz = p[2];
  const float* nb = node + static_cast<size_t>(b) * 3 * M;

  float bd[KK];
  int bi[KK];
  som_topk(M, [&](int m) {
    return som_dist_rn(px, py, pz, __ldg(nb + m), __ldg(nb + M + m), __ldg(nb + 2 * M + m));
  }, bd, bi);
  int32_t* ob = min_idx + KK * lo + n;
#pragma unroll
  for (int s = 0; s < KK; ++s) {
    ob[s * P] = bi[s];
    atomicAdd(count + static_cast<size_t>(b) * M + bi[s], 1);
    row_max[static_cast<size_t>(b) * M + bi[s]] = 1;   // every writer stores the same 1
  }
}

__global__ void __launch_bounds__(RGROUP_THREADS)
    som_group_ragged_kernel(const float* __restrict__ points, long long T,
                            const long long* __restrict__ offsets, int M, int k, int with_sn,
                            const int32_t* __restrict__ min_idx, float* __restrict__ cluster_mean,
                            float* __restrict__ x_sorted, long long ld, int32_t* node_sorted,
                            int32_t* __restrict__ pos0) {
  __shared__ int hist[RGROUP_WARPS * RAG_MAX_M];   // [warp][node] counts, then first positions
  __shared__ int offs[RAG_MAX_M + 1];
  __shared__ float cm[3 * RAG_MAX_M];
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  long long lo, hi;
  ragged_range(offsets, b, T, lo, hi);
  const int P = static_cast<int>(hi - lo), kP = k * P;
  const long long base = k * lo;                   // the cloud's first column
  const int32_t* ib = min_idx + base;
  // the sorted copies as n | node << 24, written into node_sorted's own rows first
  uint32_t* perm = reinterpret_cast<uint32_t*>(node_sorted + base);
  const float* pb = points + static_cast<size_t>(lo) * 6;
  // warp w owns the contiguous stacked rows [w*R, (w+1)*R), R a multiple of 32
  const int R = ((kP + RGROUP_WARPS - 1) / RGROUP_WARPS + 31) & ~31;
  const int j_lo = warp * R, j_hi = min(kP, j_lo + R);

  for (int i = threadIdx.x; i < RGROUP_WARPS * M; i += RGROUP_THREADS) hist[i] = 0;
  const int nbits = 32 - __clz(max(M - 1, 1));
  auto same_node = [&](int nd) {
    unsigned peers = __ballot_sync(0xffffffffu, nd >= 0);
    for (int bit = 0; bit < nbits; ++bit) {
      const bool one = (nd >> bit) & 1;
      const unsigned bal = __ballot_sync(0xffffffffu, one);
      peers &= one ? bal : ~bal;
    }
    return peers;
  };
  auto node_of = [&](int j) { return (j < j_hi) ? min(max(__ldg(ib + j), 0), M - 1) : -1; };
  __syncthreads();
  // pass 1: per-warp histogram (one lane per distinct node of a 32-row batch adds the group size)
  for (int j0 = j_lo; j0 < j_hi; j0 += 32) {
    const int nd = node_of(j0 + lane);
    const unsigned peers = same_node(nd);
    if (nd >= 0 && lane == __ffs(peers) - 1) hist[warp * M + nd] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x < M) {
    int tot = 0;
    for (int w = 0; w < RGROUP_WARPS; ++w) tot += hist[w * M + threadIdx.x];
    offs[threadIdx.x + 1] = tot;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    offs[0] = 0;
    for (int m = 0; m < M; ++m) offs[m + 1] += offs[m];
  }
  __syncthreads();
  if (threadIdx.x < M) {
    int run = offs[threadIdx.x];
    for (int w = 0; w < RGROUP_WARPS; ++w) {
      const int c = hist[w * M + threadIdx.x];
      hist[w * M + threadIdx.x] = run;
      run += c;
    }
  }
  __syncthreads();
  // pass 2: stable placement (rank inside the batch = number of lower lanes with the same node)
  for (int j0 = j_lo; j0 < j_hi; j0 += 32) {
    const int j = j0 + lane;
    const int nd = node_of(j);
    const unsigned peers = same_node(nd);
    if (nd >= 0) {
      const int pos = hist[warp * M + nd] + __popc(peers & ((1u << lane) - 1u));
      int n = j;
      while (n >= P) n -= P;
      perm[pos] = static_cast<uint32_t>(n) | (static_cast<uint32_t>(nd) << 24);
      if (j == 0) pos0[b] = static_cast<int32_t>(base + pos);
    }
    __syncwarp();
    if (nd >= 0 && lane == __ffs(peers) - 1) hist[warp * M + nd] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();   // perm (global memory) is visible to the whole block from here on
  // per-node coordinate sums over the node's rows in sorted (= ascending stacked) order:
  // som_group_kernel's order, term for term
  for (int m = warp; m < M; m += RGROUP_WARPS) {
    const int a = offs[m], e = offs[m + 1];
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (int p = a + lane; p < e; p += 128) {
      float ax[4], ay[4], az[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int q = p + 32 * u;
        const bool ok = q < e;
        const int n = ok ? min(static_cast<int>(perm[q] & 0xffffffu), P - 1) : 0;
        ax[u] = ok ? pb[static_cast<size_t>(n) * 6] : 0.f;
        ay[u] = ok ? pb[static_cast<size_t>(n) * 6 + 1] : 0.f;
        az[u] = ok ? pb[static_cast<size_t>(n) * 6 + 2] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        sx += ax[u];
        sy += ay[u];
        sz += az[u];
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sx += __shfl_xor_sync(0xffffffffu, sx, o);
      sy += __shfl_xor_sync(0xffffffffu, sy, o);
      sz += __shfl_xor_sync(0xffffffffu, sz, o);
    }
    if (lane == 0) {
      const float den = __fadd_rn(static_cast<float>(e - a), 1e-5f);
      const float mx = __fdiv_rn(sx, den), my = __fdiv_rn(sy, den), mz = __fdiv_rn(sz, den);
      cm[m] = mx;
      cm[M + m] = my;
      cm[2 * M + m] = mz;
      float* o = cluster_mean + static_cast<size_t>(b) * 3 * M;
      o[m] = mx;
      o[M + m] = my;
      o[2 * M + m] = mz;
    }
  }
  __syncthreads();
  // sorted, decentred rows; each thread rewrites the perm entries it read as flat node ids b*M + m
  const int CA = with_sn ? 6 : 3;
  float* ob = x_sorted + base;
  int32_t* nb = node_sorted + base;
  for (int p = threadIdx.x; p < kP; p += RGROUP_THREADS) {
    const uint32_t e = perm[p];
    const int n = min(static_cast<int>(e & 0xffffffu), P - 1), nd = min(static_cast<int>(e >> 24), M - 1);
    const float* src = pb + static_cast<size_t>(n) * 6;
#pragma unroll
    for (int c = 0; c < 3; ++c) ob[c * ld + p] = __fsub_rn(src[c], cm[c * M + nd]);
    for (int c = 3; c < CA; ++c) ob[c * ld + p] = src[c];
    nb[p] = b * M + nd;
  }
}

__global__ void __launch_bounds__(RAG_THREADS)
    som_decenter_ragged_kernel(const float* __restrict__ points, long long T,
                               const long long* __restrict__ offsets, int B, int M, int k,
                               int with_sn, const int32_t* __restrict__ min_idx,
                               const float* __restrict__ cluster_mean, float* __restrict__ x_aug,
                               long long ld) {
  const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g >= T) return;
  long long lo, hi;
  const int b = ragged_find(offsets, B, T, g, lo, hi);
  if (g < lo || g >= hi) return;
  const long long P = hi - lo;
  const float* p = points + static_cast<size_t>(g) * 6;
  const float* cmb = cluster_mean + static_cast<size_t>(b) * 3 * M;
  const int CA = with_sn ? 6 : 3;
  for (int s = 0; s < k; ++s) {
    const long long j = k * lo + s * P + (g - lo);
    const int id = min(max(__ldg(min_idx + j), 0), M - 1);
#pragma unroll
    for (int c = 0; c < 3; ++c) x_aug[c * ld + j] = __fsub_rn(p[c], __ldg(cmb + c * M + id));
    for (int c = 3; c < CA; ++c) x_aug[c * ld + j] = p[c];
  }
}

}  // namespace sonet

#define RAG_CHECK_COMMON(what)                                                                    \
  SONET_REQUIRE(B >= 1 && T >= 0, what ": bad dimension (B=%d, T=%lld)", B, T);                   \
  SONET_REQUIRE(M >= 1 && M <= sonet::RAG_MAX_M, what ": M=%d out of range [1,%d]", M,            \
                sonet::RAG_MAX_M);                                                                \
  SONET_REQUIRE(k >= 1 && k <= sonet::RAG_MAX_K && k <= M,                                        \
                what ": k=%d out of range [1,%d] (and k <= M=%d)", k, sonet::RAG_MAX_K, M);       \
  SONET_REQUIRE(static_cast<long long>(k) * T < (1LL << 31), what ": k*T=%lld columns too many",  \
                static_cast<long long>(k) * T);                                                   \
  SONET_REQUIRE(static_cast<long long>(B) * M < (1LL << 31), what ": B*M too large")

extern "C" int sonet_som_assign_ragged_f32(const float* points, long long T, const long long* offsets,
                                           int B, const float* node, int M, int k, int32_t* min_idx,
                                           int32_t* count, int32_t* row_max, sonet_stream_t stream) {
  using namespace sonet;
  RAG_CHECK_COMMON("som_assign_ragged");
  SONET_REQUIRE(offsets && node && count && row_max && (T == 0 || (points && min_idx)),
                "som_assign_ragged: null pointer");
  cudaStream_t st = as_stream(stream);
  const size_t bm = static_cast<size_t>(B) * M;
  cudaMemsetAsync(count, 0, bm * sizeof(int32_t), st);
  cudaMemsetAsync(row_max, 0, bm * sizeof(int32_t), st);
  if (T > 0) {
    const unsigned grid = static_cast<unsigned>((T + RAG_THREADS - 1) / RAG_THREADS);
    switch (k) {
      case 1: som_assign_ragged_kernel<1><<<grid, RAG_THREADS, 0, st>>>(points, T, offsets, B, node, M, min_idx, count, row_max); break;
      case 2: som_assign_ragged_kernel<2><<<grid, RAG_THREADS, 0, st>>>(points, T, offsets, B, node, M, min_idx, count, row_max); break;
      case 3: som_assign_ragged_kernel<3><<<grid, RAG_THREADS, 0, st>>>(points, T, offsets, B, node, M, min_idx, count, row_max); break;
      default: som_assign_ragged_kernel<4><<<grid, RAG_THREADS, 0, st>>>(points, T, offsets, B, node, M, min_idx, count, row_max); break;
    }
  }
  return check_launch("som_assign_ragged");
}

extern "C" int sonet_som_group_decenter_ragged_f32(const float* points, long long T,
                                                   const long long* offsets, int B, int M, int k,
                                                   int with_sn, const int32_t* min_idx,
                                                   float* cluster_mean, float* x_sorted,
                                                   int32_t* node_sorted, int32_t* pos0,
                                                   sonet_stream_t stream) {
  using namespace sonet;
  RAG_CHECK_COMMON("som_group_decenter_ragged");
  SONET_REQUIRE(T < (1LL << 24), "som_group_decenter_ragged: T=%lld points too many (a sorted "
                "copy packs its point index into 24 bits)", T);
  SONET_REQUIRE(with_sn == 0 || with_sn == 1, "som_group_decenter_ragged: with_sn must be 0 or 1");
  SONET_REQUIRE(offsets && cluster_mean && pos0 && (T == 0 || (points && min_idx && x_sorted && node_sorted)),
                "som_group_decenter_ragged: null pointer");
  som_group_ragged_kernel<<<B, RGROUP_THREADS, 0, as_stream(stream)>>>(
      points, T, offsets, M, k, with_sn, min_idx, cluster_mean, x_sorted, k * T, node_sorted, pos0);
  return check_launch("som_group_decenter_ragged");
}

extern "C" int sonet_som_decenter_ragged_f32(const float* points, long long T, const long long* offsets,
                                             int B, int M, int k, int with_sn, const int32_t* min_idx,
                                             const float* cluster_mean, float* x_aug,
                                             sonet_stream_t stream) {
  using namespace sonet;
  RAG_CHECK_COMMON("som_decenter_ragged");
  SONET_REQUIRE(with_sn == 0 || with_sn == 1, "som_decenter_ragged: with_sn must be 0 or 1");
  SONET_REQUIRE(offsets && cluster_mean && (T == 0 || (points && min_idx && x_aug)),
                "som_decenter_ragged: null pointer");
  if (T == 0) return SONET_OK;
  const unsigned grid = static_cast<unsigned>((T + RAG_THREADS - 1) / RAG_THREADS);
  som_decenter_ragged_kernel<<<grid, RAG_THREADS, 0, as_stream(stream)>>>(
      points, T, offsets, B, M, k, with_sn, min_idx, cluster_mean, x_aug, k * T);
  return check_launch("som_decenter_ragged");
}
