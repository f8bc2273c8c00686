// som_sort.cu — node-sorted point order for the fused max-pool path, and its finalisation.
//
// The reference pools the first PointResNet's output per SOM node with index_max on the stacked
// copies in their original order (models/networks.py:181-185). When `first_pn_out` itself is not
// needed (classifier, auto-encoder) sonet_b200 never writes it: the wgmma kernel consumes the
// stacked copies GROUPED BY NODE, so that the 16 rows an epilogue warp holds (16 consecutive
// sorted copies) usually belong to one node and the per-node max of a column is one shuffle
// reduction plus one atomic max per column (csrc/pointmlp_tc.cu, POOL variant). This file
// provides
//
//   som_sort_decenter_kernel   per cloud: bucket the k*N stacked copies by node (offsets from the
//                              node counts, slots handed out by shared-memory atomics — the order
//                              inside a node is arbitrary, max does not care) and write, in sorted
//                              order, the decentred coordinates + normals (models/networks.py:168-172)
//                              and the node id of every sorted position; also the sorted position
//                              of stacked copy 0 (the "point 0" that empty nodes gather).
//   som_group_kernel           the classifier path's version of the above in ONE launch, also
//                              producing the cluster statistics (models/networks.py:140-143): a
//                              STABLE counting sort (warp-private histograms + ballot ranking,
//                              no atomics, rows of a node stay in ascending stacked order), then
//                              per-node coordinate sums in that fixed order (bit-reproducible,
//                              independent of batch sharding), cluster_mean = sum / (count + 1e-5),
//                              then coalesced writes of the decentred rows in sorted order.
//   pool_finalize_kernel       ordered-int keys -> values with the reference's semantics
//                              (max must be > -1000, else the feature of point 0,
//                              index_max.cpp:80-81,103 + networks.py:185) and key reset.
#include <algorithm>

#include "common.cuh"

namespace sonet {

constexpr int SORT_THREADS = 1024;
constexpr int SORT_MAX_M = 256;

__global__ void __launch_bounds__(SORT_THREADS)
    som_sort_decenter_kernel(const float* __restrict__ x, const float* __restrict__ sn,
                             const float* __restrict__ cluster_mean,
                             const int32_t* __restrict__ idx32, const int32_t* __restrict__ count,
                             int N, int M, int k, float* __restrict__ x_sorted,
                             int32_t* __restrict__ node_sorted, int32_t* __restrict__ pos0) {
  __shared__ int offs[SORT_MAX_M];
  __shared__ int cursor[SORT_MAX_M];
  __shared__ float cm[3 * SORT_MAX_M];
  const int b = blockIdx.x;
  const int kN = k * N;
  if (threadIdx.x == 0) {
    int run = 0;
    for (int m = 0; m < M; ++m) {
      offs[m] = run;
      run += count[static_cast<size_t>(b) * M + m];
    }
  }
  for (int m = threadIdx.x; m < M; m += SORT_THREADS) cursor[m] = 0;
  for (int i = threadIdx.x; i < 3 * M; i += SORT_THREADS)
    cm[i] = cluster_mean[static_cast<size_t>(b) * 3 * M + i];
  __syncthreads();
  const int CA = sn ? 6 : 3;
  const float* xb = x + static_cast<size_t>(b) * 3 * N;
  const float* sb = sn ? sn + static_cast<size_t>(b) * 3 * N : nullptr;
  float* ob = x_sorted + static_cast<size_t>(b) * CA * kN;
  for (int j = threadIdx.x; j < kN; j += SORT_THREADS) {
    const int node = min(max(idx32[static_cast<size_t>(b) * kN + j], 0), M - 1);
    const int n = j % N;
    const int pos = offs[node] + atomicAdd(&cursor[node], 1);
#pragma unroll
    for (int c = 0; c < 3; ++c)
      ob[static_cast<size_t>(c) * kN + pos] = __fsub_rn(xb[c * N + n], cm[c * M + node]);
    if (sb) {
#pragma unroll
      for (int c = 0; c < 3; ++c) ob[static_cast<size_t>(3 + c) * kN + pos] = sb[c * N + n];
    }
    node_sorted[static_cast<size_t>(b) * kN + pos] = node;
    if (j == 0) pos0[b] = pos;
  }
}

// ---- statistics + stable sort + decentre in one launch ----------------------------------------------
constexpr int GROUP_THREADS = 1024, GROUP_WARPS = GROUP_THREADS / 32;

__global__ void __launch_bounds__(GROUP_THREADS)
    som_group_kernel(const float* __restrict__ x, const float* __restrict__ sn,
                     const int32_t* __restrict__ idx32, int N, int M, int k,
                     int32_t* __restrict__ count, float* __restrict__ cluster_mean,
                     float* __restrict__ x_sorted, int32_t* __restrict__ node_sorted,
                     int32_t* __restrict__ pos0, int stage) {
  extern __shared__ __align__(16) unsigned char gsm[];
  const int kN = k * N;
  uint32_t* perm = reinterpret_cast<uint32_t*>(gsm);                 // [kN] n | node << 24
  int* hist = reinterpret_cast<int*>(perm + kN);                      // [GROUP_WARPS][M]
  int* offs = hist + GROUP_WARPS * M;                                 // [M + 1]
  float* cm = reinterpret_cast<float*>(offs + M + 1);                 // [3][M]
  float* xs_stage = cm + 3 * M;                                       // [3|6][N] when `stage`
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int32_t* ib = idx32 + static_cast<size_t>(b) * kN;
  const float* xg = x + static_cast<size_t>(b) * 3 * N;
  const float* sg = sn ? sn + static_cast<size_t>(b) * 3 * N : nullptr;
  // The sum and output phases gather rows in sorted order: 4-byte gathers from global memory
  // touch 32 different L1 sectors per warp instruction (~1 sector/cycle: measured 58 us per
  // launch). With the cloud's coordinates (+ normals) staged in shared memory by coalesced
  // loads they cost a few bank-conflict cycles instead.
  if (stage) {
    for (int i = threadIdx.x; i < 3 * N; i += GROUP_THREADS) xs_stage[i] = __ldg(xg + i);
    if (sg)
      for (int i = threadIdx.x; i < 3 * N; i += GROUP_THREADS) xs_stage[3 * N + i] = __ldg(sg + i);
  }
  const float* xb = stage ? xs_stage : xg;
  // warp w owns the contiguous stacked rows [w*R, (w+1)*R), R a multiple of 32
  const int R = ((kN + GROUP_WARPS - 1) / GROUP_WARPS + 31) & ~31;
  const int j_lo = warp * R, j_hi = min(kN, j_lo + R);

  for (int i = threadIdx.x; i < GROUP_WARPS * M; i += GROUP_THREADS) hist[i] = 0;
  // lanes of the warp holding the same node id: ceil(log2 M) ballots. (MATCH.ANY does this in one
  // instruction but is far slower: ncu showed 54 % of this kernel's samples stalled behind it.)
  const int nbits = 32 - __clz(max(M - 1, 1));
  auto same_node = [&](int node) {
    unsigned peers = __ballot_sync(0xffffffffu, node >= 0);
    for (int bit = 0; bit < nbits; ++bit) {
      const bool one = (node >> bit) & 1;
      const unsigned bal = __ballot_sync(0xffffffffu, one);
      peers &= one ? bal : ~bal;
    }
    return peers;
  };
  // this warp's node ids, loaded once with all loads in flight (both passes walk them in order)
  constexpr int NBMAX = 16;                       // batches of 32 rows cached per warp
  const bool cached = R <= 32 * NBMAX;
  int nd[NBMAX];
#pragma unroll
  for (int i = 0; i < NBMAX; ++i) {
    const int j = j_lo + 32 * i + lane;
    nd[i] = (cached && j < j_hi) ? min(max(__ldg(ib + j), 0), M - 1) : -1;
  }
  __syncthreads();
  // pass 1: per-warp histogram (one lane per distinct node of a 32-row batch adds the group size)
  if (cached) {
#pragma unroll
    for (int i = 0; i < NBMAX; ++i) {
      if (j_lo + 32 * i < j_hi) {                 // warp-uniform
        const unsigned peers = same_node(nd[i]);
        if (nd[i] >= 0 && lane == __ffs(peers) - 1) hist[warp * M + nd[i]] += __popc(peers);
        __syncwarp();
      }
    }
  } else {
    for (int j0 = j_lo; j0 < j_hi; j0 += 32) {
      const int j = j0 + lane;
      const int node = (j < j_hi) ? min(max(__ldg(ib + j), 0), M - 1) : -1;
      const unsigned peers = same_node(node);
      if (node >= 0 && lane == __ffs(peers) - 1) hist[warp * M + node] += __popc(peers);
      __syncwarp();
    }
  }
  __syncthreads();
  // node totals -> node offsets; hist[w][m] becomes the first position of warp w's rows of node m
  if (threadIdx.x < M) {
    int tot = 0;
    for (int w = 0; w < GROUP_WARPS; ++w) tot += hist[w * M + threadIdx.x];
    offs[threadIdx.x + 1] = tot;
    count[static_cast<size_t>(b) * M + threadIdx.x] = tot;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    offs[0] = 0;
    for (int m = 0; m < M; ++m) offs[m + 1] += offs[m];
  }
  __syncthreads();
  if (threadIdx.x < M) {
    int run = offs[threadIdx.x];
    for (int w = 0; w < GROUP_WARPS; ++w) {
      const int c = hist[w * M + threadIdx.x];
      hist[w * M + threadIdx.x] = run;
      run += c;
    }
  }
  __syncthreads();
  // pass 2: stable placement (rank inside the batch = number of lower lanes with the same node)
  auto place = [&](int j, int node) {
    const unsigned peers = same_node(node);
    if (node >= 0) {
      const int pos = hist[warp * M + node] + __popc(peers & ((1u << lane) - 1u));
      int n = j;
      while (n >= N) n -= N;
      perm[pos] = static_cast<uint32_t>(n) | (static_cast<uint32_t>(node) << 24);
      if (j == 0) pos0[b] = pos;
    }
    __syncwarp();
    if (node >= 0 && lane == __ffs(peers) - 1) hist[warp * M + node] += __popc(peers);
    __syncwarp();
  };
  if (cached) {
#pragma unroll
    for (int i = 0; i < NBMAX; ++i)
      if (j_lo + 32 * i < j_hi) place(j_lo + 32 * i + lane, nd[i]);
  } else {
    for (int j0 = j_lo; j0 < j_hi; j0 += 32) {
      const int j = j0 + lane;
      place(j, (j < j_hi) ? min(max(__ldg(ib + j), 0), M - 1) : -1);
    }
  }
  __syncthreads();
  // per-node coordinate sums over the node's rows in sorted (= ascending stacked) order
  for (int m = warp; m < M; m += GROUP_WARPS) {
    const int lo = offs[m], hi = offs[m + 1];
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (int p = lo + lane; p < hi; p += 128) {   // four independent gathers in flight
      float ax[4], ay[4], az[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int q = p + 32 * u;
        const bool ok = q < hi;
        const int n = ok ? (perm[q] & 0xffffffu) : 0;
        ax[u] = ok ? xb[n] : 0.f;
        ay[u] = ok ? xb[N + n] : 0.f;
        az[u] = ok ? xb[2 * N + n] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {               // fixed order: ascending row
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
      const float den = __fadd_rn(static_cast<float>(hi - lo), 1e-5f);
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
  // sorted, decentred rows: coalesced stores, gathered (L1-resident) loads
  const int CA = sn ? 6 : 3;
  const float* sb = sn ? (stage ? xs_stage + 3 * N : sg) : nullptr;
  float* ob = x_sorted + static_cast<size_t>(b) * CA * kN;
  int32_t* nb = node_sorted + static_cast<size_t>(b) * kN;
  for (int p0i = threadIdx.x; p0i < kN; p0i += 4 * GROUP_THREADS) {
    float v[4][6];
    int nodes[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {                 // all gathers first ...
      const int p = p0i + u * GROUP_THREADS;
      const uint32_t e = (p < kN) ? perm[p] : 0u;
      const int n = e & 0xffffffu;
      nodes[u] = e >> 24;
#pragma unroll
      for (int c = 0; c < 3; ++c) v[u][c] = xb[c * N + n];
      if (sb) {
#pragma unroll
        for (int c = 0; c < 3; ++c) v[u][3 + c] = sb[c * N + n];
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {                 // ... then the coalesced stores
      const int p = p0i + u * GROUP_THREADS;
      if (p < kN) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
          ob[static_cast<size_t>(c) * kN + p] = __fsub_rn(v[u][c], cm[c * M + nodes[u]]);
        if (sb) {
#pragma unroll
          for (int c = 0; c < 3; ++c) ob[static_cast<size_t>(3 + c) * kN + p] = v[u][3 + c];
        }
        nb[p] = nodes[u];
      }
    }
  }
}

// M % 4 == 0: four consecutive nodes of one (cloud, channel) row per thread, 128-bit accesses
__global__ void __launch_bounds__(256)
    pool_finalize_vec_kernel(int4* __restrict__ keys, const float* __restrict__ p0, int M4,
                             int total4, float4* __restrict__ out_val) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total4) return;
  const int4 k = keys[t];
  keys[t] = make_int4(POOL_KEY_INIT, POOL_KEY_INIT, POOL_KEY_INIT, POOL_KEY_INIT);
  const float pv = __ldg(p0 + t / M4);
  out_val[t] = make_float4(pool_key_value(k.x, pv), pool_key_value(k.y, pv), pool_key_value(k.z, pv),
                           pool_key_value(k.w, pv));
}

__global__ void __launch_bounds__(256)
    pool_finalize_kernel(int32_t* __restrict__ keys, const float* __restrict__ p0, int C, int M,
                         long long total, float* __restrict__ out_val) {
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int key = keys[t];
    keys[t] = POOL_KEY_INIT;  // ready for the next forward
    out_val[t] = pool_key_value(key, __ldg(p0 + t / M));
  }
}

__global__ void __launch_bounds__(256)
    pool_keys_init_kernel(int32_t* __restrict__ keys, long long total) {
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x)
    keys[t] = POOL_KEY_INIT;
}

}  // namespace sonet

extern "C" int sonet_som_sort_decenter(const float* x, const float* sn, const float* cluster_mean,
                                       const int32_t* min_idx_i32, const int32_t* count, int B, int N,
                                       int M, int k, float* x_sorted, int32_t* node_sorted,
                                       int32_t* pos0, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && N >= 0 && k >= 1, "som_sort_decenter: bad dimension");
  SONET_REQUIRE(M >= 1 && M <= SORT_MAX_M, "som_sort_decenter: M=%d out of range", M);
  if (B == 0 || N == 0) return SONET_OK;
  SONET_REQUIRE(x && cluster_mean && min_idx_i32 && count && x_sorted && node_sorted && pos0,
                "som_sort_decenter: null pointer");
  som_sort_decenter_kernel<<<B, SORT_THREADS, 0, as_stream(stream)>>>(
      x, sn, cluster_mean, min_idx_i32, count, N, M, k, x_sorted, node_sorted, pos0);
  return check_launch("som_sort_decenter");
}

extern "C" long long sonet_som_group_smem_bytes(int N, int M, int k) {
  return static_cast<long long>(k) * N * 4 + (sonet::GROUP_WARPS * M + M + 1 + 3 * M) * 4LL + 16;
}
// + the staged copy of the cloud (coordinates, and normals when present)
static long long som_group_stage_bytes(int N, bool with_sn) {
  return static_cast<long long>(with_sn ? 6 : 3) * N * 4;
}

// the one place that decides whether and how sonet_som_group_decenter runs
static int som_group_mode(int N, int M, int k, bool with_sn, long long smem_optin) {
  if (M > sonet::SORT_MAX_M || N >= (1 << 24)) return SONET_SOM_GROUP_NONE;
  const long long smem = sonet_som_group_smem_bytes(N, M, k);
  if (smem > smem_optin) return SONET_SOM_GROUP_NONE;
  return smem + som_group_stage_bytes(N, with_sn) <= smem_optin ? SONET_SOM_GROUP_STAGED
                                                                 : SONET_SOM_GROUP_UNSTAGED;
}

extern "C" int sonet_som_group_mode(int N, int M, int k, int with_sn, long long smem_optin) {
  SONET_REQUIRE(N >= 0 && M >= 1 && k >= 1 && smem_optin >= 0,
                "som_group_mode: bad dimension (N=%d, M=%d, k=%d)", N, M, k);
  return som_group_mode(N, M, k, with_sn != 0, smem_optin);
}

extern "C" int sonet_som_group_decenter(const float* x, const float* sn, const int32_t* min_idx_i32,
                                        int B, int N, int M, int k, int32_t* count,
                                        float* cluster_mean, float* x_sorted, int32_t* node_sorted,
                                        int32_t* pos0, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && N >= 0 && k >= 1, "som_group_decenter: bad dimension");
  SONET_REQUIRE(M >= 1 && M <= SORT_MAX_M, "som_group_decenter: M=%d out of range", M);
  SONET_REQUIRE(N < (1 << 24), "som_group_decenter: N=%d too large", N);
  if (B == 0 || N == 0) return SONET_OK;
  SONET_REQUIRE(x && min_idx_i32 && count && cluster_mean && x_sorted && node_sorted && pos0,
                "som_group_decenter: null pointer");
  const long long smem = sonet_som_group_smem_bytes(N, M, k);
  const int mode = som_group_mode(N, M, k, sn != nullptr, max_smem_optin());
  SONET_REQUIRE(mode != SONET_SOM_GROUP_NONE,
                "som_group_decenter: k*N=%d rows need %lld B of shared memory (use "
                "sonet_som_assign statistics + sonet_som_sort_decenter instead)", k * N, smem);
  const int stage = mode == SONET_SOM_GROUP_STAGED;
  const long long total = stage ? smem + som_group_stage_bytes(N, sn != nullptr) : smem;
  cudaFuncSetAttribute(som_group_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       static_cast<int>(total));
  som_group_kernel<<<B, GROUP_THREADS, static_cast<size_t>(total), as_stream(stream)>>>(
      x, sn, min_idx_i32, N, M, k, count, cluster_mean, x_sorted, node_sorted, pos0, stage);
  return check_launch("som_group_decenter");
}

extern "C" int sonet_pool_keys_init(int32_t* keys, long long n, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(n >= 0, "pool_keys_init: negative size");
  if (n == 0) return SONET_OK;
  SONET_REQUIRE(keys, "pool_keys_init: null pointer");
  const int grid = static_cast<int>(std::min<long long>((n + 255) / 256, 8LL * sm_count()));
  pool_keys_init_kernel<<<grid, 256, 0, as_stream(stream)>>>(keys, n);
  return check_launch("pool_keys_init");
}

extern "C" int sonet_pool_finalize(int32_t* keys, const float* p0, int B, int C, int M,
                                   float* out_val, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 0 && M >= 1, "pool_finalize: bad dimension");
  const long long total = static_cast<long long>(B) * C * M;
  if (total == 0) return SONET_OK;
  SONET_REQUIRE(keys && p0 && out_val, "pool_finalize: null pointer");
  if (M % 4 == 0 && total / 4 < (1LL << 31) && aligned16(keys) && aligned16(out_val)) {
    const int total4 = static_cast<int>(total / 4);
    pool_finalize_vec_kernel<<<(total4 + 255) / 256, 256, 0, as_stream(stream)>>>(
        reinterpret_cast<int4*>(keys), p0, M / 4, total4, reinterpret_cast<float4*>(out_val));
  } else {
    const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, 8LL * sm_count()));
    pool_finalize_kernel<<<grid, 256, 0, as_stream(stream)>>>(keys, p0, C, M, total, out_val);
  }
  return check_launch("pool_finalize");
}
