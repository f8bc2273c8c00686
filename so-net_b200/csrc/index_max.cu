// index_max.cu — per-node indexed arg-max pool for sm_90a.
//
// Semantics follow the reference plugin (models/index_max_ext/index_max.cpp:73-112 and
// index_max_cuda.cu:10-26): for data[B,C,N], index[B,N] in [0,K):
//   max_idx[b,c,k] = first n (ascending) with index[b,n]==k that attains the maximum of
//   data[b,c,n] over that node, if the maximum is > -1000.0f; else 0.
// A NaN never passes the strict '>', so it is never an arg-max; -inf never beats the sentinel.
// index values outside [0,K) are not an error: every table access goes through
// min(unsigned(index), K-1) (im_update, im_update4), so a negative or too large id counts as node
// K-1 and never writes outside the warp's table.
//
// Design (HBM-bound: 4 B/element must stream at close to the HBM bandwidth):
//   * persistent grid, one CTA per SM; a work item is (b, group of NW channels); warp w of the CTA
//     streams channel row c = group*NW + w with 128-bit no-allocate loads (fully coalesced, 4
//     loads in flight per lane).
//   * the int32 index row of cloud b is shared by all channels: it is staged once per CTA in
//     shared memory by the TMA unit (cp.async.bulk 1-D copies, 3-stage mbarrier ring driven by a
//     dedicated producer warp) instead of being re-read from L2 by every channel.
//   * running (max, argmax) live in a per-warp shared-memory table [K][32 lanes] (bank == lane,
//     conflict free); lane-private so that no atomics are needed; ascending-n scan with a strict
//     '>' keeps the first maximum; the final cross-lane reduction breaks ties by lowest n.
//   * the masked gather that follows in the model (models/networks.py:185) is fused: the max
//     value (or data[b,c,0] for empty nodes, as idx*mask_row_max gathers point 0) is emitted too.
#include <algorithm>
#include <thread>
#include <vector>

#include "common.cuh"

namespace sonet {

constexpr int IM_CHUNK = 2048;  // points per staged index chunk (8 KB)
constexpr int IM_STAGES = 3;
constexpr int IM_UNROLL = 4;    // float4 loads in flight per lane (8 measured slower: 0.47 vs 0.355 ms)
constexpr int IM_MAX_WARPS = 16;
constexpr int IM_HDR_BYTES = 128;  // mbarriers, keeps the stages 16B aligned
constexpr float IM_SENTINEL = -1000.0f;

template <typename IdxT>
__device__ __forceinline__ void im_update(float* tval, IdxT* tidx, int lane, int K, int k, float v,
                                          int n) {
  k = min(static_cast<unsigned>(k), static_cast<unsigned>(K - 1));  // never a wild smem write
  const int e = k * 32 + lane;
  if (v > tval[e]) {
    tval[e] = v;
    tidx[e] = static_cast<IdxT>(n);
  }
}

// Four consecutive points of one lane (a float4 of data, an int4 of node ids) folded into the table
// with ALL FOUR table reads issued before the first write. im_update() alone forms a chain
// LDS -> compare -> STS per element that the compiler cannot reorder (a later element of the same
// node must see the earlier write), and the r02k ncu capture showed the kernel bound by exactly
// that chain — 45 % of the stall samples on short-scoreboard (shared-memory results) against 8 %
// on long-scoreboard (global loads). Same-node elements inside the quad are resolved in registers
// by forwarding the running value (6 integer compares), so the semantics are unchanged: strict '>'
// in ascending n keeps the first maximum.
template <typename IdxT>
__device__ __forceinline__ void im_update4(float* tval, IdxT* tidx, int lane, int K, int4 kk,
                                           float4 d, int n) {
  const unsigned kmax = static_cast<unsigned>(K - 1);
  const int k0 = min(static_cast<unsigned>(kk.x), kmax), k1 = min(static_cast<unsigned>(kk.y), kmax),
            k2 = min(static_cast<unsigned>(kk.z), kmax), k3 = min(static_cast<unsigned>(kk.w), kmax);
  const int e0 = k0 * 32 + lane, e1 = k1 * 32 + lane, e2 = k2 * 32 + lane, e3 = k3 * 32 + lane;
  const float t0 = tval[e0], t1 = tval[e1], t2 = tval[e2], t3 = tval[e3];
  const bool u0 = d.x > t0;
  const float c0 = u0 ? d.x : t0;
  const float f1 = (k1 == k0) ? c0 : t1;
  const bool u1 = d.y > f1;
  const float c1 = u1 ? d.y : f1;
  const float f2 = (k2 == k1) ? c1 : ((k2 == k0) ? c0 : t2);
  const bool u2 = d.z > f2;
  const float c2 = u2 ? d.z : f2;
  const float f3 = (k3 == k2) ? c2 : ((k3 == k1) ? c1 : ((k3 == k0) ? c0 : t3));
  const bool u3 = d.w > f3;
  if (u0) { tval[e0] = d.x; tidx[e0] = static_cast<IdxT>(n); }
  if (u1) { tval[e1] = d.y; tidx[e1] = static_cast<IdxT>(n + 1); }
  if (u2) { tval[e2] = d.z; tidx[e2] = static_cast<IdxT>(n + 2); }
  if (u3) { tval[e3] = d.w; tidx[e3] = static_cast<IdxT>(n + 3); }
}

// Cross-lane reduction of one finished row; also resets the table for the next row.
template <typename IdxT>
__device__ __forceinline__ void im_reduce_row(float* tval, IdxT* tidx, int lane, int K,
                                              const float* row, int32_t* out_idx, float* out_val) {
  for (int k = lane; k < K; k += 32) {
    float bv = IM_SENTINEL;
    int bi = 0;
#pragma unroll 8
    for (int j = 0; j < 32; ++j) {
      const int e = k * 32 + ((j + lane) & 31);  // skewed: bank == (j+lane)&31, conflict free
      const float v = tval[e];
      const int i = static_cast<int>(tidx[e]);
      if (v > bv || (v == bv && i < bi)) {
        bv = v;
        bi = i;
      }
      tval[e] = IM_SENTINEL;
      tidx[e] = 0;
    }
    out_idx[k] = bi;
    if (out_val != nullptr) out_val[k] = (bv > IM_SENTINEL) ? bv : __ldg(row);
  }
}

// VEC path: N % 4 == 0 and 16B-aligned bases. blockDim = (NW + 1) * 32; warp NW is the producer.
template <typename IdxT>
__global__ void __launch_bounds__((IM_MAX_WARPS + 1) * 32, 1)
    index_max_vec_kernel(const float* __restrict__ data, const int32_t* __restrict__ index, int B,
                         int C, int N, int K, int NW, int32_t* __restrict__ out_idx,
                         float* __restrict__ out_val) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty = full + IM_STAGES;
  int32_t* stage = reinterpret_cast<int32_t*>(smem + IM_HDR_BYTES);
  unsigned char* tables = smem + IM_HDR_BYTES + IM_STAGES * IM_CHUNK * sizeof(int32_t);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups = (C + NW - 1) / NW;
  const int items = B * groups;
  const int nch = (N + IM_CHUNK - 1) / IM_CHUNK;
  const int my_items =
      (static_cast<int>(blockIdx.x) < items) ? (items - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < IM_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], NW);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == NW) {
    // ---- producer: TMA bulk copies of the index chunks, in the order the consumers read them ----
    if (lane == 0) {
      int s = 0;
      uint32_t use = 0;  // how many times stage s has been filled before
      for (int it = 0; it < my_items; ++it) {
        const int item = blockIdx.x + it * gridDim.x;
        const int b = item / groups;
        const int32_t* irow = index + static_cast<size_t>(b) * N;
        for (int ch = 0; ch < nch; ++ch) {
          if (use > 0) mbar_wait(&empty[s], (use - 1) & 1);
          const int n0 = ch * IM_CHUNK;
          const uint32_t bytes = static_cast<uint32_t>(min(IM_CHUNK, N - n0)) * 4u;
          mbar_arrive_expect_tx(&full[s], bytes);
          bulk_g2s(stage + s * IM_CHUNK, irow + n0, bytes, &full[s]);
          if (++s == IM_STAGES) {
            s = 0;
            ++use;
          }
        }
      }
    }
    return;
  }

  // ---- consumers ------------------------------------------------------------------------------------
  const size_t per_warp = static_cast<size_t>(K) * 32 * (sizeof(float) + sizeof(IdxT));
  float* tval = reinterpret_cast<float*>(tables + warp * per_warp);
  IdxT* tidx = reinterpret_cast<IdxT*>(tval + K * 32);
  for (int e = lane; e < K * 32; e += 32) {
    tval[e] = IM_SENTINEL;
    tidx[e] = 0;
  }
  __syncwarp();

  int s = 0;
  uint32_t use = 0;
  for (int it = 0; it < my_items; ++it) {
    const int item = blockIdx.x + it * gridDim.x;
    const int b = item / groups;
    const int c = (item - b * groups) * NW + warp;
    const bool active = c < C;
    const float* row = data + (static_cast<size_t>(b) * C + (active ? c : 0)) * N;

    // Software pipeline over the row: the loads of group g+1 (IM_UNROLL x 128-bit per lane) are
    // issued before group g is folded into the table, independent of the index-chunk boundaries —
    // the first version (loads, then use, per chunk) measured 53 % of HBM with long-scoreboard as
    // the top stall: not enough bytes in flight.
    constexpr int GV = 32 * IM_UNROLL;                 // float4 per group and warp
    constexpr int GPC = IM_CHUNK / 4 / GV;             // groups per index chunk
    const int nvec_row = N >> 2;
    const int ngroups = (nvec_row + GV - 1) / GV;
    const float4* row4 = reinterpret_cast<const float4*>(row);
    float4 nxt[IM_UNROLL];
    if (active) {
#pragma unroll
      for (int u = 0; u < IM_UNROLL; ++u) {
        const int v = u * 32 + lane;
        if (v < nvec_row) nxt[u] = ldg_stream_f4(row4 + v);
      }
    }
    for (int ch = 0; ch < nch; ++ch) {
      mbar_wait(&full[s], use & 1);
      if (active) {
        const int4* sidx4 = reinterpret_cast<const int4*>(stage + s * IM_CHUNK);
        const int g_end = min(ngroups, (ch + 1) * GPC);
        for (int g = ch * GPC; g < g_end; ++g) {
          float4 d[IM_UNROLL];
#pragma unroll
          for (int u = 0; u < IM_UNROLL; ++u) d[u] = nxt[u];
          if (g + 1 < ngroups) {
#pragma unroll
            for (int u = 0; u < IM_UNROLL; ++u) {
              const int v = (g + 1) * GV + u * 32 + lane;
              if (v < nvec_row) nxt[u] = ldg_stream_f4(row4 + v);
            }
          }
#pragma unroll
          for (int u = 0; u < IM_UNROLL; ++u) {
            const int v = g * GV + u * 32 + lane;       // float4 index in the row
            if (v < nvec_row) {
              const int4 kk = sidx4[v - ch * (IM_CHUNK / 4)];
              const int n = v << 2;
              im_update4<IdxT>(tval, tidx, lane, K, kk, d[u], n);
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      if (++s == IM_STAGES) {
        s = 0;
        ++use;
      }
    }
    if (active) {
      const size_t o = (static_cast<size_t>(b) * C + c) * K;
      im_reduce_row<IdxT>(tval, tidx, lane, K, row, out_idx + o,
                          out_val ? out_val + o : nullptr);
    }
    __syncwarp();
  }
}

// Generic path (any N / alignment): same tables, scalar coalesced loads, index through L1.
template <typename IdxT>
__global__ void __launch_bounds__(IM_MAX_WARPS * 32, 1)
    index_max_scalar_kernel(const float* __restrict__ data, const int32_t* __restrict__ index,
                            int B, int C, int N, int K, int32_t* __restrict__ out_idx,
                            float* __restrict__ out_val) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int NW = blockDim.x >> 5;
  const size_t per_warp = static_cast<size_t>(K) * 32 * (sizeof(float) + sizeof(IdxT));
  float* tval = reinterpret_cast<float*>(smem + warp * per_warp);
  IdxT* tidx = reinterpret_cast<IdxT*>(tval + K * 32);
  for (int e = lane; e < K * 32; e += 32) {
    tval[e] = IM_SENTINEL;
    tidx[e] = 0;
  }
  __syncwarp();
  const long long rows = static_cast<long long>(B) * C;
  for (long long r = static_cast<long long>(blockIdx.x) * NW + warp; r < rows;
       r += static_cast<long long>(gridDim.x) * NW) {
    const int b = static_cast<int>(r / C);
    const float* row = data + r * N;
    const int32_t* irow = index + static_cast<size_t>(b) * N;
    for (int n0 = 0; n0 < N; n0 += 32 * IM_UNROLL) {
      float d[IM_UNROLL];
      int kk[IM_UNROLL];
#pragma unroll
      for (int u = 0; u < IM_UNROLL; ++u) {
        const int n = n0 + u * 32 + lane;
        if (n < N) {
          d[u] = ldg_stream_f1(row + n);
          kk[u] = __ldg(irow + n);
        }
      }
#pragma unroll
      for (int u = 0; u < IM_UNROLL; ++u) {
        const int n = n0 + u * 32 + lane;
        if (n < N) im_update<IdxT>(tval, tidx, lane, K, kk[u], d[u], n);
      }
    }
    __syncwarp();
    im_reduce_row<IdxT>(tval, tidx, lane, K, row, out_idx + r * K,
                        out_val ? out_val + r * K : nullptr);
    __syncwarp();
  }
}

template <typename IdxT>
static int launch_index_max(const float* data, const int32_t* index, int B, int C, int N, int K,
                            int32_t* out_idx, float* out_val, cudaStream_t st) {
  const size_t per_warp = static_cast<size_t>(K) * 32 * (sizeof(float) + sizeof(IdxT));
  const int limit = max_smem_optin();
  const bool vec = (N % 4 == 0) && aligned16(data) && aligned16(index);
  const size_t fixed = vec ? (IM_HDR_BYTES + IM_STAGES * IM_CHUNK * sizeof(int32_t)) : 0;
  int NW = static_cast<int>((limit - fixed) / per_warp);
  NW = std::min(NW, IM_MAX_WARPS);
  NW = std::min(NW, std::max(C, 1));
  if (NW < 1) SONET_FAIL(SONET_ERR_UNSUPPORTED, "index_max: K=%d does not fit shared memory", K);
  const size_t smem = fixed + NW * per_warp;
  const int sms = sm_count();
  if (vec) {
    auto kern = index_max_vec_kernel<IdxT>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    const int groups = (C + NW - 1) / NW;
    const long long items = static_cast<long long>(B) * groups;
    const int grid = static_cast<int>(std::min<long long>(items, sms));
    kern<<<grid, (NW + 1) * 32, smem, st>>>(data, index, B, C, N, K, NW, out_idx, out_val);
  } else {
    auto kern = index_max_scalar_kernel<IdxT>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    const long long rows = static_cast<long long>(B) * C;
    const int grid = static_cast<int>(std::min<long long>((rows + NW - 1) / NW, sms));
    kern<<<grid, NW * 32, smem, st>>>(data, index, B, C, N, K, out_idx, out_val);
  }
  return check_launch("index_max");
}

}  // namespace sonet

extern "C" int sonet_index_max_f32(const float* data, const int32_t* index, int B, int C, int N,
                                   int K, int32_t* out_idx, float* out_val,
                                   sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 0 && N >= 0, "index_max: negative dimension");
  SONET_REQUIRE(K >= 1 && K <= 256, "index_max: K=%d out of range [1,256]", K);
  if (B == 0 || C == 0) return SONET_OK;
  // N == 0: data and index have no elements, and an empty tensor's pointer may be null
  SONET_REQUIRE(out_idx && (N == 0 || (data && index)), "index_max: null pointer");
  cudaStream_t st = as_stream(stream);
  if (N == 0) {  // every node empty: idx 0; there is no point 0 to gather -> val 0
    cudaMemsetAsync(out_idx, 0, sizeof(int32_t) * static_cast<size_t>(B) * C * K, st);
    if (out_val) cudaMemsetAsync(out_val, 0, sizeof(float) * static_cast<size_t>(B) * C * K, st);
    return check_launch("index_max(memset)");
  }
  if (N <= 65536) return launch_index_max<uint16_t>(data, index, B, C, N, K, out_idx, out_val, st);
  return launch_index_max<int32_t>(data, index, B, C, N, K, out_idx, out_val, st);
}

// ---- host variants exported by the reference module (index_max.cpp:33-112) -----------------------
static void index_max_cpu_range(const float* data, const int32_t* index, int B, int C, int N, int K,
                                int32_t* out_idx, float* max_val, int c_begin, int c_end) {
  for (int b = 0; b < B; ++b)
    for (int c = c_begin; c < c_end; ++c) {
      const float* row = data + (static_cast<size_t>(b) * C + c) * N;
      const int32_t* irow = index + static_cast<size_t>(b) * N;
      float* mv = max_val + (static_cast<size_t>(b) * C + c) * K;
      int32_t* mi = out_idx + (static_cast<size_t>(b) * C + c) * K;
      for (int n = 0; n < N; ++n) {
        const int k = irow[n];
        if (row[n] > mv[k]) {
          mv[k] = row[n];
          mi[k] = n;
        }
      }
    }
}

extern "C" int sonet_index_max_cpu_f32(const float* data, const int32_t* index, int B, int C, int N,
                                       int K, int32_t* out_idx, int thread_num) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 0 && N >= 0 && K >= 1, "index_max_cpu: bad dimension");
  SONET_REQUIRE(thread_num >= 1, "index_max_cpu: thread_num must be >= 1");
  const size_t total = static_cast<size_t>(B) * C * K;
  if (total == 0) return SONET_OK;
  SONET_REQUIRE(data && index && out_idx, "index_max_cpu: null pointer");
  for (size_t i = 0, e = static_cast<size_t>(B) * N; i < e; ++i)
    SONET_REQUIRE(index[i] >= 0 && index[i] < K, "index_max_cpu: index value out of [0,K)");
  std::vector<float> max_val(total, -1000.0f);
  std::fill(out_idx, out_idx + total, 0);
  if (thread_num == 1 || C < 2) {
    index_max_cpu_range(data, index, B, C, N, K, out_idx, max_val.data(), 0, C);
    return SONET_OK;
  }
  const int T = std::min(thread_num, C);
  const int step = C / T;  // like the reference: even split, the last thread takes the remainder
  std::vector<std::thread> pool;
  for (int t = 0; t < T; ++t) {
    const int c0 = t * step, c1 = (t == T - 1) ? C : (t + 1) * step;
    pool.emplace_back(index_max_cpu_range, data, index, B, C, N, K, out_idx, max_val.data(), c0, c1);
  }
  for (auto& th : pool) th.join();
  return SONET_OK;
}

// ---- ragged clouds (networks.Encoder.forward_ragged's unfused route) ------------------------------
// data [C, ld] holds the stacked copies of a ragged batch side by side: cloud b's k*P_b copies are the
// columns k*offsets[b] .. k*offsets[b+1], in stacked order; index the cloud-local node of every column.
// Per (cloud, channel, node): the first column (cloud-local, ascending) that attains the maximum if it
// is > -1000, else column 0 and the value of the cloud's copy 0 — index_max's semantics at N = k*P_b,
// so the values are the fused ragged pool's (csrc/pointmlp_tc.cu, RAGGED) bit for bit. A CTA owns one
// cloud and IMR_G channels: a pass of shared-memory atomicMax over order-preserving keys finds each
// node's maximum, a second pass of atomicMin the lowest column that holds it (+0 and -0 compare equal,
// as under '>'); NaN and values <= -1000 never enter. Offsets are clamped as common.cuh's ragged_range
// states and node ids to [0, M-1], so nothing reads or writes out of range.
namespace sonet {

constexpr int IMR_G = 16, IMR_THREADS = 512;

__device__ __forceinline__ int imr_key(float v) {
  const int bits = __float_as_int(v == 0.f ? 0.f : v);
  return bits ^ ((bits >> 31) & 0x7fffffff);
}

__global__ void __launch_bounds__(IMR_THREADS)
    index_max_ragged_kernel(const float* __restrict__ data, int C, long long ld,
                            const int32_t* __restrict__ index, const long long* __restrict__ offsets,
                            long long T, int M, int k, int32_t* __restrict__ out_idx,
                            float* __restrict__ out_val) {
  __shared__ int skey[IMR_G * 256];
  __shared__ int sidx[IMR_G * 256];
  const int b = blockIdx.x, c0 = blockIdx.y * IMR_G, nc = min(IMR_G, C - c0);
  long long lo, hi;
  ragged_range(offsets, b, T, lo, hi);
  const long long base = k * lo;
  const int kP = static_cast<int>(k * (hi - lo));
  const float* db = data + static_cast<size_t>(c0) * ld + base;
  const int32_t* ib = index + base;
  const unsigned mmax = static_cast<unsigned>(M - 1);
  for (int e = threadIdx.x; e < IMR_G * M; e += IMR_THREADS) {
    skey[e] = POOL_KEY_INIT;
    sidx[e] = 0x7fffffff;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < kP; j += IMR_THREADS) {
    const int m = min(static_cast<unsigned>(__ldg(ib + j)), mmax);
    for (int g = 0; g < nc; ++g) {
      const float v = __ldg(db + g * ld + j);
      if (v > IM_SENTINEL) atomicMax(&skey[g * M + m], imr_key(v));
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < kP; j += IMR_THREADS) {
    const int m = min(static_cast<unsigned>(__ldg(ib + j)), mmax);
    for (int g = 0; g < nc; ++g) {
      const float v = __ldg(db + g * ld + j);
      if (v > IM_SENTINEL && imr_key(v) == skey[g * M + m]) atomicMin(&sidx[g * M + m], j);
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < nc * M; e += IMR_THREADS) {
    const int g = e / M, m = e - g * M;
    const int i = sidx[g * M + m];
    const bool hit = i != 0x7fffffff;
    const size_t o = (static_cast<size_t>(b) * C + c0 + g) * M + m;
    out_idx[o] = hit ? i : 0;
    if (out_val) out_val[o] = (hit || kP > 0) ? db[g * ld + (hit ? i : 0)] : 0.f;
  }
}

}  // namespace sonet

extern "C" int sonet_index_max_ragged_f32(const float* data, int C, long long ld, const int32_t* index,
                                          const long long* offsets, int B, long long T, int M, int k,
                                          int32_t* out_idx, float* out_val, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 0 && T >= 0 && k >= 1 && k <= 4,
                "index_max_ragged: bad dimension (B=%d, C=%d, T=%lld, k=%d)", B, C, T, k);
  SONET_REQUIRE(M >= 1 && M <= 256, "index_max_ragged: M=%d out of range [1,256]", M);
  SONET_REQUIRE(ld >= k * T && k * T < (1LL << 31),
                "index_max_ragged: row stride %lld below the k*T=%lld columns (or too many)", ld, k * T);
  SONET_REQUIRE((C + IMR_G - 1) / IMR_G <= 65535, "index_max_ragged: C=%d too large", C);
  if (B == 0 || C == 0) return SONET_OK;
  SONET_REQUIRE(offsets && out_idx && (T == 0 || (data && index)), "index_max_ragged: null pointer");
  dim3 grid(B, (C + IMR_G - 1) / IMR_G);
  index_max_ragged_kernel<<<grid, IMR_THREADS, 0, as_stream(stream)>>>(data, C, ld, index, offsets, T, M,
                                                                      k, out_idx, out_val);
  return check_launch("index_max_ragged");
}
