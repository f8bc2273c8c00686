// chamfer.cu — Chamfer distance of the auto-encoder for sm_90a.
//
// Replaces ChamferLoss.forward (models/losses.py:237-290): the reference does, per cloud, two
// Faiss IndexFlatL2 builds + two k=1 searches through host numpy (losses.py:247-276), then
// robust_norm = sqrt(sum_c d_c^2 + 1e-8) (losses.py:17-27) and means. Here the whole batch runs
// with no host round trip, and BOTH directions come from ONE evaluation of each (pred, gt) pair:
//
//   chamfer_pair_kernel   a warp owns 256 gt points (8 per lane, in registers) and streams a tile
//       of pred points from shared memory (broadcast LDS). Two columns are kept per register
//       pair, each half computed with explicitly rounded scalar ops (IEEE rn). Every squared distance is computed
//       once — exact direct differences, ((dx*dx+dy*dy)+dz*dz) with separate roundings, the
//       arithmetic of the brute-force oracle — and feeds the running minimum of its gt point
//       (in-register FMNMX) and of its pred point (in-thread FMNMX over the lane's 8 columns, one
//       REDUX.MIN across the warp, lane r%32 keeps row r). Non-negative floats order like their
//       bit patterns, so the cross-warp / cross-CTA combination is an unsigned atomicMin
//       (shared memory first, then one RED per row and CTA) straight into the caller's
//       elem_fwd / elem_bwd arrays.
//   The eval-mode loss needs only the minimum DISTANCES: sqrt(dmin + 1e-8) is the same number
//   whichever of several equidistant neighbours is selected. The arg-min indices (training:
//   the differentiable gather of losses.py:269,276) come from a second pass of the same kernel
//   that looks for the LOWEST index attaining the final minimum — the oracle's strict-'<'
//   ascending-scan tie rule — so indices stay bit-identical to the brute-force search.
//   chamfer_cloud/final   sqrt(d + 1e-8) in place, fixed-order tree sums -> per-cloud means and the
//       three scalar losses (deterministic, independent of batch sharding).
// Bound: FP32 ALU / issue (arithmetic intensity >> 100 flop/B): 8 FP + 2 FMNMX + ~0.4 per pair.
//
// Ragged ground truth (sonet_chamfer_ragged_f32): cloud b's gt points are rows offsets[b] ..
// offsets[b+1] of points [T, ld]. The same kernels run, templated on where a CTA's columns come from
// (DenseCols / RaggedCols): a flat grid.x covers every (cloud, 1024-column tile) pair through the
// host-built prefix sums tile_start [B+1], so a CTA's columns never cross a cloud boundary and a
// cloud's last tile runs only its live warps, as the dense last column CTA does. Per cloud the
// results are those of the dense entry at N = P_b: the sums run in the same fixed order, and the
// gt-side arrays hold cloud b at rows offsets[b] .. offsets[b+1], its indices cloud-local.
//
// Points with no finite nearest neighbour follow the oracle's scan, which starts from (+inf,
// index 0) and only moves on a strictly smaller distance: a point whose minimum squared distance
// over its non-NaN candidates is +inf (every candidate overflows), or that has no non-NaN
// candidate (a NaN coordinate in the point, or in every point of the other cloud), gets index 0
// and the element sqrt(d(point, other cloud's point 0) + 1e-8) in the usual arithmetic — NaN if
// either point has a NaN, +inf on overflow. fminf drops NaN, so these are exactly the points
// whose key is +inf after the value pass; chamfer_cloud_kernel rewrites them. The tile padding
// is NaN: a padded row or column is never anyone's minimum and never matches in the arg-min pass.
#include <algorithm>
#include <climits>
#include <vector>

#include "common.cuh"

namespace sonet {

constexpr int CH_WARPS = 4;            // warps per CTA, each with its own 256-column chunk
constexpr int CH_RN = 8;               // gt points per lane
constexpr int CH_COLS = 32 * CH_RN;    // 256 columns per warp
constexpr int CH_TM = 128;             // pred points per CTA tile (256: 5.4 CTAs per SM, 80 us; see r02 summary)
constexpr unsigned CH_PAD = 0x7fffffffu;  // padding coordinate (NaN bits): ignored by fminf, == nothing
constexpr unsigned CH_INF = 0x7f800000u;  // +inf bits: the key of a point with no finite neighbour

// Where the gt columns come from. The kernels take (gt, N) as the dense entry passes them, and a
// trailing Cols argument that says how to read them: tile(tx) -> this CTA's cloud b and its column
// tile tx; cloud(gt, N, b) -> cloud b. A cloud c has c.b, its column count c.N, c.col(n) =
// the offset of its column n in the gt-side arrays, c.row(pred, P) = the offset of its P entries in a
// pred-side (pred) or gt-side array, and c.coord(n, k) = coordinate k of column n.
struct DenseCols {                     // gt [B,3,N]: cloud blockIdx.z, column tile blockIdx.x
  struct Cloud {
    const float* gb;
    int b, N;
    __device__ __forceinline__ size_t col(int n) const { return static_cast<size_t>(b) * N + n; }
    __device__ __forceinline__ size_t row(bool, int P) const { return static_cast<size_t>(b) * P; }
    __device__ __forceinline__ float coord(int n, int k) const { return gb[k * N + n]; }
  };
  __device__ __forceinline__ Cloud cloud(const float* gt, int N, int b) const {
    return Cloud{gt + static_cast<size_t>(b) * 3 * N, b, N};
  }
  __device__ __forceinline__ int tile(unsigned& tx) const {
    tx = blockIdx.x;
    return blockIdx.z;
  }
};

struct RaggedCols {                    // gt = points [T, ld] (xyz first), N = ld
  long long T;
  const long long* offsets;            // [B+1]: cloud b is rows offsets[b] .. offsets[b+1]
  const int* tile_start;               // [B+1]: cloud b's column tiles are tile_start[b] .. [b+1]
  int B;
  struct Cloud {
    const float* points;
    size_t ld, lo;
    int b, N;
    __device__ __forceinline__ size_t col(int n) const { return lo + n; }
    __device__ __forceinline__ size_t row(bool pred, int P) const {
      return pred ? static_cast<size_t>(b) * P : lo;
    }
    __device__ __forceinline__ float coord(int n, int k) const { return points[(lo + n) * ld + k]; }
  };
  __device__ __forceinline__ Cloud cloud(const float* points, int ld, int b) const {
    long long lo, hi;                  // clamped: offsets that disagree with tile_start stay in range
    ragged_range(offsets, b, T, lo, hi);
    return Cloud{points, static_cast<size_t>(ld), static_cast<size_t>(lo), b,
                 static_cast<int>(hi - lo)};
  }
  __device__ __forceinline__ int tile(unsigned& tx) const {
    const int t = blockIdx.x;
    int a = 0, z = B - 1;              // the last cloud whose first tile is <= t
    while (a < z) {
      const int mid = (a + z + 1) >> 1;
      if (__ldg(tile_start + mid) <= t) a = mid;
      else z = mid - 1;
    }
    tx = t - __ldg(tile_start + a);
    return a;
  }
};

// row_key [B,Mp] / col_key (gt-side, column n of cloud c at c.col(n)): running minima as float bits
// (init 0xFFFFFFFF). IDX pass: row_key/col_key hold the FINAL minima; row_idx/col_idx (init
// INT_MAX-like) receive the lowest index attaining them.
template <bool IDX, class Cols>
__global__ void __launch_bounds__(CH_WARPS * 32)
    chamfer_pair_kernel(const float* __restrict__ pred, int Mp, const float* __restrict__ gt, int N_,
                        unsigned* __restrict__ row_key, unsigned* __restrict__ col_key,
                        int* __restrict__ row_idx, int* __restrict__ col_idx, const Cols cols) {
  __shared__ float2 srow[CH_TM][4];    // (x,x) (y,y) (z,z) pad: LDS.128 + LDS.64 -> packed operands
  __shared__ unsigned srmin[CH_TM];    // value pass: row minima of this CTA; idx pass: row arg-min
  __shared__ float srfin[IDX ? CH_TM : 1];
  __shared__ int done;                 // warps of this CTA that finished their columns
  unsigned tx;
  const int b = cols.tile(tx);
  const int m0 = blockIdx.y * CH_TM;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n0 = (tx * CH_WARPS + warp) * CH_COLS;
  const float* pb = pred + static_cast<size_t>(b) * 3 * Mp;
  const typename Cols::Cloud c = cols.cloud(gt, N_, b);
  const int N = c.N;
  const int rows = min(CH_TM, Mp - m0);
  for (int i = threadIdx.x; i < CH_TM; i += CH_WARPS * 32) {
    const int m = m0 + i;
    const float pad = __uint_as_float(CH_PAD);
    const float rx = (m < Mp) ? pb[m] : pad, ry = (m < Mp) ? pb[Mp + m] : pad,
                rz = (m < Mp) ? pb[2 * Mp + m] : pad;
    srow[i][0] = make_float2(rx, rx);
    srow[i][1] = make_float2(ry, ry);
    srow[i][2] = make_float2(rz, rz);
    srmin[i] = IDX ? 0x7fffffffu : 0xffffffffu;
    if (IDX) srfin[i] = (m < Mp) ? __uint_as_float(row_key[static_cast<size_t>(b) * Mp + m]) : -1.f;
  }
  if (threadIdx.x == 0) done = 0;
  __syncthreads();
  if (n0 >= N) return;                 // (after the only CTA-wide barrier but the last)

  // NEGATED gt coordinates, two columns per register pair: p - g == p + (-g) bit for bit, and each
  // half is rounded like the reference's scalar op (common.cuh: add2_rn / mul2_rn)
  float2 ngx[CH_RN / 2], ngy[CH_RN / 2], ngz[CH_RN / 2];
  float cmin[CH_RN];
  int cidx[CH_RN];
#pragma unroll
  for (int j = 0; j < CH_RN; ++j) {
    const int n = n0 + j * 32 + lane;
    const bool ok = n < N;
    const float pad = __uint_as_float(CH_PAD);
    const float vx = ok ? -c.coord(n, 0) : pad,
                vy = ok ? -c.coord(n, 1) : pad,
                vz = ok ? -c.coord(n, 2) : pad;
    if (j & 1) {
      ngx[j >> 1].y = vx; ngy[j >> 1].y = vy; ngz[j >> 1].y = vz;
    } else {
      ngx[j >> 1].x = vx; ngy[j >> 1].x = vy; ngz[j >> 1].x = vz;
    }
    if (IDX) {
      cmin[j] = ok ? __uint_as_float(col_key[c.col(n)]) : -1.f;  // final
      cidx[j] = 0x7fffffff;
    } else {
      cmin[j] = __int_as_float(0x7f800000);
    }
  }

  const int row_blocks = (rows + 31) >> 5;
  for (int rb = 0; rb < row_blocks; ++rb) {
    unsigned keep = IDX ? 0x7fffffffu : 0xffffffffu;   // row (rb*32 + lane): min / arg-min so far
#pragma unroll 4
    for (int ri = 0; ri < 32; ++ri) {
      const int r = rb * 32 + ri;
      const float2 px = srow[r][0], py = srow[r][1], pz = srow[r][2];
      if (!IDX) {
        float rmin = __int_as_float(0x7f800000);
#pragma unroll
        for (int j = 0; j < CH_RN / 2; ++j) {
          const float2 dx = add2_rn(px, ngx[j]), dy = add2_rn(py, ngy[j]),
                       dz = add2_rn(pz, ngz[j]);
          const float2 d = sqsum3_rn(dx, dy, dz);
          cmin[2 * j] = fminf(cmin[2 * j], d.x);
          cmin[2 * j + 1] = fminf(cmin[2 * j + 1], d.y);
          rmin = fminf(rmin, fminf(d.x, d.y));
        }
        const unsigned red = __reduce_min_sync(0xffffffffu, __float_as_uint(rmin));
        if (lane == ri) keep = red;
      } else {
        const float rf = srfin[r];
        int cand = 0x7fffffff;
#pragma unroll
        for (int j = 0; j < CH_RN / 2; ++j) {
          const float2 dx = add2_rn(px, ngx[j]), dy = add2_rn(py, ngy[j]),
                       dz = add2_rn(pz, ngz[j]);
          const float2 d = sqsum3_rn(dx, dy, dz);
          if (d.x == cmin[2 * j]) cidx[2 * j] = min(cidx[2 * j], m0 + r);        // lowest pred index
          if (d.y == cmin[2 * j + 1]) cidx[2 * j + 1] = min(cidx[2 * j + 1], m0 + r);
          if (d.x == rf) cand = min(cand, n0 + (2 * j) * 32 + lane);             // lowest gt index
          if (d.y == rf) cand = min(cand, n0 + (2 * j + 1) * 32 + lane);
        }
        const unsigned red = __reduce_min_sync(0xffffffffu, static_cast<unsigned>(cand));
        if (lane == ri) keep = red;
      }
    }
    atomicMin(&srmin[rb * 32 + lane], keep);
  }

  // columns: complete over this CTA's pred tile -> one RED per column (a plain store would do
  // when Mp <= CH_TM, but the RED keeps one code path)
#pragma unroll
  for (int j = 0; j < CH_RN; ++j) {
    const int n = n0 + j * 32 + lane;
    if (n < N) {
      if (IDX) {
        if (cidx[j] != 0x7fffffff) atomicMin(col_idx + c.col(n), cidx[j]);
      } else {
        atomicMin(col_key + c.col(n), __float_as_uint(cmin[j]));
      }
    }
  }
  // rows: combined across this CTA's warps in shared memory; the LAST warp to get here flushes.
  // (warps that returned early never touch srmin; count only the live ones)
  __syncwarp();
  __threadfence_block();
  const int live_warps = min(CH_WARPS, (N - tx * CH_WARPS * CH_COLS + CH_COLS - 1) / CH_COLS);
  int ticket = 0;
  if (lane == 0) ticket = atomicAdd(&done, 1);
  ticket = __shfl_sync(0xffffffffu, ticket, 0);
  if (ticket == live_warps - 1) {
    __threadfence_block();
    for (int i = lane; i < rows; i += 32) {
      const unsigned v = srmin[i];
      if (IDX) {
        if (v != 0x7fffffffu) atomicMin(row_idx + static_cast<size_t>(b) * Mp + m0 + i, static_cast<int>(v));
      } else {
        atomicMin(row_key + static_cast<size_t>(b) * Mp + m0 + i, v);
      }
    }
  }
}

__device__ __forceinline__ float block_sum_256(float v, float* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  const float r = red[0];
  __syncthreads();
  return r;
}

// grid = (B, 2): keys (min squared distances) of one direction of one cloud -> sqrt(d + 1e-8) in
// place and their mean. 1024 threads, fixed order: thread-strided partial sums, xor-shuffle tree
// inside each warp, then a fixed 32-term tree over the warps. A key of +inf (no finite nearest
// neighbour, see the header) becomes the distance to the other cloud's point 0, and its index 0
// when indices are asked for: (p - g)^2 == (g - p)^2, so both directions compute pred - gt.
constexpr int CC_THREADS = 1024;
template <class Cols>
__global__ void __launch_bounds__(CC_THREADS)
    chamfer_cloud_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                         float* __restrict__ elem_fwd, int Mp, float* __restrict__ elem_bwd, int N_,
                         int* __restrict__ idx_fwd, int* __restrict__ idx_bwd,
                         float* __restrict__ fwd_arr, float* __restrict__ bwd_arr, const Cols cols) {
  __shared__ float wsum[CC_THREADS / 32];
  const int b = blockIdx.x;
  const bool fwd = blockIdx.y == 0;
  const float* pb = pred + static_cast<size_t>(b) * 3 * Mp;
  const typename Cols::Cloud c = cols.cloud(gt, N_, b);
  const int P = fwd ? Mp : c.N;
  float* e = (fwd ? elem_fwd : elem_bwd) + c.row(fwd, P);
  int* idx = fwd ? idx_fwd : idx_bwd;
  float s = 0.f;
  for (int i = threadIdx.x; i < P; i += CC_THREADS) {
    float d = e[i];
    if (__float_as_uint(d) == CH_INF) {
      const int m = fwd ? i : 0, n = fwd ? 0 : i;
      const float dx = __fsub_rn(pb[m], c.coord(n, 0)),
                  dy = __fsub_rn(pb[Mp + m], c.coord(n, 1)),
                  dz = __fsub_rn(pb[2 * Mp + m], c.coord(n, 2));
      d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      if (idx) idx[c.row(fwd, P) + i] = 0;
    }
    const float v = __fsqrt_rn(__fadd_rn(d, 1e-8f));
    e[i] = v;
    s += v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = wsum[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) (fwd ? fwd_arr : bwd_arr)[b] = __fdiv_rn(t, static_cast<float>(P));
  }
}

__global__ void __launch_bounds__(256)
    chamfer_final_kernel(const float* __restrict__ fwd_arr, const float* __restrict__ bwd_arr, int B,
                         float* __restrict__ loss) {
  __shared__ float red[256];
  float s = 0.f;
  for (int i = threadIdx.x; i < B; i += 256) s += fwd_arr[i];
  const float f = block_sum_256(s, red);
  s = 0.f;
  for (int i = threadIdx.x; i < B; i += 256) s += bwd_arr[i];
  const float g = block_sum_256(s, red);
  if (threadIdx.x == 0) {
    const float fl = __fdiv_rn(f, static_cast<float>(B)), bl = __fdiv_rn(g, static_cast<float>(B));
    loss[0] = fl;
    loss[1] = bl;
    loss[2] = __fadd_rn(fl, bl);
  }
}

}  // namespace sonet

extern "C" int sonet_chamfer_f32(const float* pred, const float* gt, int B, int Mp, int N,
                                 int32_t* idx_fwd, int32_t* idx_bwd, float* elem_fwd,
                                 float* elem_bwd, float* loss_fwd_arr, float* loss_bwd_arr,
                                 float* loss, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 1 && Mp >= 1 && N >= 1, "chamfer: dimensions must be >= 1");
  SONET_REQUIRE(B <= 65535, "chamfer: B=%d exceeds grid limit", B);
  SONET_REQUIRE(pred && gt && elem_fwd && elem_bwd && loss_fwd_arr && loss_bwd_arr && loss,
                "chamfer: null pointer");
  SONET_REQUIRE((idx_fwd == nullptr) == (idx_bwd == nullptr),
                "chamfer: idx_fwd and idx_bwd go together");
  cudaStream_t st = as_stream(stream);
  // the element arrays double as the running minima (uint keys of non-negative floats)
  cudaMemsetAsync(elem_fwd, 0xff, sizeof(float) * static_cast<size_t>(B) * Mp, st);
  cudaMemsetAsync(elem_bwd, 0xff, sizeof(float) * static_cast<size_t>(B) * N, st);
  const dim3 grid((N + CH_WARPS * CH_COLS - 1) / (CH_WARPS * CH_COLS), (Mp + CH_TM - 1) / CH_TM, B);
  SONET_REQUIRE(grid.y <= 65535, "chamfer: Mp=%d exceeds grid limit", Mp);
  chamfer_pair_kernel<false><<<grid, CH_WARPS * 32, 0, st>>>(
      pred, Mp, gt, N, reinterpret_cast<unsigned*>(elem_fwd), reinterpret_cast<unsigned*>(elem_bwd),
      nullptr, nullptr, DenseCols{});
  int rc = check_launch("chamfer(pairs)");
  if (rc) return rc;
  if (idx_fwd) {
    cudaMemsetAsync(idx_fwd, 0x7f, sizeof(int32_t) * static_cast<size_t>(B) * Mp, st);
    cudaMemsetAsync(idx_bwd, 0x7f, sizeof(int32_t) * static_cast<size_t>(B) * N, st);
    chamfer_pair_kernel<true><<<grid, CH_WARPS * 32, 0, st>>>(
        pred, Mp, gt, N, reinterpret_cast<unsigned*>(elem_fwd), reinterpret_cast<unsigned*>(elem_bwd),
        idx_fwd, idx_bwd, DenseCols{});
    rc = check_launch("chamfer(arg-min)");
    if (rc) return rc;
  }
  chamfer_cloud_kernel<<<dim3(B, 2), CC_THREADS, 0, st>>>(pred, gt, elem_fwd, Mp, elem_bwd, N, idx_fwd,
                                                          idx_bwd, loss_fwd_arr, loss_bwd_arr,
                                                          DenseCols{});
  chamfer_final_kernel<<<1, 256, 0, st>>>(loss_fwd_arr, loss_bwd_arr, B, loss);
  return check_launch("chamfer");
}

extern "C" int sonet_chamfer_ragged_f32(const float* pred, int B, int Mp, const float* points,
                                        long long T, long long ld, const long long* offsets,
                                        const long long* offsets_host, int32_t* tile_start,
                                        int32_t* idx_fwd, int32_t* idx_bwd, float* elem_fwd,
                                        float* elem_bwd, float* loss_fwd_arr, float* loss_bwd_arr,
                                        float* loss, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 1 && Mp >= 1, "chamfer_ragged: B=%d and Mp=%d must be >= 1", B, Mp);
  SONET_REQUIRE(ld >= 3 && ld <= INT_MAX, "chamfer_ragged: row stride %lld outside [3, 2^31)", ld);
  SONET_REQUIRE(pred && points && offsets && offsets_host && tile_start && elem_fwd && elem_bwd &&
                    loss_fwd_arr && loss_bwd_arr && loss,
                "chamfer_ragged: null pointer");
  SONET_REQUIRE((idx_fwd == nullptr) == (idx_bwd == nullptr),
                "chamfer_ragged: idx_fwd and idx_bwd go together");
  SONET_REQUIRE(offsets_host[0] == 0 && offsets_host[B] == T,
                "chamfer_ragged: offsets must run from 0 to T=%lld", T);
  // cloud b's 1024-column tiles are flat tiles tile_start[b] .. tile_start[b+1]
  std::vector<int32_t> ts(static_cast<size_t>(B) + 1);
  long long tiles = 0;
  for (int b = 0; b < B; ++b) {
    const long long P = offsets_host[b + 1] - offsets_host[b];
    SONET_REQUIRE(P >= 1, "chamfer_ragged: cloud %d has no points (offsets must increase)", b);
    SONET_REQUIRE(P < (1LL << 24), "chamfer_ragged: cloud %d has %lld points, 2^24 or more", b, P);
    ts[b] = static_cast<int32_t>(tiles);
    tiles += (P + CH_WARPS * CH_COLS - 1) / (CH_WARPS * CH_COLS);
    SONET_REQUIRE(tiles <= INT_MAX, "chamfer_ragged: %lld column tiles exceed the grid", tiles);
  }
  ts[B] = static_cast<int32_t>(tiles);
  const dim3 grid(static_cast<unsigned>(tiles), (Mp + CH_TM - 1) / CH_TM, 1);
  SONET_REQUIRE(grid.y <= 65535, "chamfer_ragged: Mp=%d exceeds grid limit", Mp);
  cudaStream_t st = as_stream(stream);
  // from pageable memory: the copy is staged before this call returns, so ts may go
  cudaMemcpyAsync(tile_start, ts.data(), sizeof(int32_t) * ts.size(), cudaMemcpyHostToDevice, st);
  const RaggedCols cols{T, offsets, tile_start, B};
  const int ldi = static_cast<int>(ld);
  cudaMemsetAsync(elem_fwd, 0xff, sizeof(float) * static_cast<size_t>(B) * Mp, st);
  cudaMemsetAsync(elem_bwd, 0xff, sizeof(float) * static_cast<size_t>(T), st);
  chamfer_pair_kernel<false><<<grid, CH_WARPS * 32, 0, st>>>(
      pred, Mp, points, ldi, reinterpret_cast<unsigned*>(elem_fwd),
      reinterpret_cast<unsigned*>(elem_bwd), nullptr, nullptr, cols);
  int rc = check_launch("chamfer_ragged(pairs)");
  if (rc) return rc;
  if (idx_fwd) {
    cudaMemsetAsync(idx_fwd, 0x7f, sizeof(int32_t) * static_cast<size_t>(B) * Mp, st);
    cudaMemsetAsync(idx_bwd, 0x7f, sizeof(int32_t) * static_cast<size_t>(T), st);
    chamfer_pair_kernel<true><<<grid, CH_WARPS * 32, 0, st>>>(
        pred, Mp, points, ldi, reinterpret_cast<unsigned*>(elem_fwd),
        reinterpret_cast<unsigned*>(elem_bwd), idx_fwd, idx_bwd, cols);
    rc = check_launch("chamfer_ragged(arg-min)");
    if (rc) return rc;
  }
  chamfer_cloud_kernel<<<dim3(B, 2), CC_THREADS, 0, st>>>(pred, points, elem_fwd, Mp, elem_bwd, ldi,
                                                          idx_fwd, idx_bwd, loss_fwd_arr,
                                                          loss_bwd_arr, cols);
  chamfer_final_kernel<<<1, 256, 0, st>>>(loss_fwd_arr, loss_bwd_arr, B, loss);
  return check_launch("chamfer_ragged");
}
