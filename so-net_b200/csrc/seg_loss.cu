// Segmentation loss of the segmenter wrapper: mean over points of -log_softmax(score)[target].
//
// Replaces CrossEntropyLossSeg.forward (reference models/losses.py:30-43: log_softmax over the
// class axis of [B,classes,N] scores followed by NLLLoss, size_average=True, no class weights) as
// it is evaluated by models/segmenter.py:129-131 (test_model) on every forward. PyTorch runs this
// as a 32-block spatial soft-max plus three small kernels (≈50 µs at B=32, N=1024, 50 classes);
// here: one pass over the scores + a one-block deterministic final sum.
//
//   kernel 1: thread per point (coalesced over n for every class plane): max, sum of exp, the
//             target's score; block sum of the per-point losses in fp64 -> partial[block]
//             (targets equal to ignore_index = -100, NLLLoss's default, do not count; any other
//             out-of-range target makes the loss NaN — loud, PyTorch raises a device assert)
//   kernel 2: fixed-order fp64 sum of the partials, loss = sum / count.
//
// Ragged points (sonet_seg_loss_ragged_f32): score [T,C] point-major, target [T], cloud b is rows
// offsets[b] .. offsets[b+1]. The same partial kernel runs, templated on where a point's class
// scores come from (DensePoints: class planes of stride N; RaggedPoints: a row of C floats). A flat
// grid.x covers every (cloud, 256-point tile) pair through the host-built prefix sums tile_start
// [B+1], so a tile never crosses a cloud and the partials lie in (cloud, tile) order: with equal
// sizes they are the dense partials, in the dense order, and kernel 2 gives the dense loss's bits.
// One more fixed-order pass sums each cloud's own tiles into its mean, loss_array[b].
#include <climits>
#include <vector>

#include "common.cuh"

namespace sonet {

constexpr int SL_THREADS = 256;

// Where a tile's points come from. tile(tx) -> this CTA's cloud b and its 256-point tile tx;
// slot(b) -> the CTA's partial; cloud(N, b) -> cloud b. A cloud c has c.N points, c.point(n) = the
// index of point n's target, c.scores(C, n) = the offset of its class-0 score and c.cls(k) = the
// distance from there to its class-k score.
struct DensePoints {                   // score [B,C,N], target [B,N]: cloud blockIdx.y
  struct Cloud {
    int b, N;
    __device__ __forceinline__ size_t point(int n) const { return static_cast<size_t>(b) * N + n; }
    __device__ __forceinline__ size_t scores(int C, int n) const {
      return static_cast<size_t>(b) * C * N + n;
    }
    template <typename I>
    __device__ __forceinline__ size_t cls(I k) const { return static_cast<size_t>(k) * N; }
  };
  __device__ __forceinline__ Cloud cloud(int N, int b) const { return Cloud{b, N}; }
  __device__ __forceinline__ int tile(unsigned& tx) const {
    tx = blockIdx.x;
    return blockIdx.y;
  }
  __device__ __forceinline__ size_t slot(int b) const {
    return static_cast<size_t>(b) * gridDim.x + blockIdx.x;
  }
};

struct RaggedPoints {                  // score [T,C], target [T]
  long long T;
  const long long* offsets;            // [B+1]: cloud b is rows offsets[b] .. offsets[b+1]
  const int* tile_start;               // [B+1]: cloud b's tiles are tile_start[b] .. [b+1]
  int B;
  struct Cloud {
    size_t lo;
    int N;
    __device__ __forceinline__ size_t point(int n) const { return lo + n; }
    __device__ __forceinline__ size_t scores(int C, int n) const { return (lo + n) * C; }
    template <typename I>
    __device__ __forceinline__ size_t cls(I k) const { return static_cast<size_t>(k); }
  };
  __device__ __forceinline__ Cloud cloud(int, int b) const {
    long long lo, hi;                  // clamped: offsets that disagree with tile_start stay in range
    ragged_range(offsets, b, T, lo, hi);
    return Cloud{static_cast<size_t>(lo), static_cast<int>(hi - lo)};
  }
  __device__ __forceinline__ int tile(unsigned& tx) const {
    const int t = blockIdx.x;
    int a = 0, z = B - 1;              // the last cloud whose first tile is <= t (never an empty one)
    while (a < z) {
      const int mid = (a + z + 1) >> 1;
      if (__ldg(tile_start + mid) <= t) a = mid;
      else z = mid - 1;
    }
    tx = t - __ldg(tile_start + a);
    return a;
  }
  __device__ __forceinline__ size_t slot(int) const { return blockIdx.x; }
};

template <class Pts>
__global__ void __launch_bounds__(SL_THREADS)
    seg_loss_partial_kernel(const float* __restrict__ score, const long long* __restrict__ target,
                            int C, int N_, double* __restrict__ psum, int* __restrict__ pcnt,
                            const Pts pts) {
  unsigned tx;
  const int b = pts.tile(tx);
  const typename Pts::Cloud cl = pts.cloud(N_, b);
  const int n = tx * SL_THREADS + threadIdx.x;
  double loss = 0.0;
  int cnt = 0;
  if (n < cl.N) {
    const long long t = target[cl.point(n)];
    if (t != -100) {
      const float* s = score + cl.scores(C, n);
      float mx = -__int_as_float(0x7f800000);
      for (int c = 0; c < C; ++c) mx = fmaxf(mx, __ldg(s + cl.cls(c)));
      float sum = 0.f;
      for (int c = 0; c < C; ++c) sum += expf(__ldg(s + cl.cls(c)) - mx);
      if (t >= 0 && t < C) {
        const float st = __ldg(s + cl.cls(t));
        loss = static_cast<double>(-((st - mx) - logf(sum)));
      } else {
        loss = static_cast<double>(__int_as_float(0x7fc00000));
      }
      cnt = 1;
    }
  }
  __shared__ double sl[SL_THREADS / 32];
  __shared__ int sc[SL_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    loss += __shfl_xor_sync(0xffffffffu, loss, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if (lane == 0) {
    sl[warp] = loss;
    sc[warp] = cnt;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    int k = 0;
    for (int w = 0; w < SL_THREADS / 32; ++w) {
      a += sl[w];
      k += sc[w];
    }
    const size_t blk = pts.slot(b);
    psum[blk] = a;
    pcnt[blk] = k;
  }
}

__global__ void __launch_bounds__(1024)
    seg_loss_final_kernel(const double* __restrict__ psum, const int* __restrict__ pcnt, int nblk,
                          int size_average, float* __restrict__ loss) {
  // fixed assignment of partials to threads and a fixed-shape tree: bit-reproducible
  double a = 0.0;
  long long k = 0;
  for (int i = threadIdx.x; i < nblk; i += 1024) {
    a += psum[i];
    k += pcnt[i];
  }
  __shared__ double sa[32];
  __shared__ long long sk[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    k += __shfl_xor_sync(0xffffffffu, k, o);
  }
  if (lane == 0) {
    sa[warp] = a;
    sk[warp] = k;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    long long c = 0;
    for (int w = 0; w < 32; ++w) {
      t += sa[w];
      c += sk[w];
    }
    // all targets ignored: PyTorch's mean reduction gives nan (0/0) as well
    *loss = static_cast<float>(size_average ? t / static_cast<double>(c) : t);
  }
}

// Per-cloud means of the ragged partials: block b sums cloud b's tiles tile_start[b] .. [b+1] with
// a fixed assignment to threads and a fixed-shape tree. A cloud with no counted point gets 0/0 =
// NaN, as PyTorch's mean over no element.
__global__ void __launch_bounds__(SL_THREADS)
    seg_loss_cloud_kernel(const double* __restrict__ psum, const int* __restrict__ pcnt,
                          const int* __restrict__ tile_start, float* __restrict__ loss_array) {
  const int b = blockIdx.x;
  const int t1 = tile_start[b + 1];
  double a = 0.0;
  long long k = 0;
  for (int i = tile_start[b] + threadIdx.x; i < t1; i += SL_THREADS) {
    a += psum[i];
    k += pcnt[i];
  }
  __shared__ double sa[SL_THREADS / 32];
  __shared__ long long sk[SL_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    k += __shfl_xor_sync(0xffffffffu, k, o);
  }
  if (lane == 0) {
    sa[warp] = a;
    sk[warp] = k;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    long long c = 0;
    for (int w = 0; w < SL_THREADS / 32; ++w) {
      t += sa[w];
      c += sk[w];
    }
    loss_array[b] = static_cast<float>(t / static_cast<double>(c));
  }
}

}  // namespace sonet

extern "C" long long sonet_seg_loss_scratch_bytes(int B, int N) {
  if (B < 0 || N < 0) return -1;
  const long long nblk = static_cast<long long>(B) * ((N + sonet::SL_THREADS - 1) / sonet::SL_THREADS);
  return nblk * (sizeof(double) + sizeof(int)) + 16;
}

extern "C" int sonet_seg_loss_f32(const float* score, const long long* target, int B, int C, int N,
                                  int size_average, void* scratch, float* loss,
                                  sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 1 && C >= 1 && N >= 1, "seg_loss: bad dimension");
  SONET_REQUIRE(B <= 65535, "seg_loss: B=%d exceeds grid limit", B);
  SONET_REQUIRE(score && target && scratch && loss, "seg_loss: null pointer");
  const int nb = (N + SL_THREADS - 1) / SL_THREADS;
  const long long nblk = static_cast<long long>(B) * nb;
  SONET_REQUIRE(nblk < (1LL << 31), "seg_loss: too many blocks");
  double* psum = static_cast<double*>(scratch);
  int* pcnt = reinterpret_cast<int*>(psum + nblk);
  cudaStream_t st = as_stream(stream);
  seg_loss_partial_kernel<<<dim3(nb, B), SL_THREADS, 0, st>>>(score, target, C, N, psum, pcnt,
                                                               DensePoints{});
  const int rc = check_launch("seg_loss_partial");
  if (rc != SONET_OK) return rc;
  seg_loss_final_kernel<<<1, 1024, 0, st>>>(psum, pcnt, static_cast<int>(nblk), size_average, loss);
  return check_launch("seg_loss_final");
}

// at most T / 256 + B tiles: every cloud adds at most one partial tile
extern "C" long long sonet_seg_loss_ragged_scratch_bytes(int B, long long T) {
  if (B < 0 || T < 0) return -1;
  const long long tiles = T / sonet::SL_THREADS + B;
  return tiles * (sizeof(double) + sizeof(int)) + sizeof(int32_t) * (static_cast<long long>(B) + 1) +
         16;
}

extern "C" int sonet_seg_loss_ragged_f32(const float* score, const long long* target,
                                         const long long* offsets, const long long* offsets_host,
                                         int B, int C, long long T, void* scratch, float* loss,
                                         float* loss_array, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 1 && C >= 1, "seg_loss_ragged: B=%d and C=%d must be >= 1", B, C);
  SONET_REQUIRE(T >= 0, "seg_loss_ragged: T=%lld is negative", T);
  SONET_REQUIRE(score && target && offsets && offsets_host && scratch && loss && loss_array,
                "seg_loss_ragged: null pointer");
  SONET_REQUIRE(offsets_host[0] == 0 && offsets_host[B] == T,
                "seg_loss_ragged: offsets must run from 0 to T=%lld", T);
  // cloud b's 256-point tiles are flat tiles tile_start[b] .. tile_start[b+1]
  std::vector<int32_t> ts(static_cast<size_t>(B) + 1);
  long long tiles = 0;
  for (int b = 0; b < B; ++b) {
    const long long P = offsets_host[b + 1] - offsets_host[b];
    SONET_REQUIRE(P >= 0, "seg_loss_ragged: offsets decrease at cloud %d", b);
    SONET_REQUIRE(P <= INT_MAX - SL_THREADS, "seg_loss_ragged: cloud %d has %lld points, 2^31 - %d "
                  "or more", b, P, SL_THREADS);
    ts[b] = static_cast<int32_t>(tiles);
    tiles += (P + SL_THREADS - 1) / SL_THREADS;
    SONET_REQUIRE(tiles < (1LL << 31), "seg_loss_ragged: %lld partials, 2^31 or more", tiles);
  }
  ts[B] = static_cast<int32_t>(tiles);
  double* psum = static_cast<double*>(scratch);
  int* pcnt = reinterpret_cast<int*>(psum + tiles);
  int32_t* tile_start = pcnt + tiles;
  cudaStream_t st = as_stream(stream);
  // from pageable memory: the copy is staged before this call returns, so ts may go
  cudaMemcpyAsync(tile_start, ts.data(), sizeof(int32_t) * ts.size(), cudaMemcpyHostToDevice, st);
  if (tiles > 0) {                     // T = 0: no partial; the final sums are 0/0 = NaN
    seg_loss_partial_kernel<<<static_cast<unsigned>(tiles), SL_THREADS, 0, st>>>(
        score, target, C, 0, psum, pcnt, RaggedPoints{T, offsets, tile_start, B});
    const int rc = check_launch("seg_loss_ragged_partial");
    if (rc != SONET_OK) return rc;
  }
  seg_loss_final_kernel<<<1, 1024, 0, st>>>(psum, pcnt, static_cast<int>(tiles), 1, loss);
  seg_loss_cloud_kernel<<<B, SL_THREADS, 0, st>>>(psum, pcnt, tile_start, loss_array);
  return check_launch("seg_loss_ragged");
}
