// sample_points.cu — the loader's random choice of a cloud's points, for a whole batch, from a
// dataset resident in device memory (sm_90a).
//
// Replaces the head of the loaders' __getitem__: np.random.choice(P, N, replace=False) in
// data/modelnet_shrec_loader.py:198,212 (rule SUBSET), and data/shapenet_loader.py:142-154, which
// keeps the whole cloud in order and appends choice(P, N-P, replace=True) when N >= P (rule FILL).
// One CTA per cloud of the batch; its output columns are coalesced stores along N, each a 24-byte
// source row (xyz | normal) and optionally the point's part label.
//
// The source indices come from the caller (the loader's own numpy draws: reproduces it bit for
// bit) or are drawn in the kernel from the library's Philox4x32-10 (philox.cuh), keyed by
// (seed, batch position, point):
//   - SUBSET: every point i gets the key (48 random bits << 16) | i, unique because P <= 65536.
//     The N smallest keys, in ascending order, are a uniformly random ordered N-subset: the
//     distribution of permutation(P)[:N] (up to 48-bit key ties, broken by index). A radix select
//     over 12-bit digits finds the N-th smallest key by histogram passes that recompute the keys, so
//     nothing P-sized is stored. The N selected keys are then scattered by their top digit into the
//     cloud's own pc_out columns (2N of its 3N words), each digit bucket is sorted in place, and the
//     gather reads column j's key before it overwrites column j.
//   - FILL with N >= P: positions [0,P) are the cloud in order, [P,N) uniform draws from [0,P) by
//     Lemire's multiply-shift with rejection (unbiased).
#include "common.cuh"
#include "philox.cuh"

namespace sonet {

constexpr int SP_THREADS = 1024;
constexpr int SP_DIGIT = 12;                 // radix digit of the select passes
constexpr int SP_BINS = 1 << SP_DIGIT;
constexpr uint32_t SP_TAG_KEY = 3u;          // Philox stream tags (augment.cu uses 0..2)
constexpr uint32_t SP_TAG_FILL = 4u;

struct SampleArgs {
  const float* data;         // [sum P, 6]
  const int64_t* offsets;    // [S+1]
  const int32_t* labels;     // [sum P] (nullable)
  const int64_t* cloud_ids;  // [B]
  const int32_t* indices;    // [B, N] (nullable: in-kernel draws)
  float* pc_out;             // [B, 3, N]
  float* sn_out;             // [B, 3, N]
  int64_t* seg_out;          // [B, N] (nullable)
  int S, N, max_P, rule;
  uint32_t k0, k1;           // seed
};

__device__ __forceinline__ uint64_t select_key(uint32_t k0, uint32_t k1, uint32_t b, uint32_t i) {
  uint32_t c[4] = {i, b, SP_TAG_KEY, 0u};
  philox4x32_10(c, k0, k1);
  return (static_cast<uint64_t>(c[0]) << 32) | (c[1] & 0xFFFF0000u) | i;
}

// uniform in [0,P), P >= 1: Lemire's multiply-shift, rejecting low words below 2^32 mod P
__device__ __forceinline__ uint32_t fill_draw(uint32_t k0, uint32_t k1, uint32_t b, uint32_t j,
                                              uint32_t P) {
  const uint32_t thresh = (0u - P) % P;
  for (uint32_t attempt = 0;; ++attempt) {
    uint32_t c[4] = {j, b, SP_TAG_FILL, attempt};
    philox4x32_10(c, k0, k1);
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const uint64_t m = static_cast<uint64_t>(c[w]) * P;
      if (static_cast<uint32_t>(m) >= thresh) return static_cast<uint32_t>(m >> 32);
    }
  }
}

// Block-wide scan of h[SP_BINS]: finds the bin t with excl[t] < r <= excl[t] + h[t] (r in
// [1, sum h]) and stores (t, excl[t], h[t]) in res; with write_excl, h becomes the exclusive scan.
__device__ __forceinline__ void scan_find(uint32_t* h, uint32_t r, bool write_excl,
                                          uint32_t* warp_sums, uint32_t* res) {
  constexpr int PER = SP_BINS / SP_THREADS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t v[PER], sum = 0;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    v[k] = h[PER * tid + k];
    sum += v[k];
  }
  uint32_t inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const uint32_t w = warp_sums[lane];
    uint32_t wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t n = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += n;
    }
    warp_sums[lane] = wi - w;
  }
  __syncthreads();
  uint32_t run = warp_sums[warp] + inc - sum;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    if (run < r && r <= run + v[k]) {
      res[0] = PER * tid + k;
      res[1] = run;
      res[2] = v[k];
    }
    if (write_excl) h[PER * tid + k] = run;
    run += v[k];
  }
  __syncthreads();
}

__global__ void __launch_bounds__(SP_THREADS) sample_points_kernel(SampleArgs a) {
  __shared__ uint32_t s_off[SP_BINS];   // top-digit histogram -> bucket offsets -> scatter cursors
  __shared__ uint32_t s_hist[SP_BINS];  // histogram of the refinement passes
  __shared__ uint32_t s_warp[SP_THREADS / 32];
  __shared__ uint32_t s_res[3];
  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  const int N = a.N;
  int64_t cid = a.cloud_ids[b];
  cid = cid < 0 ? 0 : (cid >= a.S ? a.S - 1 : cid);
  const int64_t off = a.offsets[cid];
  int64_t P64 = a.offsets[cid + 1] - off;
  P64 = P64 < 0 ? 0 : (P64 > a.max_P ? a.max_P : P64);
  const int P = static_cast<int>(P64);
  // one word view of the cloud's pc_out: the select path keeps its keys there before the gather
  uint32_t* pu = reinterpret_cast<uint32_t*>(a.pc_out) + static_cast<size_t>(b) * 3 * N;
  uint32_t* su = reinterpret_cast<uint32_t*>(a.sn_out) + static_cast<size_t>(b) * 3 * N;
  int64_t* sego = a.seg_out ? a.seg_out + static_cast<size_t>(b) * N : nullptr;
  const float* src = a.data + off * 6;
  const int32_t* lab = a.labels ? a.labels + off : nullptr;

  auto emit = [&](int j, int idx) {
    const float2* r = reinterpret_cast<const float2*>(src + static_cast<size_t>(idx) * 6);
    const float2 v0 = __ldg(r), v1 = __ldg(r + 1), v2 = __ldg(r + 2);
    pu[j] = __float_as_uint(v0.x);
    pu[N + j] = __float_as_uint(v0.y);
    pu[2 * N + j] = __float_as_uint(v1.x);
    su[j] = __float_as_uint(v1.y);
    su[N + j] = __float_as_uint(v2.x);
    su[2 * N + j] = __float_as_uint(v2.y);
    if (sego) sego[j] = lab[idx];
  };

  if (P == 0) {  // an empty cloud has no point to draw: zeros
    for (int j = tid; j < N; j += SP_THREADS) {
      pu[j] = pu[N + j] = pu[2 * N + j] = 0u;
      su[j] = su[N + j] = su[2 * N + j] = 0u;
      if (sego) sego[j] = 0;
    }
    return;
  }
  if (a.indices) {
    const int32_t* given = a.indices + static_cast<size_t>(b) * N;
    for (int j = tid; j < N; j += SP_THREADS) {
      const int32_t g = given[j];
      emit(j, g < 0 ? 0 : (g >= P ? P - 1 : g));
    }
    return;
  }
  if (N > P || (a.rule == SONET_SAMPLE_FILL && N == P)) {
    for (int j = tid; j < N; j += SP_THREADS)
      emit(j, j < P ? j : static_cast<int>(fill_draw(a.k0, a.k1, b, j, P)));
    return;
  }

  // ---- SUBSET (or FILL with N < P): the N smallest keys ----
  for (int i = tid; i < SP_BINS; i += SP_THREADS) s_off[i] = 0;
  __syncthreads();
  for (int i = tid; i < P; i += SP_THREADS)
    atomicAdd(&s_off[select_key(a.k0, a.k1, b, i) >> (64 - SP_DIGIT)], 1u);
  __syncthreads();
  scan_find(s_off, static_cast<uint32_t>(N), true, s_warp, s_res);
  const uint32_t t0 = s_res[0];
  uint32_t r = static_cast<uint32_t>(N) - s_res[1], cnt = s_res[2];
  uint64_t prefix = t0;       // the top `consumed` bits of the N-th smallest key
  int consumed = SP_DIGIT;
  while (cnt != r) {          // the bucket holds keys beyond the N-th: refine by the next digit
    const int bits = 64 - consumed < SP_DIGIT ? 64 - consumed : SP_DIGIT;
    const int shift = 64 - consumed - bits;
    for (int i = tid; i < SP_BINS; i += SP_THREADS) s_hist[i] = 0;
    __syncthreads();
    for (int i = tid; i < P; i += SP_THREADS) {
      const uint64_t key = select_key(a.k0, a.k1, b, i);
      if ((key >> (64 - consumed)) == prefix)
        atomicAdd(&s_hist[(key >> shift) & ((1u << bits) - 1u)], 1u);
    }
    __syncthreads();
    scan_find(s_hist, r, false, s_warp, s_res);
    r -= s_res[1];
    cnt = s_res[2];
    prefix = (prefix << bits) | s_res[0];
    consumed += bits;
  }
  // exactly N keys have (key >> (64 - consumed)) <= prefix; scatter them by top digit
  const int sel_shift = 64 - consumed;
  uint32_t* khi = pu;
  uint32_t* klo = pu + N;
  for (int i = tid; i < P; i += SP_THREADS) {
    const uint64_t key = select_key(a.k0, a.k1, b, i);
    if ((key >> sel_shift) <= prefix) {
      const uint32_t pos = atomicAdd(&s_off[key >> (64 - SP_DIGIT)], 1u);
      khi[pos] = static_cast<uint32_t>(key >> 32);
      klo[pos] = static_cast<uint32_t>(key);
    }
  }
  __syncthreads();
  // s_off[d] is now the end of bucket d (d <= t0) and the start of d+1; sort each bucket
  for (uint32_t d = tid; d <= t0; d += SP_THREADS) {
    const uint32_t lo = d ? s_off[d - 1] : 0u, hi = s_off[d];
    for (uint32_t x = lo + 1; x < hi; ++x) {
      const uint32_t h = khi[x], l = klo[x];
      const uint64_t k = (static_cast<uint64_t>(h) << 32) | l;
      uint32_t y = x;
      while (y > lo && ((static_cast<uint64_t>(khi[y - 1]) << 32) | klo[y - 1]) > k) {
        khi[y] = khi[y - 1];
        klo[y] = klo[y - 1];
        --y;
      }
      khi[y] = h;
      klo[y] = l;
    }
  }
  __syncthreads();
  for (int j = tid; j < N; j += SP_THREADS) emit(j, static_cast<int>(klo[j] & 0xFFFFu));
}

}  // namespace sonet

extern "C" int sonet_sample_points_f32(const float* data, const int64_t* offsets, int S,
                                       const int32_t* labels, const int64_t* cloud_ids, int B,
                                       int N, int max_P, int rule, const int32_t* indices,
                                       unsigned long long seed, float* pc_out, float* sn_out,
                                       int64_t* seg_out, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(rule == SONET_SAMPLE_SUBSET || rule == SONET_SAMPLE_FILL,
                "sample_points: rule %d is not SONET_SAMPLE_SUBSET (0) or _FILL (1)", rule);
  SONET_REQUIRE(N >= 1, "sample_points: N=%d must be >= 1", N);
  SONET_REQUIRE(B >= 0 && B <= 65535, "sample_points: B=%d outside [0, 65535]", B);
  SONET_REQUIRE(S >= 1, "sample_points: S=%d: the dataset needs at least one cloud", S);
  SONET_REQUIRE(max_P >= 1, "sample_points: max_P=%d must be >= 1", max_P);
  SONET_REQUIRE(indices != nullptr || max_P <= SONET_SAMPLE_MAX_P,
                "sample_points: max_P=%d exceeds the in-kernel draws' envelope (%d); pass indices",
                max_P, SONET_SAMPLE_MAX_P);
  SONET_REQUIRE((labels == nullptr) == (seg_out == nullptr),
                "sample_points: labels and seg_out must be both null or both given");
  SONET_REQUIRE(data && offsets && cloud_ids && pc_out && sn_out,
                "sample_points: data, offsets, cloud_ids, pc_out and sn_out must not be null");
  if (B == 0) return SONET_OK;
  SampleArgs a;
  a.data = data;
  a.offsets = offsets;
  a.labels = labels;
  a.cloud_ids = cloud_ids;
  a.indices = indices;
  a.pc_out = pc_out;
  a.sn_out = sn_out;
  a.seg_out = seg_out;
  a.S = S;
  a.N = N;
  a.max_P = max_P;
  a.rule = rule;
  a.k0 = static_cast<uint32_t>(seed);
  a.k1 = static_cast<uint32_t>(seed >> 32);
  sample_points_kernel<<<B, SP_THREADS, 0, as_stream(stream)>>>(a);
  return check_launch("sample_points");
}
