// SHREC'16 same-label retrieval ranking (shrec16/test.py:64-99): for every query q, the items p
// with label[p] == label[q] (q itself included) ranked by d = ||f_q - f_p||_2, at most k of them.
//
// Inputs: feature [Q,D] f32, and either labels [Q] int64 or none (then label = row argmax with
// torch.max's CPU rule: lowest index on ties, the first NaN wins).
//
//   d      = float( sqrt( sum_{j=0..D-1} double(f_q[j] - f_p[j])^2 ) )
//            the difference in fp32, its square accumulated in fp64 in index order (the product of
//            two equal fp32 values is exact in fp64, so DFMA and multiply-then-add agree), sqrt in
//            fp64, one rounding to fp32. A NaN distance is stored as the canonical 0x7fc00000.
//   key    = (bits(d) with the sign cleared) << 32 | p   -- unique per candidate, NaN after +inf
//   out    = the min(group size, k) smallest keys of the query, ascending: idx = p, dist = d.
//            Slots past count hold idx -1 and dist NaN.
//   count  = min(group size, k), or -1 when the query's label is outside [0, L); such an item is
//            nobody's candidate and its row is all -1 / NaN.
//
// Device pipeline (four launches, no allocation, no host synchronisation, graph capturable):
//   1. label:  one warp per item computes the argmax (or checks the given label) and flags
//              invalid items.
//   2. group:  one CTA runs a stable counting sort of the labels: per-warp label histograms (in the
//              caller's scratch), group offsets, and the permutation of positions into group order.
//              It also lays out the work list (group, tile of RT_Q queries) as per-group tile
//              offsets, so no group size ever reaches the host.
//   3. gather: copies the features into group order, so a group is a contiguous block of rows.
//   4. rank:   a fixed grid walks the work list. A CTA holds RT_Q queries of one group (one warp
//              each) and streams the group's rows through shared memory in tiles of RT_C
//              candidates x RT_DC dims, so each tile is read once per query tile.
//
// Top-k design: radix select over the 32-bit distance key, recomputing the distances on each pass,
// then one collecting pass. It was chosen over a running sorted buffer with threshold filtering:
//   - the state per query is one 256-bin histogram in shared memory, independent of k (up to 4096)
//     and of the group size (any size up to Q), where a buffer would need 32 KB per query at
//     k = 4096 and a merge whose cost depends on the input order;
//   - every pass is the same branch-free streaming loop, and exactness holds by construction: the
//     k-th smallest distance value v* and the number kr of ties at v* that fit are found exactly,
//     and the collecting pass takes every key below v* plus the kr lowest positions equal to v*.
// A group with at most k members skips the select and costs one pass; otherwise at most four
// radix passes (8-bit digits, top first) run, stopping as soon as a digit bin closes the count.
// The collected keys go to the query's idx row, and the CTA then sorts each row in shared memory
// (bitonic, up to 4096 keys) and writes the final idx / dist.
//
// The host entry has the same arithmetic and summation order (it sorts the same unique keys), so it
// and the kernel agree bit for bit. The formatter reproduces np.savetxt(fmt='%06d %f') of the
// script's float64 [n,2] rows, without file I/O.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <thread>
#include <vector>

#include "common.cuh"

namespace sonet {

constexpr int RT_MAX_D = 1024;
constexpr int RT_MAX_K = 4096;
constexpr int RT_MAX_L = 4096;
constexpr int RT_Q = 8;                 // queries per rank CTA, one warp each
constexpr int RT_THREADS = RT_Q * 32;
constexpr int RT_CPL = 4;               // candidates per lane per tile
constexpr int RT_C = 32 * RT_CPL;       // candidates per tile
constexpr int RT_DC = 64;               // dims per staged chunk
constexpr int RT_LD = RT_DC + 1;        // odd row stride: lane-per-candidate reads hit 32 banks
constexpr int RT_GROUP_THREADS = 1024;
constexpr unsigned RT_NAN_KEY = 0x7fc00000u;

static_assert(RT_C * RT_LD * 4 >= RT_MAX_K * 8, "the sort buffer reuses the candidate tile");

// Distance key of an fp64 sum of squares: sqrt in fp64, one rounding to fp32, sign cleared,
// every NaN made canonical so that NaNs order by position alone.
__host__ __device__ __forceinline__ unsigned dist_key(double sum) {
#ifdef __CUDA_ARCH__
  const unsigned u = __float_as_uint(__double2float_rn(__dsqrt_rn(sum))) & 0x7fffffffu;
#else
  const float f = static_cast<float>(std::sqrt(sum));
  unsigned u;
  std::memcpy(&u, &f, 4);
  u &= 0x7fffffffu;
#endif
  return u > 0x7f800000u ? RT_NAN_KEY : u;
}

// Row argmax with torch.max's CPU rule (as seg_iou.cu's argmax_step): NaN beats everything and
// the lowest index wins among NaNs; otherwise the larger value, then the lower index. A total
// order, so any reduction tree gives the sequential answer.
__device__ __forceinline__ bool amax_better(float v, int i, float bv, int bi) {
  const bool vn = v != v, bn = bv != bv;
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}

__global__ void __launch_bounds__(256)
    retrieval_label_kernel(const float* __restrict__ feature, const long long* __restrict__ label_in,
                           int Q, int D, int L, int k, int* __restrict__ grp,
                           long long* __restrict__ label_out, long long* __restrict__ idx,
                           float* __restrict__ dist, int32_t* __restrict__ count) {
  const int q = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= Q) return;
  long long lab;
  if (label_in != nullptr) {
    lab = label_in[q];
  } else {
    const float* f = feature + static_cast<size_t>(q) * D;
    float best = f[0];
    int bi = 0;
    for (int j = lane; j < D; j += 32) {  // each lane in index order, then a tree over lanes
      const float v = f[j];
      if (amax_better(v, j, best, bi)) { best = v; bi = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float v = __shfl_xor_sync(0xffffffffu, best, o);
      const int i = __shfl_xor_sync(0xffffffffu, bi, o);
      if (amax_better(v, i, best, bi)) { best = v; bi = i; }
    }
    lab = bi;
  }
  const bool valid = lab >= 0 && lab < L;
  if (lane == 0) {
    grp[q] = valid ? static_cast<int>(lab) : -1;
    if (label_out != nullptr) label_out[q] = lab;
  }
  if (!valid) {
    for (int j = lane; j < k; j += 32) {
      idx[static_cast<size_t>(q) * k + j] = -1;
      dist[static_cast<size_t>(q) * k + j] = __uint_as_float(RT_NAN_KEY);
    }
    if (lane == 0) count[q] = -1;
  }
}

// Exclusive scan of four consecutive values per thread over a 1024-thread block.
__device__ __forceinline__ void block_scan4(int v[4], int* s_warp, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int local = v[0] + v[1] + v[2] + v[3];
  int incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = s_warp[lane], wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    s_warp[lane] = wi - w;
    if (lane == 31) s_warp[32] = wi;
  }
  __syncthreads();
  int run = s_warp[warp] + incl - local;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = v[i];
    v[i] = run;
    run += c;
  }
  total = s_warp[32];
  __syncthreads();
}

// Stable counting sort of the labels in one CTA. Warp w owns the items [w*seg, (w+1)*seg); within
// a warp, items go in index order 32 at a time and __match_any_sync ranks equal labels by lane.
__global__ void __launch_bounds__(RT_GROUP_THREADS)
    retrieval_group_kernel(const int* __restrict__ grp, int Q, int L, int* __restrict__ whist,
                           int* __restrict__ offs, int* __restrict__ tile_off,
                           int* __restrict__ perm) {
  __shared__ int s_off[RT_MAX_L];
  __shared__ int s_warp[33];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int seg = (Q + 31) / 32;
  const int i0 = min(Q, warp * seg), i1 = min(Q, i0 + seg);
  int* wh = whist + static_cast<size_t>(warp) * L;
  for (int l = lane; l < L; l += 32) wh[l] = 0;
  __syncwarp();
  for (int b = i0; b < i1; b += 32) {
    const int i = b + lane;
    const int g = i < i1 ? grp[i] : -1;
    const unsigned m = __match_any_sync(0xffffffffu, g);
    if (g >= 0 && lane == __ffs(m) - 1) wh[g] += __popc(m);
    __syncwarp();
  }
  __syncthreads();
  for (int l = tid; l < L; l += RT_GROUP_THREADS) {  // per label: bases of the warps, and the total
    int run = 0;
    for (int w = 0; w < 32; ++w) {
      const int c = whist[static_cast<size_t>(w) * L + l];
      whist[static_cast<size_t>(w) * L + l] = run;
      run += c;
    }
    s_off[l] = run;
  }
  __syncthreads();
  int n[4], t[4], total, tiles;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int l = tid * 4 + i;
    n[i] = l < L ? s_off[l] : 0;
    t[i] = (n[i] + RT_Q - 1) / RT_Q;
  }
  block_scan4(n, s_warp, total);
  block_scan4(t, s_warp, tiles);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int l = tid * 4 + i;
    if (l < L) {
      s_off[l] = n[i];
      offs[l] = n[i];
      tile_off[l] = t[i];
    }
  }
  if (tid == 0) {
    offs[L] = total;
    tile_off[L] = tiles;
  }
  __syncthreads();
  const unsigned lt = (1u << lane) - 1u;
  for (int b = i0; b < i1; b += 32) {
    const int i = b + lane;
    const int g = i < i1 ? grp[i] : -1;
    const unsigned m = __match_any_sync(0xffffffffu, g);
    int base = 0;
    if (g >= 0) {
      base = wh[g];
      perm[s_off[g] + base + __popc(m & lt)] = i;
    }
    __syncwarp();
    if (g >= 0 && lane == __ffs(m) - 1) wh[g] = base + __popc(m);
    __syncwarp();
  }
}

__global__ void retrieval_gather_kernel(const float* __restrict__ feature, const int* __restrict__ perm,
                                        const int* __restrict__ offs, int L, int D,
                                        float* __restrict__ gathered) {
  const long long n = static_cast<long long>(offs[L]) * D;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < n;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = e / D;
    gathered[e] = feature[static_cast<long long>(perm[r]) * D + (e - r * D)];
  }
}

struct RankSmem {
  union {
    float cand[RT_C * RT_LD];
    unsigned long long sort[RT_MAX_K];
  };
  float query[RT_Q][RT_DC];
  int hist[RT_Q][256];
};

// One streaming pass over the group's candidates: per tile, the distance keys of this warp's query
// to the tile's RT_C candidates (lane holds candidates lane + 32*c), then visit(tile0, keys).
template <typename Visit>
__device__ __forceinline__ void rank_pass(RankSmem& sm, const float* __restrict__ G, int s, int n,
                                          int q0, int D, bool busy, Visit visit) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int tile0 = 0; tile0 < n; tile0 += RT_C) {
    double acc[RT_CPL];
#pragma unroll
    for (int c = 0; c < RT_CPL; ++c) acc[c] = 0.0;
    for (int d0 = 0; d0 < D; d0 += RT_DC) {
      const int dc = min(RT_DC, D - d0);
      __syncthreads();
      for (int r = warp; r < RT_C; r += RT_Q) {
        const int j = tile0 + r;
        const float* src = G + static_cast<size_t>(s + j) * D + d0;
        for (int x = lane; x < dc; x += 32) sm.cand[r * RT_LD + x] = j < n ? src[x] : 0.0f;
      }
      {
        const int j = q0 + warp;
        const float* src = G + static_cast<size_t>(s + j) * D + d0;
        for (int x = lane; x < dc; x += 32) sm.query[warp][x] = j < n ? src[x] : 0.0f;
      }
      __syncthreads();
      if (busy) {
        const float* cq = sm.query[warp];
        const float* cc = sm.cand + lane * RT_LD;
        for (int x = 0; x < dc; ++x) {
          const float qv = cq[x];
#pragma unroll
          for (int c = 0; c < RT_CPL; ++c) {
            const double df = static_cast<double>(__fsub_rn(qv, cc[c * 32 * RT_LD + x]));
            acc[c] = __fma_rn(df, df, acc[c]);
          }
        }
      }
    }
    unsigned key[RT_CPL];
#pragma unroll
    for (int c = 0; c < RT_CPL; ++c) key[c] = dist_key(acc[c]);
    if (busy) visit(tile0, key);
  }
}

__global__ void __launch_bounds__(RT_THREADS, 4)
    retrieval_rank_kernel(const float* __restrict__ G, const int* __restrict__ perm,
                          const int* __restrict__ offs, const int* __restrict__ tile_off, int L,
                          int D, int k, long long* __restrict__ idx, float* __restrict__ dist,
                          int32_t* __restrict__ count) {
  __shared__ __align__(16) RankSmem sm;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const unsigned lt = (1u << lane) - 1u;
  const int items = tile_off[L];
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    int lo = 0, hi = L - 1;  // the last group whose first tile is at or before `item`
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (tile_off[mid] <= item) lo = mid; else hi = mid - 1;
    }
    const int s = offs[lo], n = offs[lo + 1] - s;
    const int q0 = (item - tile_off[lo]) * RT_Q;
    const bool active = q0 + warp < n;
    const long long qrow = active ? static_cast<long long>(perm[s + q0 + warp]) * k : 0;
    const int cnt = min(n, k);

    // select: the key threshold thr and how many keys equal to it are taken (eq_take)
    unsigned thr = 0xffffffffu, prefix = 0;
    int eq_take = 0x7fffffff, kr = k;
    bool busy = active && n > k;
    for (int shift = 24; shift >= 0; shift -= 8) {
      if (!__syncthreads_or(busy)) break;
      for (int b = lane; b < 256; b += 32) sm.hist[warp][b] = 0;
      __syncwarp();
      const unsigned hmask = shift == 24 ? 0u : (0xffffffffu << (shift + 8));
      rank_pass(sm, G, s, n, q0, D, busy, [&](int tile0, const unsigned* key) {
#pragma unroll
        for (int c = 0; c < RT_CPL; ++c)
          if (tile0 + c * 32 + lane < n && ((key[c] ^ prefix) & hmask) == 0)
            atomicAdd(&sm.hist[warp][(key[c] >> shift) & 255u], 1);
      });
      __syncwarp();
      if (busy) {
        int h[8], sum = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) { h[i] = sm.hist[warp][lane * 8 + i]; sum += h[i]; }
        int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += t;
        }
        const unsigned owner = __ballot_sync(0xffffffffu, incl >= kr && incl - sum < kr);
        const int src = __ffs(owner) - 1;
        int digit = 0, before = incl - sum, hb = 0;
        if (lane == src) {
          for (int i = 0; i < 8; ++i) {
            if (before + h[i] >= kr) { digit = lane * 8 + i; hb = h[i]; break; }
            before += h[i];
          }
        }
        digit = __shfl_sync(0xffffffffu, digit, src);
        before = __shfl_sync(0xffffffffu, before, src);
        hb = __shfl_sync(0xffffffffu, hb, src);
        prefix |= static_cast<unsigned>(digit) << shift;
        kr -= before;
        if (hb == kr) {          // the whole bin fits: take every key with this prefix
          thr = prefix | ((1u << shift) - 1u);
          busy = false;
        } else if (shift == 0) { // v* found: take kr of its ties, lowest positions first
          thr = prefix;
          eq_take = kr;
          busy = false;
        }
      }
    }

    // collect: keys below thr, and the first eq_take keys equal to thr in position order
    int taken = 0, eq_seen = 0;
    __syncthreads();
    rank_pass(sm, G, s, n, q0, D, active, [&](int tile0, const unsigned* key) {
#pragma unroll
      for (int c = 0; c < RT_CPL; ++c) {
        const int j = tile0 + c * 32 + lane;
        const bool ok = j < n;
        const bool eq = ok && key[c] == thr;
        const unsigned eqb = __ballot_sync(0xffffffffu, eq);
        const bool take = ok && (key[c] < thr || (eq && eq_seen + __popc(eqb & lt) < eq_take));
        eq_seen += __popc(eqb);
        const unsigned tb = __ballot_sync(0xffffffffu, take);
        if (take)
          idx[qrow + taken + __popc(tb & lt)] =
              static_cast<long long>((static_cast<unsigned long long>(key[c]) << 32) |
                                     static_cast<unsigned>(perm[s + j]));
        taken += __popc(tb);
      }
    });
    __syncthreads();

    // sort each query's cnt keys and write the row
    int P = 1;
    while (P < cnt) P <<= 1;
    for (int w = 0; w < RT_Q && q0 + w < n; ++w) {
      const long long row = static_cast<long long>(perm[s + q0 + w]) * k;
      for (int i = tid; i < P; i += RT_THREADS)
        sm.sort[i] = i < cnt ? static_cast<unsigned long long>(idx[row + i]) : ~0ull;
      __syncthreads();
      for (int kk = 2; kk <= P; kk <<= 1) {
        for (int j = kk >> 1; j > 0; j >>= 1) {
          for (int i = tid; i < P; i += RT_THREADS) {
            const int ij = i ^ j;
            if (ij > i) {
              const unsigned long long a = sm.sort[i], b = sm.sort[ij];
              if ((a > b) == ((i & kk) == 0)) { sm.sort[i] = b; sm.sort[ij] = a; }
            }
          }
          __syncthreads();
        }
      }
      for (int i = tid; i < k; i += RT_THREADS) {
        const unsigned long long key = i < cnt ? sm.sort[i] : 0ull;
        idx[row + i] = i < cnt ? static_cast<long long>(key & 0xffffffffull) : -1;
        dist[row + i] = __uint_as_float(i < cnt ? static_cast<unsigned>(key >> 32) : RT_NAN_KEY);
      }
      if (tid == 0) count[perm[s + q0 + w]] = cnt;
      __syncthreads();
    }
  }
}

// ---- scratch layout --------------------------------------------------------------------------------
struct RetrievalScratch {
  size_t grp, perm, offs, tile_off, whist, gathered, bytes;
};

static size_t align256(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }

static RetrievalScratch retrieval_scratch(int Q, int D, int L) {
  RetrievalScratch r;
  size_t o = 0;
  r.grp = o;      o = align256(o + sizeof(int) * Q);
  r.perm = o;     o = align256(o + sizeof(int) * Q);
  r.offs = o;     o = align256(o + sizeof(int) * (L + 1));
  r.tile_off = o; o = align256(o + sizeof(int) * (L + 1));
  r.whist = o;    o = align256(o + sizeof(int) * 32 * static_cast<size_t>(L));
  r.gathered = o; o = align256(o + sizeof(float) * static_cast<size_t>(Q) * D);
  r.bytes = o;
  return r;
}

static int retrieval_check(const char* what, int Q, int D, int L, int k) {
  SONET_REQUIRE(Q >= 0, "%s: Q=%d must be >= 0", what, Q);
  SONET_REQUIRE(D >= 1 && D <= RT_MAX_D, "%s: D=%d outside [1, %d]", what, D, RT_MAX_D);
  SONET_REQUIRE(k >= 1 && k <= RT_MAX_K, "%s: k=%d outside [1, %d]", what, k, RT_MAX_K);
  SONET_REQUIRE(L >= 1 && L <= RT_MAX_L, "%s: L=%d outside [1, %d]", what, L, RT_MAX_L);
  SONET_REQUIRE(static_cast<long long>(Q) * k < (1LL << 31), "%s: Q*k=%lld must be < 2^31", what,
                static_cast<long long>(Q) * k);
  return SONET_OK;
}

// ---- host entry: the same arithmetic over host pointers ----------------------------------------------
static void retrieval_cpu_range(const float* feature, const int* grp, const int* members,
                                const int* offs, int D, int k, long long* idx, float* dist,
                                int32_t* count, int q0, int q1) {
  std::vector<unsigned long long> keys;
  for (int q = q0; q < q1; ++q) {
    long long* oi = idx + static_cast<size_t>(q) * k;
    float* od = dist + static_cast<size_t>(q) * k;
    const int g = grp[q];
    int cnt = 0;
    if (g >= 0) {
      const int s = offs[g], n = offs[g + 1] - s;
      const float* fq = feature + static_cast<size_t>(q) * D;
      keys.resize(n);
      for (int j = 0; j < n; ++j) {
        const int p = members[s + j];
        const float* fp = feature + static_cast<size_t>(p) * D;
        double acc = 0.0;
        for (int x = 0; x < D; ++x) {
          const double df = static_cast<double>(fq[x] - fp[x]);
          acc += df * df;  // exact product: equal to the device's DFMA
        }
        keys[j] = (static_cast<unsigned long long>(dist_key(acc)) << 32) | static_cast<unsigned>(p);
      }
      cnt = std::min(n, k);
      std::partial_sort(keys.begin(), keys.begin() + cnt, keys.end());
      for (int i = 0; i < cnt; ++i) {
        oi[i] = static_cast<long long>(keys[i] & 0xffffffffull);
        const unsigned u = static_cast<unsigned>(keys[i] >> 32);
        std::memcpy(od + i, &u, 4);
      }
    }
    for (int i = cnt; i < k; ++i) {
      oi[i] = -1;
      std::memcpy(od + i, &RT_NAN_KEY, 4);
    }
    count[q] = g >= 0 ? cnt : -1;
  }
}

// ---- formatter: np.savetxt(fmt='%06d %f') of the float64 rows (id, dist) -----------------------------
static char* put_digits(char* p, unsigned long long v, int width) {
  char tmp[24];
  int n = 0;
  do { tmp[n++] = static_cast<char>('0' + v % 10); v /= 10; } while (v != 0);
  for (int i = n; i < width; ++i) *p++ = '0';
  while (n > 0) *p++ = tmp[--n];
  return p;
}

// '%06d' % float(id): Python formats the integer value of the double.
static char* put_id(char* p, long long id) {
  const double v = static_cast<double>(id);
  if (v >= 9223372036854775808.0) return put_digits(p, static_cast<unsigned long long>(v), 6);
  const long long i = static_cast<long long>(v);
  if (i >= 0) return put_digits(p, static_cast<unsigned long long>(i), 6);
  *p++ = '-';
  return put_digits(p, 0ull - static_cast<unsigned long long>(i), 5);
}

// '%f' % float(d): exact decimal, rounded half to even to 6 places; nan/inf spelled as Python does.
static char* put_f(char* p, float d) {
  const double v = d;
  if (std::isnan(v)) { std::memcpy(p, "nan", 3); return p + 3; }
  if (std::isinf(v)) {
    if (v < 0) *p++ = '-';
    std::memcpy(p, "inf", 3);
    return p + 3;
  }
  if (!std::signbit(v) && v < 4294967296.0) {
    unsigned long long ip = static_cast<unsigned long long>(v), q = 0;
    const double frac = v - static_cast<double>(ip);  // exact
    if (frac >= 0x1p-26) {
      // v has a 24-bit significand and v >= 2^-26, so frac is a multiple of 2^-49
      const unsigned long long F = static_cast<unsigned long long>(frac * 0x1p49);
      const unsigned long long N = F * 15625ull;  // frac * 1e6 = N / 2^43, N < 2^63
      q = N >> 43;
      const unsigned long long r = N & ((1ull << 43) - 1), half = 1ull << 42;
      if (r > half || (r == half && (q & 1))) ++q;
      if (q == 1000000ull) { ++ip; q = 0; }
    }  // below 2^-26 the value rounds to 0.000000
    p = put_digits(p, ip, 1);
    *p++ = '.';
    return put_digits(p, q, 6);
  }
  char buf[64];
  const int n = std::snprintf(buf, sizeof buf, "%f", v);
  std::memcpy(p, buf, n);
  return p + n;
}

static long long format_query(const long long* ids, const long long* idx, const float* dist,
                              int cnt, char* out) {
  char row[96];
  long long total = 0;
  for (int i = 0; i < cnt; ++i) {
    char* e = put_id(row, ids[idx[i]]);
    *e++ = ' ';
    e = put_f(e, dist[i]);
    *e++ = '\n';
    const long long n = e - row;
    if (out != nullptr) std::memcpy(out + total, row, n);
    total += n;
  }
  return total;
}

template <typename F>
static void parallel_for(int n, int threads, F fn) {
  const int T = std::max(1, std::min(threads, n));
  if (T == 1) {
    fn(0, n);
    return;
  }
  std::vector<std::thread> pool;
  for (int t = 0; t < T; ++t)
    pool.emplace_back(fn, static_cast<int>(static_cast<long long>(n) * t / T),
                      static_cast<int>(static_cast<long long>(n) * (t + 1) / T));
  for (auto& th : pool) th.join();
}

}  // namespace sonet

extern "C" long long sonet_retrieval_scratch_bytes(int Q, int D, int L, int k) {
  using namespace sonet;
  if (retrieval_check("retrieval_scratch_bytes", Q, D, L, k) != SONET_OK) return SONET_ERR_BAD_ARG;
  return static_cast<long long>(retrieval_scratch(Q, D, L).bytes);
}

extern "C" int sonet_retrieval_rank_f32(const float* feature, const long long* label_in, int Q,
                                        int D, int L, int k, void* scratch, long long scratch_bytes,
                                        long long* idx, float* dist, int32_t* count,
                                        long long* label_out, sonet_stream_t stream) {
  using namespace sonet;
  const int rc = retrieval_check("retrieval_rank", Q, D, L, k);
  if (rc != SONET_OK) return rc;
  if (Q == 0) return SONET_OK;
  SONET_REQUIRE(feature && scratch && idx && dist && count, "retrieval_rank: null pointer");
  const RetrievalScratch S = retrieval_scratch(Q, D, L);
  SONET_REQUIRE(scratch_bytes >= static_cast<long long>(S.bytes),
                "retrieval_rank: scratch of %lld bytes, %lld needed", scratch_bytes,
                static_cast<long long>(S.bytes));
  SONET_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 255u) == 0,
                "retrieval_rank: scratch must be 256-byte aligned");
  char* base = static_cast<char*>(scratch);
  int* grp = reinterpret_cast<int*>(base + S.grp);
  int* perm = reinterpret_cast<int*>(base + S.perm);
  int* offs = reinterpret_cast<int*>(base + S.offs);
  int* tile_off = reinterpret_cast<int*>(base + S.tile_off);
  int* whist = reinterpret_cast<int*>(base + S.whist);
  float* gathered = reinterpret_cast<float*>(base + S.gathered);
  cudaStream_t st = as_stream(stream);

  retrieval_label_kernel<<<(Q + 7) / 8, 256, 0, st>>>(feature, label_in, Q, D, L, k, grp, label_out,
                                                      idx, dist, count);
  int rc2 = check_launch("retrieval_label");
  if (rc2 != SONET_OK) return rc2;
  retrieval_group_kernel<<<1, RT_GROUP_THREADS, 0, st>>>(grp, Q, L, whist, offs, tile_off, perm);
  rc2 = check_launch("retrieval_group");
  if (rc2 != SONET_OK) return rc2;
  const long long elems = static_cast<long long>(Q) * D;
  const int gblocks = static_cast<int>(std::min<long long>((elems + 255) / 256, sm_count() * 8LL));
  retrieval_gather_kernel<<<gblocks, 256, 0, st>>>(feature, perm, offs, L, D, gathered);
  rc2 = check_launch("retrieval_gather");
  if (rc2 != SONET_OK) return rc2;
  const long long max_items = (Q + RT_Q - 1) / RT_Q + static_cast<long long>(L);
  const int rblocks = static_cast<int>(std::min<long long>(max_items, sm_count() * 4LL));
  retrieval_rank_kernel<<<rblocks, RT_THREADS, 0, st>>>(gathered, perm, offs, tile_off, L, D, k, idx,
                                                        dist, count);
  return check_launch("retrieval_rank");
}

extern "C" int sonet_retrieval_rank_cpu_f32(const float* feature, const long long* label_in, int Q,
                                            int D, int L, int k, long long* idx, float* dist,
                                            int32_t* count, long long* label_out, int thread_num) {
  using namespace sonet;
  const int rc = retrieval_check("retrieval_rank_cpu", Q, D, L, k);
  if (rc != SONET_OK) return rc;
  SONET_REQUIRE(thread_num >= 1, "retrieval_rank_cpu: thread_num must be >= 1");
  if (Q == 0) return SONET_OK;
  SONET_REQUIRE(feature && idx && dist && count, "retrieval_rank_cpu: null pointer");
  std::vector<int> grp(Q), offs(L + 1, 0), members(Q);
  for (int q = 0; q < Q; ++q) {
    long long lab;
    if (label_in != nullptr) {
      lab = label_in[q];
    } else {
      const float* f = feature + static_cast<size_t>(q) * D;
      float best = f[0];
      int bi = 0;
      for (int j = 1; j < D; ++j) {  // torch.max's CPU rule, sequentially
        const float v = f[j];
        if ((best == best) && (v > best || v != v)) { best = v; bi = j; }
      }
      lab = bi;
    }
    if (label_out != nullptr) label_out[q] = lab;
    grp[q] = (lab >= 0 && lab < L) ? static_cast<int>(lab) : -1;
    if (grp[q] >= 0) ++offs[grp[q] + 1];
  }
  for (int l = 0; l < L; ++l) offs[l + 1] += offs[l];
  std::vector<int> fill(offs.begin(), offs.end() - 1);
  for (int q = 0; q < Q; ++q)
    if (grp[q] >= 0) members[fill[grp[q]]++] = q;
  // at least 2^22 distance terms per thread: below that, starting a thread costs more than it saves
  double work = 0.0;
  for (int l = 0; l < L; ++l) {
    const double n = offs[l + 1] - offs[l];
    work += n * n * D;
  }
  const int T = static_cast<int>(std::max(1.0, std::min<double>(thread_num, work / (1 << 22))));
  parallel_for(Q, T, [&](int q0, int q1) {
    retrieval_cpu_range(feature, grp.data(), members.data(), offs.data(), D, k, idx, dist, count, q0,
                        q1);
  });
  return SONET_OK;
}

extern "C" long long sonet_retrieval_format_cpu(const long long* ids, const long long* idx,
                                                const float* dist, const int32_t* count, int Q,
                                                int k, long long* offsets, char* out,
                                                int thread_num) {
  using namespace sonet;
  SONET_REQUIRE(Q >= 0 && k >= 1, "retrieval_format: Q=%d, k=%d", Q, k);
  SONET_REQUIRE(thread_num >= 1, "retrieval_format: thread_num must be >= 1");
  SONET_REQUIRE(offsets != nullptr, "retrieval_format: null offsets");
  if (Q == 0) {
    if (out == nullptr) offsets[0] = 0;
    return out == nullptr ? 0 : offsets[0];
  }
  SONET_REQUIRE(ids && idx && dist && count, "retrieval_format: null pointer");
  for (int q = 0; q < Q; ++q) {
    SONET_REQUIRE(count[q] >= 0 && count[q] <= k,
                  "retrieval_format: count[%d]=%d outside [0, k=%d] (a label outside the range?)", q,
                  count[q], k);
    for (int i = 0; i < count[q]; ++i) {
      const long long p = idx[static_cast<size_t>(q) * k + i];
      SONET_REQUIRE(p >= 0 && p < Q, "retrieval_format: idx[%d,%d]=%lld outside [0, Q=%d)", q, i, p,
                    Q);
    }
  }
  const int T = std::max(1, std::min(thread_num, Q / 64));
  if (out == nullptr) {  // size query: per-query byte offsets
    offsets[0] = 0;
    parallel_for(Q, T, [&](int q0, int q1) {
      for (int q = q0; q < q1; ++q)
        offsets[q + 1] = format_query(ids, idx + static_cast<size_t>(q) * k,
                                      dist + static_cast<size_t>(q) * k, count[q], nullptr);
    });
    for (int q = 0; q < Q; ++q) offsets[q + 1] += offsets[q];
    return offsets[Q];
  }
  std::vector<char> bad(Q, 0);
  parallel_for(Q, T, [&](int q0, int q1) {
    for (int q = q0; q < q1; ++q) {
      const long long n = format_query(ids, idx + static_cast<size_t>(q) * k,
                                       dist + static_cast<size_t>(q) * k, count[q], nullptr);
      if (offsets[q] < 0 || offsets[q + 1] - offsets[q] != n) {
        bad[q] = 1;
        continue;
      }
      format_query(ids, idx + static_cast<size_t>(q) * k, dist + static_cast<size_t>(q) * k,
                   count[q], out + offsets[q]);
    }
  });
  for (int q = 0; q < Q; ++q)
    SONET_REQUIRE(!bad[q], "retrieval_format: offsets do not match the size query at query %d", q);
  return offsets[Q];
}
