// Part-segmentation IoU of the reference's metric (models/losses.py:73-189, compute_iou_np_array /
// compute_iou, as called by part-seg/train.py:95), one launch for the whole batch.
//
// Inputs: score [B,C,N] f32, seg [B,N] int64, label [B] int64, and a part table in CSR form:
// category k owns part_ids[part_offsets[k] .. part_offsets[k+1]) in table order.
//
//   pred[b,n]   = argmax over c of score[b,c,n]; ties go to the lowest c; a NaN wins, and the first
//                 NaN among NaNs (torch.max(score, dim=1) on CPU tensors).
//   for each part p of category label[b], in table order:
//     I = #{n : seg==p and pred==p},  U = #{n : seg==p or pred==p}
//     iou_p = 1.0 if U == 0 else I / (U + 0.0001)          (double, as Python evaluates it)
//   iou_shape[b] = (((iou_0 + iou_1) + ...) + iou_{P-1}) / P  (double, left to right)
//   correct[b]  = #{n : pred == seg}
//
// The left-to-right sum equals numpy's np.asarray(iou_pc).mean() bit for bit while P < 8 (numpy
// sums blocks of fewer than 8 elements sequentially; the default table has at most 6 parts per
// category). A custom table with 8 or more parts in one category may differ from numpy in the last
// ulp. seg values may be any integer: values that are not a part of the category never match.
//
// Device layout: one CTA per cloud. Threads stride over points and read score[b,:,n] coalesced along
// n; three integer counters per part of the cloud's category (gt hits G, predicted hits P, both I;
// U = G + P - I) live in shared memory and are bumped with shared atomics, so the result does not
// depend on the order the threads run in. Warp 0 then turns the counters into IoUs and the mean in
// double. No scratch, no allocation, no host synchronisation: the call is CUDA-graph capturable.
// The whole batch is a few MB of scores, so the launch dominates; one launch is the design target.
//
// Errors: the host entry returns SONET_ERR_BAD_ARG for a label outside [0, num_categories), a
// malformed table or a part id outside [0, C). The device entry cannot read device memory without
// synchronising, so it writes iou_shape[b] = NaN for a cloud whose label is outside the table (or
// whose category has no part or more than SEG_IOU_MAX_PARTS); pred and correct are still written.
// Its caller validates the table on the host before uploading it.
#include <algorithm>
#include <cmath>
#include <thread>
#include <vector>

#include "common.cuh"

namespace sonet {

constexpr int SEG_IOU_THREADS = 256;
constexpr int SEG_IOU_MAX_PARTS = 256;

// Running argmax over the class axis with torch.max's CPU rules. Branch-free, so that the host
// loop over points vectorises.
__host__ __device__ __forceinline__ void argmax_step(float v, int c, float& best, int& bi) {
  const bool take = (best == best) & ((v > best) | (v != v));
  best = take ? v : best;
  bi = take ? c : bi;
}

__host__ __device__ __forceinline__ double part_iou(int g, int p, int i) {
  const int u = g + p - i;
  return u == 0 ? 1.0 : static_cast<double>(i) / (static_cast<double>(u) + 0.0001);
}

__global__ void __launch_bounds__(SEG_IOU_THREADS)
    seg_iou_kernel(const float* __restrict__ score, const long long* __restrict__ seg,
                   const long long* __restrict__ label, int C, int N,
                   const int32_t* __restrict__ part_offsets, const int32_t* __restrict__ part_ids,
                   int num_categories, double* __restrict__ iou_shape, long long* __restrict__ pred,
                   int32_t* __restrict__ correct) {
  __shared__ int s_ids[SEG_IOU_MAX_PARTS];
  __shared__ int s_g[SEG_IOU_MAX_PARTS], s_p[SEG_IOU_MAX_PARTS], s_i[SEG_IOU_MAX_PARTS];
  __shared__ double s_iou[SEG_IOU_MAX_PARTS];
  __shared__ int s_correct;

  const int b = blockIdx.x;
  const long long lab = label[b];
  int first = 0, np = 0;
  if (lab >= 0 && lab < num_categories) {
    first = part_offsets[lab];
    np = part_offsets[lab + 1] - first;
  }
  const bool valid = np >= 1 && np <= SEG_IOU_MAX_PARTS;
  if (!valid) np = 0;
  for (int j = threadIdx.x; j < np; j += SEG_IOU_THREADS) {
    s_ids[j] = part_ids[first + j];
    s_g[j] = s_p[j] = s_i[j] = 0;
  }
  if (threadIdx.x == 0) s_correct = 0;
  __syncthreads();

  const float* sc = score + static_cast<size_t>(b) * C * N;
  const long long* sg = seg + static_cast<size_t>(b) * N;
  int my_correct = 0;
  for (int n = threadIdx.x; n < N; n += SEG_IOU_THREADS) {
    float best = __ldg(sc + n);
    int bi = 0;
#pragma unroll 10
    for (int c = 1; c < C; ++c) argmax_step(__ldg(sc + static_cast<size_t>(c) * N + n), c, best, bi);
    const long long s = __ldg(sg + n);
    my_correct += (s == bi);
    if (pred != nullptr) pred[static_cast<size_t>(b) * N + n] = bi;
    // first slot of each id: a part listed twice reads the counters of its first listing
    int gs = -1, ps = -1;
    for (int j = 0; j < np; ++j) {
      const int id = s_ids[j];
      if (gs < 0 && id == s) gs = j;
      if (ps < 0 && id == bi) ps = j;
    }
    if (gs >= 0) atomicAdd(&s_g[gs], 1);
    if (ps >= 0) atomicAdd(&s_p[ps], 1);
    if (gs >= 0 && gs == ps) atomicAdd(&s_i[gs], 1);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) my_correct += __shfl_xor_sync(0xffffffffu, my_correct, o);
  if ((threadIdx.x & 31) == 0 && my_correct != 0) atomicAdd(&s_correct, my_correct);
  __syncthreads();

  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  for (int j = lane; j < np; j += 32) {
    int f = 0;
    while (s_ids[f] != s_ids[j]) ++f;
    s_iou[j] = part_iou(s_g[f], s_p[f], s_i[f]);
  }
  __syncwarp();
  if (lane == 0) {
    if (valid) {
      double sum = 0.0;
      for (int j = 0; j < np; ++j) sum += s_iou[j];
      iou_shape[b] = sum / static_cast<double>(np);
    } else {
      iou_shape[b] = __longlong_as_double(0x7ff8000000000000LL);
    }
    if (correct != nullptr) correct[b] = s_correct;
  }
}

// Ragged twin: score [T,C] point-major, seg [T], shape b owns points offsets[b] .. offsets[b+1]. The
// same argmax, counters and IoU arithmetic as seg_iou_kernel, one CTA per shape; pred [T] holds the
// argmax of every point. A shape whose offsets are not inside [0, T] and ordered gets NaN.
__global__ void __launch_bounds__(SEG_IOU_THREADS)
    seg_iou_ragged_kernel(const float* __restrict__ score, const long long* __restrict__ seg,
                          const long long* __restrict__ label, const long long* __restrict__ offsets,
                          int C, long long T, const int32_t* __restrict__ part_offsets,
                          const int32_t* __restrict__ part_ids, int num_categories,
                          double* __restrict__ iou_shape, long long* __restrict__ pred,
                          int32_t* __restrict__ correct) {
  __shared__ int s_ids[SEG_IOU_MAX_PARTS];
  __shared__ int s_g[SEG_IOU_MAX_PARTS], s_p[SEG_IOU_MAX_PARTS], s_i[SEG_IOU_MAX_PARTS];
  __shared__ double s_iou[SEG_IOU_MAX_PARTS];
  __shared__ int s_correct;

  const int b = blockIdx.x;
  const long long lab = label[b];
  long long n0 = offsets[b], n1 = offsets[b + 1];
  const bool range_ok = n0 >= 0 && n0 <= n1 && n1 <= T;
  if (!range_ok) n0 = n1 = 0;
  int first = 0, np = 0;
  if (lab >= 0 && lab < num_categories) {
    first = part_offsets[lab];
    np = part_offsets[lab + 1] - first;
  }
  const bool valid = range_ok && np >= 1 && np <= SEG_IOU_MAX_PARTS;
  if (!valid) np = 0;
  for (int j = threadIdx.x; j < np; j += SEG_IOU_THREADS) {
    s_ids[j] = part_ids[first + j];
    s_g[j] = s_p[j] = s_i[j] = 0;
  }
  if (threadIdx.x == 0) s_correct = 0;
  __syncthreads();

  int my_correct = 0;
  for (long long n = n0 + threadIdx.x; n < n1; n += SEG_IOU_THREADS) {
    const float* row = score + static_cast<size_t>(n) * C;
    float best = __ldg(row);
    int bi = 0;
#pragma unroll 10
    for (int c = 1; c < C; ++c) argmax_step(__ldg(row + c), c, best, bi);
    const long long s = __ldg(seg + n);
    my_correct += (s == bi);
    if (pred != nullptr) pred[n] = bi;
    int gs = -1, ps = -1;
    for (int j = 0; j < np; ++j) {
      const int id = s_ids[j];
      if (gs < 0 && id == s) gs = j;
      if (ps < 0 && id == bi) ps = j;
    }
    if (gs >= 0) atomicAdd(&s_g[gs], 1);
    if (ps >= 0) atomicAdd(&s_p[ps], 1);
    if (gs >= 0 && gs == ps) atomicAdd(&s_i[gs], 1);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) my_correct += __shfl_xor_sync(0xffffffffu, my_correct, o);
  if ((threadIdx.x & 31) == 0 && my_correct != 0) atomicAdd(&s_correct, my_correct);
  __syncthreads();

  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  for (int j = lane; j < np; j += 32) {
    int f = 0;
    while (s_ids[f] != s_ids[j]) ++f;
    s_iou[j] = part_iou(s_g[f], s_p[f], s_i[f]);
  }
  __syncwarp();
  if (lane == 0) {
    if (valid) {
      double sum = 0.0;
      for (int j = 0; j < np; ++j) sum += s_iou[j];
      iou_shape[b] = sum / static_cast<double>(np);
    } else {
      iou_shape[b] = __longlong_as_double(0x7ff8000000000000LL);
    }
    if (correct != nullptr) correct[b] = s_correct;
  }
}

// ---- host entry: the same arithmetic over host pointers -----------------------------------------
static void seg_iou_cpu_range(const float* score, const long long* seg, const long long* label, int C,
                              int N, const int32_t* part_offsets, const int32_t* part_ids,
                              double* iou_shape, long long* pred, int32_t* correct, int b0, int b1) {
  std::vector<int> g, p, i, bis(N);
  for (int b = b0; b < b1; ++b) {
    const float* sc = score + static_cast<size_t>(b) * C * N;
    const long long* sg = seg + static_cast<size_t>(b) * N;
    const int first = part_offsets[label[b]];
    const int np = part_offsets[label[b] + 1] - first;
    const int32_t* ids = part_ids + first;
    g.assign(np, 0);
    p.assign(np, 0);
    i.assign(np, 0);
    std::vector<float> best(sc, sc + N);
    std::fill(bis.begin(), bis.end(), 0);
    for (int c = 1; c < C; ++c) {  // class-major: streams each score row once
      const float* row = sc + static_cast<size_t>(c) * N;
      for (int n = 0; n < N; ++n) argmax_step(row[n], c, best[n], bis[n]);
    }
    int corr = 0;
    for (int n = 0; n < N; ++n) {
      const long long s = sg[n];
      const int bi = bis[n];
      corr += (s == bi);
      if (pred != nullptr) pred[static_cast<size_t>(b) * N + n] = bi;
      int gs = -1, ps = -1;
      for (int j = 0; j < np; ++j) {
        if (gs < 0 && ids[j] == s) gs = j;
        if (ps < 0 && ids[j] == bi) ps = j;
      }
      if (gs >= 0) ++g[gs];
      if (ps >= 0) ++p[ps];
      if (gs >= 0 && gs == ps) ++i[gs];
    }
    double sum = 0.0;
    for (int j = 0; j < np; ++j) {
      int f = 0;
      while (ids[f] != ids[j]) ++f;
      sum += part_iou(g[f], p[f], i[f]);
    }
    iou_shape[b] = sum / static_cast<double>(np);
    if (correct != nullptr) correct[b] = corr;
  }
}

static void seg_iou_ragged_cpu_range(const float* score, const long long* seg, const long long* label,
                                     const long long* offsets, int C, const int32_t* part_offsets,
                                     const int32_t* part_ids, double* iou_shape, long long* pred,
                                     int32_t* correct, int b0, int b1) {
  std::vector<int> g, p, i;
  for (int b = b0; b < b1; ++b) {
    const int first = part_offsets[label[b]];
    const int np = part_offsets[label[b] + 1] - first;
    const int32_t* ids = part_ids + first;
    g.assign(np, 0);
    p.assign(np, 0);
    i.assign(np, 0);
    int corr = 0;
    for (long long n = offsets[b]; n < offsets[b + 1]; ++n) {
      const float* row = score + static_cast<size_t>(n) * C;
      float best = row[0];
      int bi = 0;
      for (int c = 1; c < C; ++c) argmax_step(row[c], c, best, bi);
      const long long s = seg[n];
      corr += (s == bi);
      if (pred != nullptr) pred[n] = bi;
      int gs = -1, ps = -1;
      for (int j = 0; j < np; ++j) {
        if (gs < 0 && ids[j] == s) gs = j;
        if (ps < 0 && ids[j] == bi) ps = j;
      }
      if (gs >= 0) ++g[gs];
      if (ps >= 0) ++p[ps];
      if (gs >= 0 && gs == ps) ++i[gs];
    }
    double sum = 0.0;
    for (int j = 0; j < np; ++j) {
      int f = 0;
      while (ids[f] != ids[j]) ++f;
      sum += part_iou(g[f], p[f], i[f]);
    }
    iou_shape[b] = sum / static_cast<double>(np);
    if (correct != nullptr) correct[b] = corr;
  }
}

}  // namespace sonet

extern "C" int sonet_seg_iou_f32(const float* score, const long long* seg, const long long* label,
                                 int B, int C, int N, const int32_t* part_offsets,
                                 const int32_t* part_ids, int num_categories, double* iou_shape,
                                 long long* pred, int32_t* correct, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 1 && N >= 0 && num_categories >= 1, "seg_iou: bad dimension");
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(score && seg && label && part_offsets && part_ids && iou_shape,
                "seg_iou: null pointer");
  seg_iou_kernel<<<B, SEG_IOU_THREADS, 0, as_stream(stream)>>>(
      score, seg, label, C, N, part_offsets, part_ids, num_categories, iou_shape, pred, correct);
  return check_launch("seg_iou");
}

extern "C" int sonet_seg_iou_cpu_f32(const float* score, const long long* seg, const long long* label,
                                     int B, int C, int N, const int32_t* part_offsets,
                                     const int32_t* part_ids, int num_categories, double* iou_shape,
                                     long long* pred, int32_t* correct, int thread_num) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 1 && N >= 0 && num_categories >= 1, "seg_iou_cpu: bad dimension");
  SONET_REQUIRE(thread_num >= 1, "seg_iou_cpu: thread_num must be >= 1");
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(score && seg && label && part_offsets && part_ids && iou_shape,
                "seg_iou_cpu: null pointer");
  SONET_REQUIRE(part_offsets[0] == 0, "seg_iou_cpu: part_offsets[0] must be 0");
  for (int k = 0; k < num_categories; ++k) {
    const int np = part_offsets[k + 1] - part_offsets[k];
    SONET_REQUIRE(np >= 1 && np <= SEG_IOU_MAX_PARTS,
                  "seg_iou_cpu: category %d has %d parts (1..%d allowed)", k, np, SEG_IOU_MAX_PARTS);
  }
  for (int j = 0; j < part_offsets[num_categories]; ++j)
    SONET_REQUIRE(part_ids[j] >= 0 && part_ids[j] < C, "seg_iou_cpu: part id %d outside [0, C=%d)",
                  part_ids[j], C);
  for (int b = 0; b < B; ++b)
    SONET_REQUIRE(label[b] >= 0 && label[b] < num_categories,
                  "seg_iou_cpu: label[%d]=%lld outside the part table (%d categories)", b, label[b],
                  num_categories);
  // at least 2^20 score elements per thread: below that, starting a thread costs more than it saves
  const long long work = (static_cast<long long>(B) * C * N) >> 20;
  const int T = static_cast<int>(std::min<long long>({thread_num, B, std::max(work, 1LL)}));
  if (T == 1) {
    seg_iou_cpu_range(score, seg, label, C, N, part_offsets, part_ids, iou_shape, pred, correct, 0, B);
    return SONET_OK;
  }
  std::vector<std::thread> pool;
  for (int t = 0; t < T; ++t) {
    const int b0 = static_cast<int>(static_cast<long long>(B) * t / T);
    const int b1 = static_cast<int>(static_cast<long long>(B) * (t + 1) / T);
    pool.emplace_back(seg_iou_cpu_range, score, seg, label, C, N, part_offsets, part_ids, iou_shape,
                      pred, correct, b0, b1);
  }
  for (auto& th : pool) th.join();
  return SONET_OK;
}

extern "C" int sonet_seg_iou_ragged_f32(const float* score, const long long* seg, const long long* label,
                                        const long long* offsets, int B, int C, long long T,
                                        const int32_t* part_offsets, const int32_t* part_ids,
                                        int num_categories, double* iou_shape, long long* pred,
                                        int32_t* correct, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 1 && T >= 0 && num_categories >= 1, "seg_iou_ragged: bad dimension");
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(score && seg && label && offsets && part_offsets && part_ids && iou_shape,
                "seg_iou_ragged: null pointer");
  seg_iou_ragged_kernel<<<B, SEG_IOU_THREADS, 0, as_stream(stream)>>>(
      score, seg, label, offsets, C, T, part_offsets, part_ids, num_categories, iou_shape, pred,
      correct);
  return check_launch("seg_iou_ragged");
}

extern "C" int sonet_seg_iou_ragged_cpu_f32(const float* score, const long long* seg,
                                            const long long* label, const long long* offsets, int B,
                                            int C, long long T, const int32_t* part_offsets,
                                            const int32_t* part_ids, int num_categories,
                                            double* iou_shape, long long* pred, int32_t* correct,
                                            int thread_num) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 1 && T >= 0 && num_categories >= 1, "seg_iou_ragged_cpu: bad dimension");
  SONET_REQUIRE(thread_num >= 1, "seg_iou_ragged_cpu: thread_num must be >= 1");
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(score && seg && label && offsets && part_offsets && part_ids && iou_shape,
                "seg_iou_ragged_cpu: null pointer");
  SONET_REQUIRE(offsets[0] == 0 && offsets[B] == T,
                "seg_iou_ragged_cpu: offsets must run from 0 to T=%lld (got %lld .. %lld)", T,
                offsets[0], offsets[B]);
  for (int b = 0; b < B; ++b)
    SONET_REQUIRE(offsets[b] <= offsets[b + 1], "seg_iou_ragged_cpu: offsets decrease at shape %d", b);
  SONET_REQUIRE(part_offsets[0] == 0, "seg_iou_ragged_cpu: part_offsets[0] must be 0");
  for (int k = 0; k < num_categories; ++k) {
    const int np = part_offsets[k + 1] - part_offsets[k];
    SONET_REQUIRE(np >= 1 && np <= SEG_IOU_MAX_PARTS,
                  "seg_iou_ragged_cpu: category %d has %d parts (1..%d allowed)", k, np,
                  SEG_IOU_MAX_PARTS);
  }
  for (int j = 0; j < part_offsets[num_categories]; ++j)
    SONET_REQUIRE(part_ids[j] >= 0 && part_ids[j] < C,
                  "seg_iou_ragged_cpu: part id %d outside [0, C=%d)", part_ids[j], C);
  for (int b = 0; b < B; ++b)
    SONET_REQUIRE(label[b] >= 0 && label[b] < num_categories,
                  "seg_iou_ragged_cpu: label[%d]=%lld outside the part table (%d categories)", b,
                  label[b], num_categories);
  // at least 2^20 score elements per thread, as the fixed-N entry
  const long long work = (T * C) >> 20;
  const int T_ = static_cast<int>(std::min<long long>({thread_num, B, std::max(work, 1LL)}));
  if (T_ == 1) {
    seg_iou_ragged_cpu_range(score, seg, label, offsets, C, part_offsets, part_ids, iou_shape, pred,
                             correct, 0, B);
    return SONET_OK;
  }
  std::vector<std::thread> pool;
  for (int t = 0; t < T_; ++t) {
    const int b0 = static_cast<int>(static_cast<long long>(B) * t / T_);
    const int b1 = static_cast<int>(static_cast<long long>(B) * (t + 1) / T_);
    pool.emplace_back(seg_iou_ragged_cpu_range, score, seg, label, offsets, C, part_offsets, part_ids,
                      iou_shape, pred, correct, b0, b1);
  }
  for (auto& th : pool) th.join();
  return SONET_OK;
}
