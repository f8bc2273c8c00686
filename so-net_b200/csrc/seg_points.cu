// seg_points.cu — SOM assignment and decentring of ragged point clouds for the segmenter's per-point
// head (segmenter.Model.score_points): every point of each shape, not only the N sampled ones.
//
// One chunk of rows [row0, row0 + rows) of a stacked ragged set points [T, 6] (xyz | normal, cloud b
// owns rows offsets[b] .. offsets[b+1]) is laid out as one batch row of k*rows_pad columns, copy-major
// like the encoder's stacked copies (column s*rows_pad + r is copy s of row r):
//
//   gidx[s*rows_pad + r]       = b*M + m_s     flat (cloud, node) id of the s-th nearest node
//   x_aug[c][s*rows_pad + r]   = x_c - cm[b,c,m_s] (c < 3), then the normal     (the first PointResNet's input)
//   pt[c][s*rows_pad + r]      = x_dec | x | cm[b,:,m_s] | normal               (layer 1's per-point rows)
//
// m_s is the s-th nearest of cloud b's M loader nodes by the SOM assignment rule of common.cuh
// (som_topk: sonet_som_assign's bits). cm is the cluster mean the encoder computed on the sampled
// batch (Encoder.som_node). Columns of rows r >= rows are padding: zeros and node 0 of cloud 0, so
// that whatever reads them stays finite and in range.
//
// Each row finds its cloud by a binary search over offsets on the device (common.cuh, ragged_find):
// one launch per chunk, no host round trip per cloud. offsets are not read on the host; a row outside
// [offsets[0], offsets[B]) of non-monotone offsets lands in cloud 0 or B-1 (the Python caller
// validates offsets once).
#include <algorithm>

#include "common.cuh"

namespace sonet {

constexpr int SEGPT_MAX_M = 256;
constexpr int SEGPT_MAX_K = 4;
constexpr int SEGPT_THREADS = 256;

template <int KK>
__global__ void __launch_bounds__(SEGPT_THREADS)
    seg_points_assign_kernel(const float* __restrict__ points, long long total,
                             const long long* __restrict__ offsets, int B, const float* __restrict__ node,
                             const float* __restrict__ cluster_mean, int M, int with_sn,
                             long long row0, int rows, int rows_pad, int32_t* __restrict__ gidx,
                             float* __restrict__ x_aug, float* __restrict__ pt) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows_pad) return;
  const size_t KR = static_cast<size_t>(KK) * rows_pad;
  const int CA = with_sn ? 6 : 3, CP = with_sn ? 12 : 9;
  if (r >= rows) {
#pragma unroll
    for (int s = 0; s < KK; ++s) {
      const size_t j = static_cast<size_t>(s) * rows_pad + r;
      gidx[j] = 0;
      for (int c = 0; c < CA; ++c) x_aug[c * KR + j] = 0.f;
      for (int c = 0; c < CP; ++c) pt[c * KR + j] = 0.f;
    }
    return;
  }
  const long long g = row0 + r;
  long long lo, hi;   // the cloud's rows: unused, a row outside it still takes the cloud found
  const int b = ragged_find(offsets, B, total, g, lo, hi);
  const float* p = points + static_cast<size_t>(g) * 6;
  const float px = p[0], py = p[1], pz = p[2];
  const float* nb = node + static_cast<size_t>(b) * 3 * M;
  float bd[KK];
  int bi[KK];
  som_topk(M, [&](int m) {
    return som_dist_rn(px, py, pz, __ldg(nb + m), __ldg(nb + M + m), __ldg(nb + 2 * M + m));
  }, bd, bi);

  const float* cm = cluster_mean + static_cast<size_t>(b) * 3 * M;
  const float xv[3] = {px, py, pz};
#pragma unroll
  for (int s = 0; s < KK; ++s) {
    const int id = min(max(bi[s], 0), M - 1);
    const size_t j = static_cast<size_t>(s) * rows_pad + r;
    gidx[j] = b * M + id;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float ctr = __ldg(cm + c * M + id);
      const float dec = __fsub_rn(xv[c], ctr);   // som_decenter_kernel's x_decentered
      x_aug[c * KR + j] = dec;
      pt[c * KR + j] = dec;
      pt[(3 + c) * KR + j] = xv[c];
      pt[(6 + c) * KR + j] = ctr;
      if (with_sn) {
        x_aug[(3 + c) * KR + j] = p[3 + c];
        pt[(9 + c) * KR + j] = p[3 + c];
      }
    }
  }
}

}  // namespace sonet

extern "C" int sonet_seg_points_assign_f32(const float* points, long long total,
                                           const long long* offsets, int B, const float* node,
                                           const float* cluster_mean, int M, int k, int with_sn,
                                           long long row0, int rows, int rows_pad, int32_t* gidx,
                                           float* x_aug, float* pt, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 1 && total >= 0 && rows >= 0 && rows_pad >= rows && row0 >= 0,
                "seg_points_assign: bad dimension (B=%d, total=%lld, row0=%lld, rows=%d, rows_pad=%d)",
                B, total, row0, rows, rows_pad);
  SONET_REQUIRE(M >= 1 && M <= SEGPT_MAX_M, "seg_points_assign: M=%d out of range [1,%d]", M,
                SEGPT_MAX_M);
  SONET_REQUIRE(k >= 1 && k <= SEGPT_MAX_K && k <= M,
                "seg_points_assign: k=%d out of range [1,%d] (and k <= M=%d)", k, SEGPT_MAX_K, M);
  SONET_REQUIRE(with_sn == 0 || with_sn == 1, "seg_points_assign: with_sn must be 0 or 1");
  SONET_REQUIRE(row0 + rows <= total, "seg_points_assign: rows [%lld, %lld) outside the %lld points",
                row0, row0 + rows, total);
  SONET_REQUIRE(static_cast<long long>(k) * rows_pad * (with_sn ? 12 : 9) < (1LL << 31),
                "seg_points_assign: chunk of %d rows too large", rows_pad);
  SONET_REQUIRE(static_cast<long long>(B) * M < (1LL << 31), "seg_points_assign: B*M too large");
  if (rows_pad == 0) return SONET_OK;
  SONET_REQUIRE(points && offsets && node && cluster_mean && gidx && x_aug && pt,
                "seg_points_assign: null pointer");
  const int grid = (rows_pad + SEGPT_THREADS - 1) / SEGPT_THREADS;
  cudaStream_t st = as_stream(stream);
  switch (k) {
    case 1: seg_points_assign_kernel<1><<<grid, SEGPT_THREADS, 0, st>>>(points, total, offsets, B, node, cluster_mean, M, with_sn, row0, rows, rows_pad, gidx, x_aug, pt); break;
    case 2: seg_points_assign_kernel<2><<<grid, SEGPT_THREADS, 0, st>>>(points, total, offsets, B, node, cluster_mean, M, with_sn, row0, rows, rows_pad, gidx, x_aug, pt); break;
    case 3: seg_points_assign_kernel<3><<<grid, SEGPT_THREADS, 0, st>>>(points, total, offsets, B, node, cluster_mean, M, with_sn, row0, rows, rows_pad, gidx, x_aug, pt); break;
    default: seg_points_assign_kernel<4><<<grid, SEGPT_THREADS, 0, st>>>(points, total, offsets, B, node, cluster_mean, M, with_sn, row0, rows, rows_pad, gidx, x_aug, pt); break;
  }
  return check_launch("seg_points_assign");
}
