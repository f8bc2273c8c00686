// train.cu — train-mode kernels of the point-wise layers (SURVEY.md §8f-2) for sm_90a.
//
// The reference trains through EquivariantLayer = Conv1d(k=1) -> MyBatchNorm1d (batch statistics,
// models/layers.py:22-70) -> ReLU (or ELU), and back-propagates through the per-node pool as the backward
// of a gather (models/networks.py:185). PyTorch runs that as conv + batch_norm + relu (+ three
// backward kernels each) and a zero-fill + scatter for the gather. Here:
//
//   bn forward (3 launches)      one fp64 record of sums per (cloud, channel) of x[B,C,P], the
//                                records folded in ascending cloud order into the batch statistics,
//                                then y = act(gamma * (x - mean) * invstd + beta) in ONE elementwise pass
//   bn backward (3 launches)     per-(cloud, channel) records of the sums of g and g*xhat (g = dy
//                                times the activation's derivative at the recomputed BN output z:
//                                [z > 0] for ReLU, z > 0 ? 1 : exp(z) for ELU), folded like the
//                                forward's, then dx = gamma*invstd*(g - mean(g) - xhat*mean(g*xhat));
//                                dgamma, dbeta fall out of the sums
//   instance_norm (1 launch)     per-row statistics of z[B,C,P] (InstanceNorm, eval and train
//                                alike) and y = act(gamma*(z-mean)*invstd + beta), optionally reduced
//                                to the k-copy mean or the max over groups of K; its backward is
//                                the bn backward on the [1, B*C, P] view
//   index_max_backward           grad of first_pn_out through the masked gather: zero-fill +
//                                scatter-add of grad[b,c,k] at idx[b,c,k] (duplicates — every empty
//                                node gathers point 0 — are added by ONE thread in ascending k)
//   tc_pack_device               fp32 weights -> wgmma hi/lo blob ON THE DEVICE (weights change
//                                every optimizer step; the eval path packs on the host once), also
//                                transposed: the dgrad GEMM dx = W^T dy runs on the same generic
//                                wgmma layer kernel as the forward (csrc/pointwise_tc.cu); and the
//                                activations x as the weight operand of the wgrad GEMM
//
// All reductions are two-stage with fp64 partial sums in a fixed order: bit-reproducible.
#include <algorithm>
#include <cmath>
#include <type_traits>

#include "tc_common.cuh"

namespace sonet {

// d elu(z) / dz, from the BN output z (alpha = 1: exp(z) = elu(z) + 1 below 0)
__device__ __forceinline__ float elu_grad(float z) { return z > 0.f ? 1.f : expf(z); }

// y = act(gamma*(x-mean)*invstd + beta); grid (ceil(P/1024), C, B)
template <bool ELU>
__global__ void __launch_bounds__(256)
    bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                    const float* __restrict__ invstd, const float* __restrict__ gamma,
                    const float* __restrict__ beta, int C, int P, int relu, float* __restrict__ y) {
  const int c = blockIdx.y, b = blockIdx.z;
  const float is = invstd[c], ga = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f, mu = mean[c];
  const size_t o = (static_cast<size_t>(b) * C + c) * P;
  for (int p = blockIdx.x * 1024 + threadIdx.x; p < min(P, (static_cast<int>(blockIdx.x) + 1) * 1024);
       p += 256) {
    const float v = fmaf(ga, (x[o + p] - mu) * is, be);
    y[o + p] = ELU ? elu1(v) : (relu ? fmaxf(v, 0.f) : v);
  }
}

// dx = gamma*invstd*(g - dbeta/n - xhat*dgamma/n)
template <bool ELU>
__global__ void __launch_bounds__(256)
    bn_bwd_apply_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                        const float* __restrict__ mean, const float* __restrict__ invstd,
                        const float* __restrict__ gamma, const float* __restrict__ beta,
                        const float* __restrict__ dgamma, const float* __restrict__ dbeta, int C,
                        int P, int relu, float inv_n, float* __restrict__ dx) {
  const int c = blockIdx.y, b = blockIdx.z;
  const float is = invstd[c], ga = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f, mu = mean[c];
  const float k0 = dbeta[c] * inv_n, k1 = dgamma[c] * inv_n;
  const size_t o = (static_cast<size_t>(b) * C + c) * P;
  for (int p = blockIdx.x * 1024 + threadIdx.x; p < min(P, (static_cast<int>(blockIdx.x) + 1) * 1024);
       p += 256) {
    const float xh = (x[o + p] - mu) * is;
    float g = dy[o + p];
    if (ELU) g *= elu_grad(fmaf(ga, xh, be));
    else if (relu && !(fmaf(ga, xh, be) > 0.f)) g = 0.f;
    dx[o + p] = ga * is * (g - k0 - xh * k1);
  }
}

// ---- instance normalisation (nn.InstanceNorm1d/2d, affine, no running statistics) -----------------
// Row r = b*C + c of z [B,C,P] is normalised by its own biased statistics: y = act(gamma_c * (z -
// mean_r) * invstd_r + beta_c). The row is staged on chip once; the statistics are exact two-pass
// (mean, then sum (z - mean)^2) with fp64 accumulation, every thread summing its strided elements in
// ascending order and the partial sums combined by a fixed butterfly / warp order: bit-reproducible.
// A constant row gives var = 0, z - mean = 0 and y = act(beta) exactly. The output pass can fold the
// k-copy mean (copy j of point n at j*N + n, summed (a+b)+c in fp32 and scaled like kcopy_mean_kernel)
// or the max over consecutive groups of K (after the activation, fmaxf like the rowmax kernels).
constexpr int IN_THREADS = 256;
constexpr int IN_WARP_ROW_MAX = 1024;      // rows up to this length: a warp per row, 8 rows per CTA
constexpr int IN_ROW_SMEM_MAX = 16384;     // longer rows up to this length: a CTA per row, staged
                                           // in 64 KB of shared memory; beyond it z is read again

__device__ __forceinline__ double in_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);   // same bits in all lanes
  return v;
}

// thread t of nt writes its share of the output row o from the row s (shared or global memory)
template <int ACT, int RED>
__device__ __forceinline__ void in_write_row(const float* s, int P, int k, float mu, float is, float ga,
                                             float be, float* o, int t, int nt) {
  if constexpr (RED == SONET_REDUCE_NONE) {
    for (int p = t; p < P; p += nt) o[p] = act_fn<ACT>(fmaf(ga, (s[p] - mu) * is, be));
  } else if constexpr (RED == SONET_REDUCE_KCOPY_MEAN) {
    const int N = P / k;
    const float w = (k == 2) ? 0.5f : (k == 3 ? (1.0f / 3.0f) : __fdiv_rn(1.0f, (float)k));
    for (int n = t; n < N; n += nt) {
      float acc = act_fn<ACT>(fmaf(ga, (s[n] - mu) * is, be));
      for (int j = 1; j < k; ++j)
        acc = __fadd_rn(acc, act_fn<ACT>(fmaf(ga, (s[j * N + n] - mu) * is, be)));
      o[n] = __fmul_rn(w, acc);
    }
  } else {
    const int G = P / k;
    for (int g = t; g < G; g += nt) {
      const float* q = s + static_cast<size_t>(g) * k;
      float m = act_fn<ACT>(fmaf(ga, (q[0] - mu) * is, be));
      for (int j = 1; j < k; ++j) m = fmaxf(m, act_fn<ACT>(fmaf(ga, (q[j] - mu) * is, be)));
      o[g] = m;
    }
  }
}

__device__ __forceinline__ long long in_out_len(int P, int k, int red) {
  return red == SONET_REDUCE_NONE ? P : P / k;
}

// rows with P <= IN_WARP_ROW_MAX: warp w of the CTA owns row 8*blockIdx.x + w, staged in srow[w]
template <int ACT, int RED>
__global__ void __launch_bounds__(IN_THREADS)
    instance_norm_warp_kernel(const float* z, const float* __restrict__ gamma,
                              const float* __restrict__ beta, long long R, int C, int P, float eps,
                              int k, float* out, float* __restrict__ save_mean,
                              float* __restrict__ save_invstd) {
  extern __shared__ float in_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r = static_cast<long long>(blockIdx.x) * (IN_THREADS / 32) + warp;
  if (r >= R) return;                                   // warp-uniform; no CTA barrier below
  float* s = in_smem + static_cast<size_t>(warp) * P;
  const float* zr = z + r * P;
  double a = 0.0;
  for (int p = lane; p < P; p += 32) {
    const float v = zr[p];
    s[p] = v;
    a += v;
  }
  const double mean = in_warp_sum(a) / P;
  double q = 0.0;
  for (int p = lane; p < P; p += 32) {                  // the lane's own elements: no sync needed
    const double d = static_cast<double>(s[p]) - mean;
    q = fma(d, d, q);
  }
  const double var = in_warp_sum(q) / P;
  const float mu = static_cast<float>(mean);
  const float is = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  const int c = static_cast<int>(r % C);
  if (lane == 0 && save_mean) {
    save_mean[r] = mu;
    save_invstd[r] = is;
  }
  __syncwarp();
  in_write_row<ACT, RED>(s, P, k, mu, is, gamma ? gamma[c] : 1.f, beta ? beta[c] : 0.f,
                         out + r * in_out_len(P, k, RED), lane, 32);
}

__device__ __forceinline__ double in_block_sum(double v, double* red) {
  v = in_warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int w = 0; w < IN_THREADS / 32; ++w) s += red[w];
  __syncthreads();                                      // red is reused by the next sum
  return s;
}

// longer rows: CTA blockIdx.x owns row r; STAGED keeps it in shared memory, else z is re-read
template <int ACT, int RED, bool STAGED>
__global__ void __launch_bounds__(IN_THREADS)
    instance_norm_row_kernel(const float* z, const float* __restrict__ gamma,
                             const float* __restrict__ beta, int C, int P, float eps, int k,
                             float* out, float* __restrict__ save_mean,
                             float* __restrict__ save_invstd) {
  extern __shared__ float in_smem[];
  __shared__ double red[IN_THREADS / 32];
  const long long r = blockIdx.x;
  const float* zr = z + r * P;
  double a = 0.0;
  for (int p = threadIdx.x; p < P; p += IN_THREADS) {
    const float v = zr[p];
    if (STAGED) in_smem[p] = v;
    a += v;
  }
  const double mean = in_block_sum(a, red) / P;
  double q = 0.0;
  for (int p = threadIdx.x; p < P; p += IN_THREADS) {
    const double d = static_cast<double>(STAGED ? in_smem[p] : zr[p]) - mean;
    q = fma(d, d, q);
  }
  const double var = in_block_sum(q, red) / P;          // its barriers also publish in_smem
  const float mu = static_cast<float>(mean);
  const float is = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  const int c = static_cast<int>(r % C);
  if (threadIdx.x == 0 && save_mean) {
    save_mean[r] = mu;
    save_invstd[r] = is;
  }
  // without a reduction out may alias z: each element is read and written by the same thread,
  // after every thread's statistics reads (the barriers above)
  in_write_row<ACT, RED>(STAGED ? in_smem : zr, P, k, mu, is, gamma ? gamma[c] : 1.f,
                         beta ? beta[c] : 0.f, out + r * in_out_len(P, k, RED), threadIdx.x,
                         IN_THREADS);
}

template <int ACT, int RED>
static void launch_instance_norm(const float* z, const float* gamma, const float* beta, long long R,
                                 int C, int P, float eps, int k, float* out, float* save_mean,
                                 float* save_invstd, cudaStream_t st) {
  if (P <= IN_WARP_ROW_MAX) {
    const int rows = IN_THREADS / 32;
    instance_norm_warp_kernel<ACT, RED>
        <<<static_cast<unsigned>((R + rows - 1) / rows), IN_THREADS, sizeof(float) * rows * P, st>>>(
            z, gamma, beta, R, C, P, eps, k, out, save_mean, save_invstd);
  } else if (P <= IN_ROW_SMEM_MAX) {
    const int smem = static_cast<int>(sizeof(float)) * P;
    cudaFuncSetAttribute(instance_norm_row_kernel<ACT, RED, true>,
                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    instance_norm_row_kernel<ACT, RED, true><<<static_cast<unsigned>(R), IN_THREADS, smem, st>>>(
        z, gamma, beta, C, P, eps, k, out, save_mean, save_invstd);
  } else {
    instance_norm_row_kernel<ACT, RED, false><<<static_cast<unsigned>(R), IN_THREADS, 0, st>>>(
        z, gamma, beta, C, P, eps, k, out, save_mean, save_invstd);
  }
}

template <int ACT>
static void launch_instance_norm_red(int reduce, const float* z, const float* gamma,
                                     const float* beta, long long R, int C, int P, float eps, int k,
                                     float* out, float* save_mean, float* save_invstd,
                                     cudaStream_t st) {
  if (reduce == SONET_REDUCE_KCOPY_MEAN)
    launch_instance_norm<ACT, SONET_REDUCE_KCOPY_MEAN>(z, gamma, beta, R, C, P, eps, k, out, save_mean,
                                                       save_invstd, st);
  else if (reduce == SONET_REDUCE_GROUP_MAX)
    launch_instance_norm<ACT, SONET_REDUCE_GROUP_MAX>(z, gamma, beta, R, C, P, eps, k, out, save_mean,
                                                      save_invstd, st);
  else
    launch_instance_norm<ACT, SONET_REDUCE_NONE>(z, gamma, beta, R, C, P, eps, k, out, save_mean,
                                                 save_invstd, st);
}

// Where row r = b*C + c of a launch over x lies and how long it is, from the extent argument
// `ext` of the kernel. Dense x [B,C,P]: ext = P, row r at r*P, P long. Ragged x [C, ld] (a [1,C,L]
// layer output of a ragged batch): ext = RaggedCols, cloud b owns the columns cols[b] .. cols[b+1]
// (clamped into [0, ld] like common.cuh's ragged_range), so row (b, c) starts at c*ld + cols[b]. The
// ragged record launch runs all three record kernels over every row; each takes the rows of its own
// length class, the dense launch's choice at P = the row's length.
struct RaggedCols {
  int C;
  long long ld;
  const long long* cols;
};
template <class Ext> constexpr bool kRaggedExt = !std::is_same<Ext, int>::value;
__device__ __forceinline__ long long row_start(int P, long long r) { return r * P; }
__device__ __forceinline__ int row_len(int P, long long) { return P; }
__device__ __forceinline__ void row_range(const RaggedCols& e, long long r, long long& lo,
                                          long long& hi) {
  ragged_range(e.cols, static_cast<int>(r / e.C), e.ld, lo, hi);
}
__device__ __forceinline__ long long row_start(const RaggedCols& e, long long r) {
  long long lo, hi;
  row_range(e, r, lo, hi);
  return (r % e.C) * e.ld + lo;
}
__device__ __forceinline__ int row_len(const RaggedCols& e, long long r) {
  long long lo, hi;
  row_range(e, r, lo, hi);
  return static_cast<int>(hi - lo);
}

// grad_data[b,c,idx[b,c,k]] += grad_out[b,c,k], k ascending, one thread per (b,c) row, idx clamped
// into the row. ext: N (grad_data [B,C,N]) or RaggedCols (grad [C, ld], row_start's layout)
template <class Ext = int>
__global__ void __launch_bounds__(128)
    index_max_backward_kernel(const float* __restrict__ grad_out, const int32_t* __restrict__ idx,
                              long long rows, Ext ext, int K, float* __restrict__ grad_data) {
  const long long r = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int N = row_len(ext, r);
  if constexpr (kRaggedExt<Ext>) {
    if (N < 1) return;
  }
  float* g = grad_data + row_start(ext, r);
  const float* go = grad_out + r * K;
  const int32_t* ix = idx + r * K;
  for (int k = 0; k < K; ++k) {
    const int n = min(max(ix[k], 0), N - 1);
    g[n] += go[k];
  }
}

// ---- device-side weight packing for the wgmma layer ---------------------------------------------
__global__ void __launch_bounds__(256)
    absmax_kernel(const float* __restrict__ w, long long n, unsigned* __restrict__ out_bits) {
  float m = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    m = fmaxf(m, fabsf(w[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out_bits, __float_as_uint(m));   // non-negative floats
}
// The pre-scale of a GRADIENT operand with max |g| = absmax (NaN elements do not count): tc::pow2_scale,
// except that an infinite max gives NaN. The saturating fp16 split would turn an infinite gradient
// into +-131008 and its results finite; a NaN scale makes them non-finite instead. Weight packs keep
// pow2_scale's 1: an infinite weight propagates by itself (hi = inf, lo = NaN).
__device__ inline float grad_scale(float absmax) {
  return isinf(absmax) ? __int_as_float(0x7fffffff) : tc::pow2_scale(absmax);
}
// scale2[0] = the power-of-two pre-scale of the tensor (tc::pow2_scale, or grad_scale when grad),
// scale2[1] = 1/scale
__global__ void scale_from_absmax_kernel(const unsigned* __restrict__ bits, int grad,
                                         float* __restrict__ scale2) {
  const float m = __uint_as_float(*bits);
  const float sc = grad ? grad_scale(m) : tc::pow2_scale(m);
  scale2[0] = sc;
  scale2[1] = 1.f / sc;
}
// Packs the logical matrix Wl [N][K] times scale2[0] into the generic layer's blob (tc::wblob) with
// kch K chunks, zero-padded. Wl[n][k] = src[n * sn + (k / kp) * sb + (k % kp) * sk]:
//   W [N][K]:                     sn = K, sk = 1, kp = K, sb = 0
//   W^T, of W [K][N]:             sn = 1, sk = N, kp = K, sb = 0
//   x [B][N][P] with k = (b, p):  sn = P, sk = 1, kp = P, sb = N * P
// Consecutive threads take consecutive k of one row n: the reads are coalesced unless sk > 1.
// NPROD = 1 (the one-product wgrad) writes the hi images only, the bytes the GEMM then reads: half
// the stores, in the same layout.
template <int NPROD>
__global__ void __launch_bounds__(256)
    tc_pack_device_kernel(const float* __restrict__ src, int N, int K, long long sn, long long sk,
                          int kp, long long sb, const float* __restrict__ scale2,
                          unsigned char* __restrict__ blob, int kch) {
  const int kext = kch * tc::wblob::KCH;
  const long long total = static_cast<long long>(tc::wblob::npad(N)) * kext;
  const float sc = scale2[0];
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(t / kext), k = static_cast<int>(t - static_cast<long long>(n) * kext);
    float w = 0.f;
    if (n < N && k < K) w = src[n * sn + (k / kp) * sb + (k % kp) * sk] * sc;
    long long hi, lo;
    tc::wblob::elem_off(N, kch, n, k, hi, lo);
    if (NPROD == 3)
      tc::put_weight(blob + hi, blob + lo, w);
    else   // put_weight's hi half
      *reinterpret_cast<__half*>(blob + hi) = __float2half_rn(w);
  }
}
static void launch_tc_pack(const float* src, int N, int K, long long sn, long long sk, int kp,
                           long long sb, const float* scale2, void* blob, int kch, cudaStream_t st,
                           int nprod = 3) {
  const long long total = static_cast<long long>(tc::wblob::npad(N)) * kch * tc::wblob::KCH;
  const unsigned grid = static_cast<unsigned>(std::min<long long>((total + 255) / 256, 16384));
  unsigned char* b = static_cast<unsigned char*>(blob);
  if (nprod == 1)
    tc_pack_device_kernel<1><<<grid, 256, 0, st>>>(src, N, K, sn, sk, kp, sb, scale2, b, kch);
  else
    tc_pack_device_kernel<3><<<grid, 256, 0, st>>>(src, N, K, sn, sk, kp, sb, scale2, b, kch);
}

// absmax without atomics: CTA b writes the max of its grid-stride share to partial[b], then one
// thread takes the max of the partials in ascending order and forms the scale like
// scale_from_absmax_kernel (the max of a set is order-free; this keeps the entry graph-capturable
// without a memset and free of atomics)
constexpr int ABSMAX_SLOTS = 256;
__global__ void __launch_bounds__(256)
    absmax_partial_kernel(const float* __restrict__ w, long long n, float* __restrict__ partial) {
  float m = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    m = fmaxf(m, fabsf(w[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float wm[8];
  if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) m = fmaxf(m, wm[k]);
    partial[blockIdx.x] = m;
  }
}
__global__ void scale_from_partials_kernel(const float* __restrict__ partial, int nb,
                                           float* __restrict__ scale2) {
  float m = 0.f;
  for (int b = 0; b < nb; ++b) m = fmaxf(m, partial[b]);
  const float sc = tc::pow2_scale(m);
  scale2[0] = sc;
  scale2[1] = 1.f / sc;
}

// ---- wgrad helpers ------------------------------------------------------------------------------------
// Per-channel power-of-two pre-scale of dy [B][C][P]: cscale[c] = s_c with max_{b,p} |s_c dy[b,c,p]|
// in [256,512) (grad_scale: 1 for an all-zero channel, NaN for one holding +-inf), cscale[C + c] = 1/s_c. Gradients of one
// layer span many decades between channels; with ONE scale per tensor the small channels' values
// would fall into fp16's subnormal range and lose their relative precision (each row of dW is its
// own parameter's gradient). One CTA per channel.
__global__ void __launch_bounds__(256)
    channel_scale_kernel(const float* __restrict__ t, int B, int C, int P, float* __restrict__ cscale) {
  const int c = blockIdx.x;
  float m = 0.f;
  for (int b = 0; b < B; ++b) {
    const float* r = t + (static_cast<size_t>(b) * C + c) * P;
    for (int p = threadIdx.x; p < P; p += blockDim.x) m = fmaxf(m, fabsf(r[p]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float wm[8];
  if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) m = fmaxf(m, wm[w]);
    const float sc = grad_scale(m);
    cscale[c] = sc;
    cscale[C + c] = 1.f / sc;
  }
}
// dyT[k = b*P + p][co] = dy[b][co][p] * cscale[co] (powers of two): the "activation" operand of the
// wgrad GEMM in the [K][rows] layout the generic wgmma layer consumes. 32x32 smem tiles.
__global__ void __launch_bounds__(256)
    transpose_scale_kernel(const float* __restrict__ dy, int C, int P, const float* __restrict__ cscale,
                           float* __restrict__ dyT) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, p = p0 + tx;
    tile[i][tx] = (c < C && p < P) ? dy[(static_cast<size_t>(b) * C + c) * P + p] * cscale[c] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int p = p0 + i, c = c0 + tx;
    if (p < P && c < C) dyT[(static_cast<size_t>(b) * P + p) * C + c] = tile[tx][i];
  }
}
// dWT [Cin][Cout] = the raw GEMM sum * (1/s_x) * (1/s_co): undoes x's pre-scale and each dy channel's.
// Both factors are powers of two, so the fp64 product is exact and the result is rounded once. In
// fp32, sum / s_x (= s_co dW) overflows where dW > FLT_MAX / s_co although dW itself is finite.
__global__ void __launch_bounds__(256)
    col_unscale_kernel(float* __restrict__ dWT, long long n, int Cout, const float* __restrict__ inv_x,
                       const float* __restrict__ inv_c) {
  const double ix = static_cast<double>(*inv_x);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dWT[i] = static_cast<float>(static_cast<double>(dWT[i]) * ix * static_cast<double>(inv_c[i % Cout]));
}
// the GEMM's epilogue scale in the wgrad: 1, the unscale is col_unscale_kernel's
__device__ const float kUnitScale = 1.f;

// ---- train-mode BatchNorm: per-cloud records ------------------------------------------------------
// Row r = b*C + c of x [B,C,P] gets one fp64 record whose value depends on that row alone: the row's
// elements are summed in a fixed order chosen from P only (never from B, C or the SM count), so the
// records of a cloud are the same bits whichever batch or data-parallel shard it lands in.
// Forward: {pivot = x[r,0], sum d, sum d*d}, d = x - pivot. Backward: {sum g, sum g*xhat}, g = dy *
// [gamma*xhat + beta > 0] for ReLU, dy * elu_grad(gamma*xhat + beta) for ELU, dy for none. Every
// term is accumulated in fp64.
//
// The forward sums are shifted by a pivot drawn from the channel. var = E[d^2] - E[d]^2 then cancels
// only by 1 + (mean - pivot)^2 / var, a few units for any such pivot, where E[x^2] - mean^2 would
// cancel by (mean/std)^2: with fp32 sums that is a relative error of ~(mean/std)^2 * 2^-24 in var,
// 1e-2 at mean/std = 1e3 (channels behind a large bias, near-dead inputs). d is exact in fp64, d*d
// too, and a constant channel gives var = 0.
constexpr int BNC_WARP_P = 1024;           // rows up to this length: a warp per row, else a CTA

template <bool BWD, int ACT>
struct BncRow {
  const float *xr, *gr;
  float mu, is, ga, be;
  double pivot;
  template <class Ext>
  __device__ __forceinline__ BncRow(const float* x, const float* dy, const float* mean,
                                    const float* invstd, const float* gamma, const float* beta,
                                    long long r, int C, Ext ext) {
    const int c = static_cast<int>(r % C);
    xr = x + row_start(ext, r);
    gr = BWD ? dy + row_start(ext, r) : nullptr;
    mu = BWD ? mean[c] : 0.f;
    is = BWD ? invstd[c] : 1.f;
    ga = BWD && gamma ? gamma[c] : 1.f;
    be = BWD && beta ? beta[c] : 0.f;
    pivot = BWD ? 0.0 : static_cast<double>(xr[0]);
  }
  __device__ __forceinline__ void add(int p, double& a0, double& a1) const {
    if (BWD) {
      const float xh = (xr[p] - mu) * is;
      float g = gr[p];
      if (ACT == SONET_ACT_ELU) g *= elu_grad(fmaf(ga, xh, be));
      else if (ACT == SONET_ACT_RELU && !(fmaf(ga, xh, be) > 0.f)) g = 0.f;
      a0 += static_cast<double>(g);
      a1 = fma(static_cast<double>(g), static_cast<double>(xh), a1);
    } else {
      const double d = static_cast<double>(xr[p]) - pivot;
      a0 += d;
      a1 = fma(d, d, a1);
    }
  }
  __device__ __forceinline__ void store(double* rec, long long r, double a0, double a1) const {
    if (BWD) {
      rec[r * SONET_BN_REC_BWD] = a0;
      rec[r * SONET_BN_REC_BWD + 1] = a1;
    } else {
      rec[r * SONET_BN_REC_FWD] = pivot;
      rec[r * SONET_BN_REC_FWD + 1] = a0;
      rec[r * SONET_BN_REC_FWD + 2] = a1;
    }
  }
};

// the point kernel's dense rows are one value long whatever its P argument says
__device__ __forceinline__ int point_ext(int) { return 1; }
__device__ __forceinline__ const RaggedCols& point_ext(const RaggedCols& e) { return e; }

// P == 1 (MyLinear's [B,C,1] view): a thread per row, consecutive threads on consecutive channels.
// A ragged row of no columns (refused by the callers) gets the record of nothing, all zeros.
template <bool BWD, int ACT, class Ext = int>
__global__ void __launch_bounds__(256)
    bn_cloud_point_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                          const float* __restrict__ mean, const float* __restrict__ invstd,
                          const float* __restrict__ gamma, const float* __restrict__ beta, long long R,
                          int C, Ext ext, double* __restrict__ rec) {
  const long long r = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= R) return;
  if constexpr (kRaggedExt<Ext>) {
    const int P = row_len(ext, r);
    if (P > 1) return;
    if (P == 0) {
      for (int i = 0; i < (BWD ? SONET_BN_REC_BWD : SONET_BN_REC_FWD); ++i)
        rec[r * (BWD ? SONET_BN_REC_BWD : SONET_BN_REC_FWD) + i] = 0.0;
      return;
    }
  }
  const BncRow<BWD, ACT> row(x, dy, mean, invstd, gamma, beta, r, C, point_ext(ext));
  double a0 = 0.0, a1 = 0.0;
  row.add(0, a0, a1);
  row.store(rec, r, a0, a1);
}

// 1 < P <= BNC_WARP_P: warp w of the CTA owns row 8*blockIdx.x + w; lanes take p = lane, lane+32, ...
template <bool BWD, int ACT, class Ext = int>
__global__ void __launch_bounds__(256)
    bn_cloud_warp_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                         const float* __restrict__ mean, const float* __restrict__ invstd,
                         const float* __restrict__ gamma, const float* __restrict__ beta, long long R,
                         int C, Ext ext, double* __restrict__ rec) {
  const long long r = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= R) return;                                   // warp-uniform
  const int P = row_len(ext, r);
  if constexpr (kRaggedExt<Ext>) {
    if (P <= 1 || P > BNC_WARP_P) return;               // warp-uniform
  }
  const BncRow<BWD, ACT> row(x, dy, mean, invstd, gamma, beta, r, C, ext);
  double a0 = 0.0, a1 = 0.0;
  for (int p = lane; p < P; p += 32) row.add(p, a0, a1);
  a0 = in_warp_sum(a0);
  a1 = in_warp_sum(a1);
  if (lane == 0) row.store(rec, r, a0, a1);
}

// P > BNC_WARP_P: CTA blockIdx.x owns row r; thread t takes p = t, t+256, ..., then the warp
// butterfly and the 8 warp sums in ascending order
template <bool BWD, int ACT, class Ext = int>
__global__ void __launch_bounds__(256)
    bn_cloud_cta_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                        const float* __restrict__ mean, const float* __restrict__ invstd,
                        const float* __restrict__ gamma, const float* __restrict__ beta, int C, Ext ext,
                        double* __restrict__ rec) {
  static_assert(IN_THREADS == 256, "in_block_sum sums 8 warps");
  __shared__ double red[IN_THREADS / 32];
  const long long r = blockIdx.x;
  if constexpr (kRaggedExt<Ext>) {
    if (row_len(ext, r) <= BNC_WARP_P) return;          // CTA-uniform, before any barrier
  }
  const BncRow<BWD, ACT> row(x, dy, mean, invstd, gamma, beta, r, C, ext);
  const int P = row_len(ext, r);
  double a0 = 0.0, a1 = 0.0;
  for (int p = threadIdx.x; p < P; p += IN_THREADS) row.add(p, a0, a1);
  a0 = in_block_sum(a0, red);
  a1 = in_block_sum(a1, red);
  if (threadIdx.x == 0) row.store(rec, r, a0, a1);
}

template <bool BWD, int ACT>
static void launch_bn_cloud(const float* x, const float* dy, const float* mean, const float* invstd,
                            const float* gamma, const float* beta, long long R, int C, int P,
                            double* rec, cudaStream_t st) {
  if (P == 1)
    bn_cloud_point_kernel<BWD, ACT><<<static_cast<unsigned>((R + 255) / 256), 256, 0, st>>>(
        x, dy, mean, invstd, gamma, beta, R, C, P, rec);
  else if (P <= BNC_WARP_P)
    bn_cloud_warp_kernel<BWD, ACT><<<static_cast<unsigned>((R + 7) / 8), 256, 0, st>>>(
        x, dy, mean, invstd, gamma, beta, R, C, P, rec);
  else
    bn_cloud_cta_kernel<BWD, ACT><<<static_cast<unsigned>(R), IN_THREADS, 0, st>>>(
        x, dy, mean, invstd, gamma, beta, C, P, rec);
}

// the ragged rows have every length: all three kernels run, each on the rows of its class
template <bool BWD, int ACT>
static void launch_bn_cloud_ragged(const float* x, const float* dy, const float* mean,
                                   const float* invstd, const float* gamma, const float* beta, int B,
                                   int C, long long ld, const long long* cols, double* rec,
                                   cudaStream_t st) {
  const long long R = static_cast<long long>(B) * C;
  const RaggedCols ext{C, ld, cols};
  bn_cloud_point_kernel<BWD, ACT><<<static_cast<unsigned>((R + 255) / 256), 256, 0, st>>>(
      x, dy, mean, invstd, gamma, beta, R, C, ext, rec);
  bn_cloud_warp_kernel<BWD, ACT><<<static_cast<unsigned>((R + 7) / 8), 256, 0, st>>>(
      x, dy, mean, invstd, gamma, beta, R, C, ext, rec);
  bn_cloud_cta_kernel<BWD, ACT><<<static_cast<unsigned>(R), IN_THREADS, 0, st>>>(
      x, dy, mean, invstd, gamma, beta, C, ext, rec);
}

// How many values record b of a fold stands for, and n, their total. Dense: P each, Bg*P in all.
// Ragged: cloud b's own column count cols[b+1] - cols[b] (clamped into [0, L]), L in all.
struct DenseCounts {
  int P;
  __device__ __forceinline__ double count(int) const { return static_cast<double>(P); }
  __device__ __forceinline__ double total(int Bg) const { return static_cast<double>(Bg) * P; }
};
struct RaggedCounts {
  const long long* cols;
  long long L;
  __device__ __forceinline__ double count(int b) const {
    long long lo, hi;
    ragged_range(cols, b, L, lo, hi);
    return static_cast<double>(hi - lo);
  }
  __device__ __forceinline__ double total(int) const { return static_cast<double>(L); }
};

// the forward records of Bg clouds, ascending, onto cloud 0's pivot p; then mean = p + E[x - p] and
// the biased var = E[(x - p)^2] - E[x - p]^2 (F.batch_norm normalises with it). Shifting record b of
// n_b values by s = p_b - p (exact: both are fp32 values) is the identity
// sum (x - p) = sum d_b + n_b s, sum (x - p)^2 = sum d_b^2 + 2 s sum d_b + n_b s^2.
template <class Counts>
__global__ void bn_sync_stats_kernel(const double* __restrict__ rec, int Bg, int C, Counts cnt,
                                     float eps, float* __restrict__ mean, float* __restrict__ var,
                                     float* __restrict__ invstd) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double p = rec[static_cast<size_t>(c) * SONET_BN_REC_FWD];
  double s1 = 0.0, s2 = 0.0;
  for (int b = 0; b < Bg; ++b) {
    const double nb = cnt.count(b);
    const double* q = rec + (static_cast<size_t>(b) * C + c) * SONET_BN_REC_FWD;
    const double s = q[0] - p;
    s1 += q[1] + nb * s;
    s2 += q[2] + 2.0 * s * q[1] + nb * s * s;
  }
  const double n = cnt.total(Bg);
  const double md = s1 / n;                                        // mean - pivot
  double v = s2 / n - md * md;
  if (v < 0.0) v = 0.0;
  mean[c] = static_cast<float>(p + md);
  var[c] = static_cast<float>(v);
  invstd[c] = static_cast<float>(1.0 / sqrt(v + static_cast<double>(eps)));
}

__global__ void bn_sync_bwd_final_kernel(const double* __restrict__ rec, int Bg, int C,
                                         float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s0 = 0.0, s1 = 0.0;
  for (int b = 0; b < Bg; ++b) {
    const double* q = rec + (static_cast<size_t>(b) * C + c) * SONET_BN_REC_BWD;
    s0 += q[0];
    s1 += q[1];
  }
  dbeta[c] = static_cast<float>(s0);
  dgamma[c] = static_cast<float>(s1);
}
}  // namespace sonet

extern "C" int sonet_bn_cloud_partials_f32(const float* x, const float* dy, const float* mean,
                                           const float* invstd, const float* gamma, const float* beta,
                                           int B, int C, int P, int act, int backward, double* rec,
                                           sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE_ACT(act, "bn_cloud_partials");
  SONET_REQUIRE(B >= 1 && C >= 1 && P >= 1 && B <= 65535 && C <= 65535,
                "bn_cloud_partials: bad dims B=%d C=%d P=%d", B, C, P);
  SONET_REQUIRE(x && rec && (!backward || (dy && mean && invstd)), "bn_cloud_partials: null pointer");
  const long long R = static_cast<long long>(B) * C;
  SONET_REQUIRE(R < (1LL << 31), "bn_cloud_partials: too many rows B*C=%lld", R);
  cudaStream_t st = as_stream(stream);
  if (!backward)
    launch_bn_cloud<false, SONET_ACT_NONE>(x, nullptr, nullptr, nullptr, nullptr, nullptr, R, C, P, rec, st);
  else if (act == SONET_ACT_ELU)
    launch_bn_cloud<true, SONET_ACT_ELU>(x, dy, mean, invstd, gamma, beta, R, C, P, rec, st);
  else if (act == SONET_ACT_RELU)
    launch_bn_cloud<true, SONET_ACT_RELU>(x, dy, mean, invstd, gamma, beta, R, C, P, rec, st);
  else
    launch_bn_cloud<true, SONET_ACT_NONE>(x, dy, mean, invstd, gamma, beta, R, C, P, rec, st);
  return check_launch("bn_cloud_partials");
}

extern "C" int sonet_bn_sync_forward_f32(const double* rec, const float* x, const float* gamma,
                                         const float* beta, int Bg, int B, int C, int P, float eps,
                                         int act, float* y, float* mean, float* var, float* invstd,
                                         sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE_ACT(act, "bn_sync_forward");
  SONET_REQUIRE(B >= 1 && C >= 1 && P >= 1 && Bg >= B && Bg <= 65535 && C <= 65535,
                "bn_sync_forward: bad dims Bg=%d B=%d C=%d P=%d", Bg, B, C, P);
  SONET_REQUIRE(rec && x && y && mean && var && invstd, "bn_sync_forward: null pointer");
  cudaStream_t st = as_stream(stream);
  bn_sync_stats_kernel<<<(C + 127) / 128, 128, 0, st>>>(rec, Bg, C, DenseCounts{P}, eps, mean, var,
                                                     invstd);
  const dim3 grid((P + 1023) / 1024, C, B);
  if (act == SONET_ACT_ELU)
    bn_apply_kernel<true><<<grid, 256, 0, st>>>(x, mean, invstd, gamma, beta, C, P, 0, y);
  else
    bn_apply_kernel<false><<<grid, 256, 0, st>>>(x, mean, invstd, gamma, beta, C, P, act, y);
  return check_launch("bn_sync_forward");
}

extern "C" int sonet_bn_sync_backward_f32(const double* rec, const float* dy, const float* x,
                                          const float* mean, const float* invstd, const float* gamma,
                                          const float* beta, int Bg, int B, int C, int P, int act,
                                          float* dx, float* dgamma, float* dbeta, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE_ACT(act, "bn_sync_backward");
  SONET_REQUIRE(B >= 1 && C >= 1 && P >= 1 && Bg >= B && Bg <= 65535 && C <= 65535,
                "bn_sync_backward: bad dims Bg=%d B=%d C=%d P=%d", Bg, B, C, P);
  SONET_REQUIRE(rec && dy && x && mean && invstd && dx && dgamma && dbeta,
                "bn_sync_backward: null pointer");
  cudaStream_t st = as_stream(stream);
  bn_sync_bwd_final_kernel<<<(C + 127) / 128, 128, 0, st>>>(rec, Bg, C, dgamma, dbeta);
  const dim3 grid((P + 1023) / 1024, C, B);
  const float inv_n = static_cast<float>(1.0 / (static_cast<double>(Bg) * P));
  if (act == SONET_ACT_ELU)
    bn_bwd_apply_kernel<true><<<grid, 256, 0, st>>>(dy, x, mean, invstd, gamma, beta, dgamma, dbeta, C, P,
                                                    0, inv_n, dx);
  else
    bn_bwd_apply_kernel<false><<<grid, 256, 0, st>>>(dy, x, mean, invstd, gamma, beta, dgamma, dbeta, C, P,
                                                     act, inv_n, dx);
  return check_launch("bn_sync_backward");
}

// ---- ragged batches: x [C, L], cloud b owning the columns cols[b] .. cols[b+1] ---------------------
static int bn_ragged_dims(const char* what, int B, int C, long long L) {
  using namespace sonet;
  SONET_REQUIRE(B >= 1 && C >= 1 && B <= 65535 && C <= 65535, "%s: bad dims B=%d C=%d", what, B, C);
  SONET_REQUIRE(L >= 1 && L < (1LL << 31), "%s: L=%lld columns outside [1, 2^31)", what, L);
  return SONET_OK;
}

extern "C" int sonet_bn_cloud_partials_ragged_f32(const float* x, const float* dy, const float* mean,
                                                  const float* invstd, const float* gamma,
                                                  const float* beta, int C, long long ld,
                                                  const long long* col_offsets, int B, int act,
                                                  int backward, double* rec, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE_ACT(act, "bn_cloud_partials_ragged");
  if (int rc = bn_ragged_dims("bn_cloud_partials_ragged", B, C, ld)) return rc;
  SONET_REQUIRE(x && col_offsets && rec && (!backward || (dy && mean && invstd)),
                "bn_cloud_partials_ragged: null pointer");
  cudaStream_t st = as_stream(stream);
  if (!backward)
    launch_bn_cloud_ragged<false, SONET_ACT_NONE>(x, nullptr, nullptr, nullptr, nullptr, nullptr, B, C,
                                                  ld, col_offsets, rec, st);
  else if (act == SONET_ACT_ELU)
    launch_bn_cloud_ragged<true, SONET_ACT_ELU>(x, dy, mean, invstd, gamma, beta, B, C, ld, col_offsets,
                                                rec, st);
  else if (act == SONET_ACT_RELU)
    launch_bn_cloud_ragged<true, SONET_ACT_RELU>(x, dy, mean, invstd, gamma, beta, B, C, ld, col_offsets,
                                                 rec, st);
  else
    launch_bn_cloud_ragged<true, SONET_ACT_NONE>(x, dy, mean, invstd, gamma, beta, B, C, ld, col_offsets,
                                                 rec, st);
  return check_launch("bn_cloud_partials_ragged");
}

extern "C" int sonet_bn_ragged_forward_f32(const double* rec, const long long* col_offsets, int B,
                                           const float* x, const float* gamma, const float* beta, int C,
                                           long long L, float eps, int act, float* y, float* mean,
                                           float* var, float* invstd, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE_ACT(act, "bn_ragged_forward");
  if (int rc = bn_ragged_dims("bn_ragged_forward", B, C, L)) return rc;
  SONET_REQUIRE(rec && col_offsets && x && y && mean && var && invstd, "bn_ragged_forward: null pointer");
  cudaStream_t st = as_stream(stream);
  bn_sync_stats_kernel<<<(C + 127) / 128, 128, 0, st>>>(rec, B, C, RaggedCounts{col_offsets, L}, eps,
                                                        mean, var, invstd);
  const int P = static_cast<int>(L);
  const dim3 grid((P + 1023) / 1024, C, 1);
  if (act == SONET_ACT_ELU)
    bn_apply_kernel<true><<<grid, 256, 0, st>>>(x, mean, invstd, gamma, beta, C, P, 0, y);
  else
    bn_apply_kernel<false><<<grid, 256, 0, st>>>(x, mean, invstd, gamma, beta, C, P, act, y);
  return check_launch("bn_ragged_forward");
}

extern "C" int sonet_bn_ragged_backward_f32(const double* rec, const long long* col_offsets, int B,
                                            const float* dy, const float* x, const float* mean,
                                            const float* invstd, const float* gamma, const float* beta,
                                            int C, long long L, int act, float* dx, float* dgamma,
                                            float* dbeta, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE_ACT(act, "bn_ragged_backward");
  if (int rc = bn_ragged_dims("bn_ragged_backward", B, C, L)) return rc;
  SONET_REQUIRE(rec && col_offsets && dy && x && mean && invstd && dx && dgamma && dbeta,
                "bn_ragged_backward: null pointer");
  cudaStream_t st = as_stream(stream);
  bn_sync_bwd_final_kernel<<<(C + 127) / 128, 128, 0, st>>>(rec, B, C, dgamma, dbeta);
  const int P = static_cast<int>(L);
  const dim3 grid((P + 1023) / 1024, C, 1);
  const float inv_n = static_cast<float>(1.0 / static_cast<double>(L));
  if (act == SONET_ACT_ELU)
    bn_bwd_apply_kernel<true><<<grid, 256, 0, st>>>(dy, x, mean, invstd, gamma, beta, dgamma, dbeta, C, P,
                                                    0, inv_n, dx);
  else
    bn_bwd_apply_kernel<false><<<grid, 256, 0, st>>>(dy, x, mean, invstd, gamma, beta, dgamma, dbeta, C, P,
                                                     act, inv_n, dx);
  return check_launch("bn_ragged_backward");
}

extern "C" int sonet_instance_norm_f32(const float* z, const float* gamma, const float* beta, int B,
                                       int C, int P, float eps, int act, int reduce, int k, float* out,
                                       float* save_mean, float* save_invstd, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE_ACT(act, "instance_norm");
  SONET_REQUIRE(reduce == SONET_REDUCE_NONE || reduce == SONET_REDUCE_KCOPY_MEAN ||
                    reduce == SONET_REDUCE_GROUP_MAX,
                "instance_norm: reduction code %d is not SONET_REDUCE_NONE (0), _KCOPY_MEAN (1) or "
                "_GROUP_MAX (2)", reduce);
  SONET_REQUIRE(B >= 1 && C >= 1, "instance_norm: bad dims B=%d C=%d", B, C);
  SONET_REQUIRE(P >= 2, "instance_norm: Expected more than 1 spatial element (got P=%d)", P);
  SONET_REQUIRE(reduce == SONET_REDUCE_NONE || (k >= 1 && P % k == 0),
                "instance_norm: P=%d is not divisible by the %s k=%d", P,
                reduce == SONET_REDUCE_KCOPY_MEAN ? "copy count" : "group size", k);
  SONET_REQUIRE(z && out, "instance_norm: null pointer");
  SONET_REQUIRE((save_mean == nullptr) == (save_invstd == nullptr),
                "instance_norm: save_mean and save_invstd are given together or not at all");
  SONET_REQUIRE(reduce == SONET_REDUCE_NONE || out != z, "instance_norm: a reduced output cannot alias z");
  const long long R = static_cast<long long>(B) * C;
  SONET_REQUIRE(R < (1LL << 31), "instance_norm: too many rows");
  cudaStream_t st = as_stream(stream);
  if (act == SONET_ACT_ELU)
    launch_instance_norm_red<SONET_ACT_ELU>(reduce, z, gamma, beta, R, C, P, eps, k, out, save_mean,
                                            save_invstd, st);
  else if (act == SONET_ACT_RELU)
    launch_instance_norm_red<SONET_ACT_RELU>(reduce, z, gamma, beta, R, C, P, eps, k, out, save_mean,
                                             save_invstd, st);
  else
    launch_instance_norm_red<SONET_ACT_NONE>(reduce, z, gamma, beta, R, C, P, eps, k, out, save_mean,
                                             save_invstd, st);
  return check_launch("instance_norm");
}

extern "C" int sonet_index_max_backward_f32(const float* grad_out, const int32_t* idx, int B, int C,
                                            int N, int K, float* grad_data, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 0 && N >= 1 && K >= 1, "index_max_backward: bad dims");
  const long long rows = static_cast<long long>(B) * C;
  if (rows == 0) return SONET_OK;
  SONET_REQUIRE(grad_out && idx && grad_data, "index_max_backward: null pointer");
  cudaStream_t st = as_stream(stream);
  cudaMemsetAsync(grad_data, 0, sizeof(float) * static_cast<size_t>(rows) * N, st);
  index_max_backward_kernel<<<static_cast<unsigned>((rows + 127) / 128), 128, 0, st>>>(
      grad_out, idx, rows, N, K, grad_data);
  return check_launch("index_max_backward");
}

extern "C" int sonet_index_max_ragged_backward_f32(const float* grad_out, const int32_t* idx,
                                                   const long long* col_offsets, int B, int C, int M,
                                                   long long ld, float* grad, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 1 && C >= 1 && M >= 1 && M <= 256 && B <= 65535 && C <= 65535,
                "index_max_ragged_backward: bad dims B=%d C=%d M=%d", B, C, M);
  SONET_REQUIRE(ld >= 1 && ld < (1LL << 31), "index_max_ragged_backward: ld=%lld outside [1, 2^31)", ld);
  SONET_REQUIRE(grad_out && idx && col_offsets && grad, "index_max_ragged_backward: null pointer");
  cudaStream_t st = as_stream(stream);
  const long long rows = static_cast<long long>(B) * C;
  cudaMemsetAsync(grad, 0, sizeof(float) * static_cast<size_t>(C) * ld, st);
  index_max_backward_kernel<<<static_cast<unsigned>((rows + 127) / 128), 128, 0, st>>>(
      grad_out, idx, rows, RaggedCols{C, ld, col_offsets}, M, grad);
  return check_launch("index_max_ragged_backward");
}

extern "C" long long sonet_pointwise_tc_blob_bytes(int Cout, int Cin);

extern "C" int sonet_pointwise_tc_pack_device(const float* W, int Cout, int Cin, int transpose,
                                              void* blob, float* scale2, unsigned* scratch_bits,
                                              sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(W && blob && scale2 && scratch_bits && Cout >= 1 && Cin >= 1,
                "pointwise_tc_pack_device: bad args");
  cudaStream_t st = as_stream(stream);
  const long long n = static_cast<long long>(Cout) * Cin;
  cudaMemsetAsync(scratch_bits, 0, sizeof(unsigned), st);
  absmax_kernel<<<static_cast<unsigned>(std::min<long long>((n + 255) / 256, 1024)), 256, 0, st>>>(
      W, n, scratch_bits);
  scale_from_absmax_kernel<<<1, 1, 0, st>>>(scratch_bits, 0, scale2);
  if (transpose)   // W^T [Cin][Cout]
    launch_tc_pack(W, Cin, Cout, 1, Cin, Cout, 0, scale2, blob, tc::wblob::kchunks(Cout), st);
  else
    launch_tc_pack(W, Cout, Cin, Cin, 1, Cin, 0, scale2, blob, tc::wblob::kchunks(Cin), st);
  return check_launch("pointwise_tc_pack_device");
}

// G matrices [G][Cout][Cin] on the device -> G consecutive blobs (sonet_pointwise_tc_blob_bytes each)
// with ONE power-of-two pre-scale, computed on the device: the same bytes and scale as the host's
// sonet_pointwise_tc_pack_groups. scratch: SONET_ABSMAX_SLOTS floats.
extern "C" int sonet_pointwise_tc_pack_groups_device(const float* W, int G, int Cout, int Cin, void* blob,
                                                     float* scale2, float* scratch,
                                                     sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(G >= 1 && Cout >= 1 && Cin >= 1, "pointwise_tc_pack_groups_device: bad dimension "
                "G=%d Cout=%d Cin=%d", G, Cout, Cin);
  SONET_REQUIRE(W && blob && scale2 && scratch, "pointwise_tc_pack_groups_device: null pointer");
  SONET_REQUIRE(aligned16(blob), "pointwise_tc_pack_groups_device: blob must be 16-byte aligned");
  static_assert(ABSMAX_SLOTS == SONET_ABSMAX_SLOTS, "scratch size of the header");
  cudaStream_t st = as_stream(stream);
  const long long per = static_cast<long long>(Cout) * Cin, n = per * G;
  const int nb = static_cast<int>(std::min<long long>((n + 255) / 256, ABSMAX_SLOTS));
  absmax_partial_kernel<<<nb, 256, 0, st>>>(W, n, scratch);
  scale_from_partials_kernel<<<1, 1, 0, st>>>(scratch, nb, scale2);
  const long long bytes = tc::wblob::bytes(Cout, Cin);
  for (int g = 0; g < G; ++g)
    launch_tc_pack(W + g * per, Cout, Cin, Cin, 1, Cin, 0, scale2, static_cast<unsigned char*>(blob) + g * bytes,
                   tc::wblob::kchunks(Cin), st);
  return check_launch("pointwise_tc_pack_groups_device");
}

// power-of-two pre-scale of a gradient operand on the device: scale2[0] = s with max|s*t| in [256,512)
// (grad_scale: NaN elements are ignored, 1 when all are zero, NaN when one is +-inf), scale2[1] = 1/s
extern "C" int sonet_absmax_scale_f32(const float* t, long long n, float* scale2, unsigned* scratch_bits,
                                      sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(t && scale2 && scratch_bits && n >= 1, "absmax_scale: bad args");
  cudaStream_t st = as_stream(stream);
  cudaMemsetAsync(scratch_bits, 0, sizeof(unsigned), st);
  absmax_kernel<<<static_cast<unsigned>(std::min<long long>((n + 255) / 256, 2048)), 256, 0, st>>>(
      t, n, scratch_bits);
  scale_from_absmax_kernel<<<1, 1, 0, st>>>(scratch_bits, 1, scale2);
  return check_launch("absmax_scale");
}

extern "C" int sonet_pointwise_tc_forward_dev(const float* x0, int C0, int B, int P, const void* blob,
                                              const float* inv_scale_dev, const float* act_scale_dev,
                                              const float* shift, int Cout, int relu, int splits,
                                              float* out, float* scratch, sonet_stream_t stream);
extern "C" int sonet_pointwise_tc_forward_dev_f16(const float* x0, int C0, int B, int P,
                                                  const void* blob, const float* inv_scale_dev,
                                                  const float* act_scale_dev, const float* shift,
                                                  int Cout, int relu, int splits, float* out,
                                                  float* scratch, sonet_stream_t stream);

// wgrad of a 1x1 convolution on wgmma: dW[co][ci] = sum_{b,p} dy[b,co,p] * x[b,ci,p].
// Written as the generic layer GEMM out[rows = co][n = ci] = sum_k A[k][co] * Wl[ci][k] with the
// contraction index k = (b, p): A = dy transposed to [K][Cout] (and pre-scaled: gradients are far
// below fp16's normal range), Wl = x packed as a weight blob, K split over CTAs with a
// deterministic reduce. Result: dWT [Cin][Cout] (the caller views it transposed).
// Scratch (device): dyT  Kpad*Cout floats, blob sonet_wgrad_blob_bytes(), part splits*Cin*Cout floats,
// small: sonet_wgrad_small_floats(Cout) floats.
extern "C" long long sonet_wgrad_small_floats(int Cout) { return 8 + 2LL * Cout; }
extern "C" long long sonet_wgrad_kpad(int B, int P, int splits) {
  const long long K = static_cast<long long>(B) * P;
  const long long q = 64LL * splits;
  return (K + q - 1) / q * q;
}
extern "C" long long sonet_wgrad_blob_bytes(int Cin, long long Kpad) {
  return sonet::tc::wblob::bytes(Cin, Kpad);
}
// nprod = 1: the one-product twin. dyT keeps fp32 (the generic kernel rounds its activation operand
// itself); x is packed as hi images only, into the same blob layout and size.
static int wgrad_tc(const float* dy, const float* x, int B, int Cout, int Cin, int P, int splits,
                    float* dyT, void* blob, float* part, float* small, float* dWT,
                    sonet_stream_t stream, int nprod) {
  using namespace sonet;
  SONET_REQUIRE(dy && x && dyT && blob && part && small && dWT, "wgrad_tc: null pointer");
  SONET_REQUIRE(B >= 1 && P >= 1 && Cout >= 64 && Cout % 64 == 0 && Cin >= 1 && splits >= 1 &&
                    B <= 65535,
                "wgrad_tc: needs Cout %% 64 == 0 (got Cout=%d, Cin=%d)", Cout, Cin);
  cudaStream_t st = as_stream(stream);
  const long long K = static_cast<long long>(B) * P;
  const long long Kpad = sonet_wgrad_kpad(B, P, splits);
  SONET_REQUIRE(Kpad < (1LL << 31), "wgrad_tc: too many points");
  float* s_x = small;             // [2]
  unsigned* bits = reinterpret_cast<unsigned*>(small + 6);
  float* s_dy = small + 8;        // [2 * Cout]: per-channel scales, then their inverses
  channel_scale_kernel<<<Cout, 256, 0, st>>>(dy, B, Cout, P, s_dy);
  int rc = sonet_absmax_scale_f32(x, static_cast<long long>(B) * Cin * P, s_x, bits, stream);
  if (rc) return rc;
  if (Kpad > K)   // zero rows of the padded tail (the matching weight columns are packed as zeros too)
    cudaMemsetAsync(dyT + K * Cout, 0, sizeof(float) * static_cast<size_t>(Kpad - K) * Cout, st);
  transpose_scale_kernel<<<dim3((P + 31) / 32, (Cout + 31) / 32, B), 256, 0, st>>>(dy, Cout, P, s_dy, dyT);
  // x as the weight matrix [Cin][k = (b, p)], zero-padded up to Kpad
  launch_tc_pack(x, Cin, static_cast<int>(K), P, 1, P, static_cast<long long>(Cin) * P, s_x, blob,
                 tc::wblob::kchunks(Kpad), st, nprod);
  rc = check_launch("wgrad_tc(prepare)");
  if (rc) return rc;
  // activations: dyT viewed as [B'=1][C'=Kpad][P'=Cout] (already scaled: no act pre-scale needed);
  // the GEMM writes the raw sums, col_unscale undoes x's scale and each dy channel's
  void* unit = nullptr;
  if (cudaGetSymbolAddress(&unit, kUnitScale) != cudaSuccess) return check_launch("wgrad_tc(unit scale)");
  rc = (nprod == 1 ? sonet_pointwise_tc_forward_dev_f16 : sonet_pointwise_tc_forward_dev)(
      dyT, static_cast<int>(Kpad), 1, Cout, blob, static_cast<const float*>(unit), nullptr, nullptr, Cin,
      0, splits, dWT, part, stream);
  if (rc) return rc;
  const long long n = static_cast<long long>(Cin) * Cout;
  col_unscale_kernel<<<static_cast<unsigned>(std::min<long long>((n + 255) / 256, 2048)), 256, 0, st>>>(
      dWT, n, Cout, s_x + 1, s_dy + Cout);
  return check_launch("wgrad_tc(unscale)");
}

extern "C" int sonet_wgrad_tc_f32(const float* dy, const float* x, int B, int Cout, int Cin, int P,
                                  int splits, float* dyT, void* blob, float* part, float* small,
                                  float* dWT, sonet_stream_t stream) {
  return wgrad_tc(dy, x, B, Cout, Cin, P, splits, dyT, blob, part, small, dWT, stream, 3);
}

// the one-product twin (SONET_TRAIN_TC=fp16): same arguments and scratch sizes
extern "C" int sonet_wgrad_tc_f16(const float* dy, const float* x, int B, int Cout, int Cin, int P,
                                  int splits, float* dyT, void* blob, float* part, float* small,
                                  float* dWT, sonet_stream_t stream) {
  return wgrad_tc(dy, x, B, Cout, Cin, P, splits, dyT, blob, part, small, dWT, stream, 1);
}
