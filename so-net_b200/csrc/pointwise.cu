// pointwise.cu — point-wise shared-MLP layer (1x1 conv + folded BN + ReLU), fp32 CUDA-core path.
//
// Replaces EquivariantLayer / MyConv2d(1x1) eval forward (models/layers.py:203-210, 282-296):
//   out[b,co,p] = act(scale[co] * sum_ci Wt[ci,co] * X[b,ci,p] + shift[co] (+ addend[b,co,g(p)]))
// with X the virtual concat of two channel-first tensors (no torch.cat materialisation).
//
// This is the exact-fp32 path (bit-level IEEE fp32 FMA accumulation; parity 1e-6 vs the
// reference). Register-tiled SGEMM: BMxBN output tile per CTA, 256 threads, BK=8 K-slabs,
// double-buffered shared memory with register prefetch (one __syncthreads per slab), 128-bit
// global loads of the activation rows (P contiguous) and of the transposed weights, conflict-free
// 128-bit shared loads (4x4 sub-tiles strided by BM/2, BN/2), fused epilogue.
// Also: MyLinear (small GEMV-like), row max, gathers used between the layers.
#include <algorithm>

#include <cuda_pipeline.h>

#include "common.cuh"

namespace sonet {

constexpr int PW_BK = 8;

// max(a, b) that is NaN when either operand is NaN, as PyTorch's relu and max are (fmaxf returns
// the other operand). One FMNMX.NAN; for every non-NaN input the same bits as fmaxf.
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// ELU: the ELU epilogue instead of relu ? ReLU : identity (relu is ignored).
// wvec: Cout % 4 == 0 and Wt 16-byte aligned -> 128-bit weight loads.
template <int BM, int BN, int TM, int TN, bool VECP, bool ELU>
__global__ void __launch_bounds__(256, 2)
    pointwise_kernel(const float* __restrict__ x0, int C0, const float* __restrict__ x1, int C1,
                     int P, const float* __restrict__ Wt, int wvec, const float* __restrict__ scale,
                     const float* __restrict__ shift, int Cout, int relu,
                     const float* __restrict__ addend, const int32_t* __restrict__ gidx, int G,
                     float* __restrict__ out) {
  static_assert((BM / TM) * (BN / TN) == 256, "256 threads");
  constexpr int SM_ = TM / 4, SN_ = TN / 4;      // 4x4 sub-tiles per thread
  constexpr int A_F4 = BM * PW_BK / 4 / 256;     // float4 weight loads per thread (may be 0)
  constexpr int B_F4 = BN * PW_BK / 4;           // float4 activation loads per CTA
  __shared__ __align__(16) float As[2][PW_BK][BM];
  __shared__ __align__(16) float Bs[2][PW_BK][BN];

  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int b = blockIdx.z;
  const int co0 = blockIdx.y * BM, p0 = blockIdx.x * BN;
  const int Cin = C0 + C1;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  // ---- global -> register staging -------------------------------------------------------------
  constexpr int A_ITEMS = (A_F4 > 0) ? A_F4 : 1;
  float4 ra[A_ITEMS];
  float4 rb;
  auto load_tiles = [&](int k0) {
    // weights: Wt[k0+kk][co0 + 4*q .. +4]
#pragma unroll
    for (int i = 0; i < A_ITEMS; ++i) {
      const int e = tid + i * 256;  // float4 index in the BK x BM slab
      const int kk = e / (BM / 4), q = e % (BM / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (A_F4 > 0 || e < BM * PW_BK / 4) {
        const int ci = k0 + kk, co = co0 + q * 4;
        if (ci < Cin) {
          const float* src = Wt + static_cast<size_t>(ci) * Cout + co;
          if (wvec && co + 3 < Cout) {
            v = __ldg(reinterpret_cast<const float4*>(src));
          } else {
            if (co < Cout) v.x = __ldg(src);
            if (co + 1 < Cout) v.y = __ldg(src + 1);
            if (co + 2 < Cout) v.z = __ldg(src + 2);
            if (co + 3 < Cout) v.w = __ldg(src + 3);
          }
        }
      }
      ra[i] = v;
    }
    // activations: X[b][k0+kk][p0 + 4*q .. +4]
    {
      const int e = tid;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (e < B_F4) {
        const int kk = e / (BN / 4), q = e % (BN / 4);
        const int ci = k0 + kk, p = p0 + q * 4;
        if (ci < Cin && p < P) {
          const float* src = (ci < C0)
                                 ? x0 + (static_cast<size_t>(b) * C0 + ci) * P + p
                                 : x1 + (static_cast<size_t>(b) * C1 + (ci - C0)) * P + p;
          if (VECP) {
            v = __ldg(reinterpret_cast<const float4*>(src));
          } else {
            v.x = __ldg(src);
            if (p + 1 < P) v.y = __ldg(src + 1);
            if (p + 2 < P) v.z = __ldg(src + 2);
            if (p + 3 < P) v.w = __ldg(src + 3);
          }
        }
      }
      rb = v;
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_ITEMS; ++i) {
      const int e = tid + i * 256;
      if (A_F4 > 0 || e < BM * PW_BK / 4) {
        const int kk = e / (BM / 4), q = e % (BM / 4);
        *reinterpret_cast<float4*>(&As[buf][kk][q * 4]) = ra[i];
      }
    }
    if (tid < B_F4) {
      const int kk = tid / (BN / 4), q = tid % (BN / 4);
      *reinterpret_cast<float4*>(&Bs[buf][kk][q * 4]) = rb;
    }
  };

  const int nk = (Cin + PW_BK - 1) / PW_BK;
  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * PW_BK);
#pragma unroll
    for (int kk = 0; kk < PW_BK; ++kk) {
      float a[TM], bb[TN];
#pragma unroll
      for (int s = 0; s < SM_; ++s) {
        const float4 v = *reinterpret_cast<const float4*>(&As[buf][kk][s * (BM / SM_) + ty * 4]);
        a[s * 4 + 0] = v.x; a[s * 4 + 1] = v.y; a[s * 4 + 2] = v.z; a[s * 4 + 3] = v.w;
      }
#pragma unroll
      for (int s = 0; s < SN_; ++s) {
        const float4 v = *reinterpret_cast<const float4*>(&Bs[buf][kk][s * (BN / SN_) + tx * 4]);
        bb[s * 4 + 0] = v.x; bb[s * 4 + 1] = v.y; bb[s * 4 + 2] = v.z; bb[s * 4 + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

  // ---- epilogue -------------------------------------------------------------------------------------
  int gcol[TN];
  if (addend != nullptr) {
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int p = p0 + (j / 4) * (BN / SN_) + tx * 4 + (j % 4);
      gcol[j] = (p < P) ? min(max(__ldg(gidx + static_cast<size_t>(b) * P + p), 0), G - 1) : 0;
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int co = co0 + (i / 4) * (BM / SM_) + ty * 4 + (i % 4);
    if (co >= Cout) continue;
    const float sc = scale ? __ldg(scale + co) : 1.f;
    const float sh = shift ? __ldg(shift + co) : 0.f;
    const float* arow =
        addend ? addend + (static_cast<size_t>(b) * Cout + co) * G : nullptr;
    float* orow = out + (static_cast<size_t>(b) * Cout + co) * P;
#pragma unroll
    for (int s = 0; s < SN_; ++s) {
      const int p = p0 + s * (BN / SN_) + tx * 4;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float t = fmaf(acc[i][s * 4 + j], sc, sh);
        if (arow) t += __ldg(arow + gcol[s * 4 + j]);
        v[j] = ELU ? elu1(t) : (relu ? fmax_nan(t, 0.f) : t);
      }
      if (VECP) {
        if (p < P) *reinterpret_cast<float4*>(orow + p) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (p + j < P) orow[p + j] = v[j];
      }
    }
  }
}

template <int BM, int BN, int TM, int TN>
static void launch_pointwise(bool vecp, dim3 grid, cudaStream_t st, const float* x0, int C0,
                             const float* x1, int C1, int P, const float* Wt, int wvec,
                             const float* scale, const float* shift, int Cout, int act,
                             const float* addend, const int32_t* gidx, int G, float* out) {
  const int relu = act == SONET_ACT_RELU;
  if (act == SONET_ACT_ELU) {
    if (vecp)
      pointwise_kernel<BM, BN, TM, TN, true, true><<<grid, 256, 0, st>>>(
          x0, C0, x1, C1, P, Wt, wvec, scale, shift, Cout, relu, addend, gidx, G, out);
    else
      pointwise_kernel<BM, BN, TM, TN, false, true><<<grid, 256, 0, st>>>(
          x0, C0, x1, C1, P, Wt, wvec, scale, shift, Cout, relu, addend, gidx, G, out);
  } else if (vecp) {
    pointwise_kernel<BM, BN, TM, TN, true, false><<<grid, 256, 0, st>>>(
        x0, C0, x1, C1, P, Wt, wvec, scale, shift, Cout, relu, addend, gidx, G, out);
  } else {
    pointwise_kernel<BM, BN, TM, TN, false, false><<<grid, 256, 0, st>>>(
        x0, C0, x1, C1, P, Wt, wvec, scale, shift, Cout, relu, addend, gidx, G, out);
  }
}

// ---- MyLinear: out[b,co] = act(scale*(W[co,:].x[b,:]) + shift): warp per output element -----------
// (ELU in all three MyLinear kernels: the ELU epilogue, relu ignored)
template <bool ELU>
__global__ void __launch_bounds__(256)
    linear_kernel(const float* __restrict__ x, int B, int Cin, const float* __restrict__ W,
                  const float* __restrict__ scale, const float* __restrict__ shift, int Cout,
                  int relu, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp_id = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long total = static_cast<long long>(B) * Cout;
  if (warp_id >= total) return;
  const int b = static_cast<int>(warp_id / Cout), co = static_cast<int>(warp_id % Cout);
  const float* xr = x + static_cast<size_t>(b) * Cin;
  const float* wr = W + static_cast<size_t>(co) * Cin;
  float s = 0.f;
  for (int i = lane; i < Cin; i += 32) s = fmaf(__ldg(wr + i), __ldg(xr + i), s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    float t = fmaf(s, scale ? scale[co] : 1.f, shift ? shift[co] : 0.f);
    out[warp_id] = ELU ? elu1(t) : (relu ? fmax_nan(t, 0.f) : t);
  }
}

// ---- MyLinear, blocked: a block owns CT output channels for all clouds ------------------------------
// The warp-per-output kernel above re-reads a weight row once per cloud (B x Cout x Cin loads through
// L1: 22 us for [64,1024]->512). Here the CT weight rows of a block are staged in shared memory once,
// each warp takes clouds warp, warp+8, ... two at a time (one LDS.128 of weights feeds two clouds'
// FMAs), lanes stride the K axis in float4, and a butterfly reduces the 2*CT sums. Weight traffic:
// once; activation traffic: (Cout/CT) x B x Cin from L2. Requires Cin % 4 == 0 and 16-byte aligned rows.
template <int CT, bool ELU>
__global__ void __launch_bounds__(256)
    linear_block_kernel(const float* __restrict__ x, int B, int Cin, const float* __restrict__ W,
                        const float* __restrict__ scale, const float* __restrict__ shift, int Cout,
                        int relu, float* __restrict__ out) {
  extern __shared__ __align__(16) float lb_w[];           // [CT][Cin]
  const int co0 = blockIdx.x * CT;
  const int c4 = Cin >> 2;
  float4* sw = reinterpret_cast<float4*>(lb_w);
  for (int i = threadIdx.x; i < CT * c4; i += 256) {
    const int c = i / c4, k = i - c * c4;
    sw[i] = (co0 + c < Cout) ? __ldg(reinterpret_cast<const float4*>(W + static_cast<size_t>(co0 + c) * Cin) + k)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int b0 = 2 * warp; b0 < B; b0 += 16) {
    const bool two = b0 + 1 < B;
    const float4* xa = reinterpret_cast<const float4*>(x + static_cast<size_t>(b0) * Cin);
    const float4* xb = reinterpret_cast<const float4*>(x + static_cast<size_t>(two ? b0 + 1 : b0) * Cin);
    float acc[2][CT];
#pragma unroll
    for (int c = 0; c < CT; ++c) acc[0][c] = acc[1][c] = 0.f;
#pragma unroll 2
    for (int k = lane; k < c4; k += 32) {
      const float4 va = __ldg(xa + k), vb = __ldg(xb + k);
#pragma unroll
      for (int c = 0; c < CT; ++c) {
        const float4 w = sw[c * c4 + k];
        acc[0][c] = fmaf(w.w, va.w, fmaf(w.z, va.z, fmaf(w.y, va.y, fmaf(w.x, va.x, acc[0][c]))));
        acc[1][c] = fmaf(w.w, vb.w, fmaf(w.z, vb.z, fmaf(w.y, vb.y, fmaf(w.x, vb.x, acc[1][c]))));
      }
    }
#pragma unroll
    for (int c = 0; c < CT; ++c)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        acc[0][c] += __shfl_xor_sync(0xffffffffu, acc[0][c], o);
        acc[1][c] += __shfl_xor_sync(0xffffffffu, acc[1][c], o);
      }
    // lane c writes channel c of cloud b0, lane CT + c of cloud b0 + 1
    if (lane < 2 * CT) {
      const int h = lane / CT, c = lane - h * CT;
      float v = 0.f;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int cc = 0; cc < CT; ++cc)
          if (hh == h && cc == c) v = acc[hh][cc];
      const int co = co0 + c;
      if (co < Cout && (h == 0 || two)) {
        const float t = fmaf(v, scale ? __ldg(scale + co) : 1.f, shift ? __ldg(shift + co) : 0.f);
        out[static_cast<size_t>(b0 + h) * Cout + co] = ELU ? elu1(t) : (relu ? fmax_nan(t, 0.f) : t);
      }
    }
  }
}

// ---- MyLinear, tiled: a block owns a [16 clouds x 16 channels] output tile ------------------------
// The FC layers are latency-, not throughput-bound (67 MFLOP at [64,1024]->512): what matters is how
// many dependent memory round trips a block makes. Here ALL operand bytes of the tile (16 rows of x,
// 16 rows of W) are requested up front with 16-byte cp.async in four K stages, so the fetch latency is
// paid once and the FMAs of stage s overlap the arrival of stages s+1..3. Thread (cloud, channel)
// computes one output from shared memory: the x row is a broadcast, the 16 weight rows of a warp sit
// 4 banks apart (row stride Cin + 4 floats) -> conflict-free LDS.128. Summation order depends on K
// only (four interleaved partial sums, k ascending): results do not depend on the batch composition.
constexpr int LT_B = 16, LT_C = 16, LT_STAGES = 4;

template <bool ELU>
__global__ void __launch_bounds__(256)
    linear_tile_kernel(const float* __restrict__ x, int B, int Cin, const float* __restrict__ W,
                       const float* __restrict__ scale, const float* __restrict__ shift, int Cout,
                       int relu, float* __restrict__ out) {
  extern __shared__ __align__(16) float lt_smem[];
  const int c4 = Cin >> 2;               // float4 columns per row
  const int ld4 = c4 + 1;                // padded row stride in float4
  float4* xs = reinterpret_cast<float4*>(lt_smem);          // [LT_B][ld4]
  float4* ws = xs + LT_B * ld4;                              // [LT_C][ld4]
  const int b0 = blockIdx.y * LT_B, co0 = blockIdx.x * LT_C;
  const int per = (c4 + LT_STAGES - 1) / LT_STAGES;
  for (int s = 0; s < LT_STAGES; ++s) {
    const int k0 = s * per, k1 = min(c4, k0 + per);
    const int cols = max(0, k1 - k0);
    for (int i = threadIdx.x; i < (LT_B + LT_C) * cols; i += 256) {
      const int row = i / cols, k = k0 + (i - row * cols);
      float4* dst = xs + row * ld4 + k;   // rows LT_B.. continue into ws
      const float* src = nullptr;
      if (row < LT_B) {
        if (b0 + row < B) src = x + static_cast<size_t>(b0 + row) * Cin;
      } else if (co0 + row - LT_B < Cout) {
        src = W + static_cast<size_t>(co0 + row - LT_B) * Cin;
      }
      if (src != nullptr)
        __pipeline_memcpy_async(dst, reinterpret_cast<const float4*>(src) + k, 16);
      else
        *dst = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __pipeline_commit();
  }
  const int cloud = threadIdx.x >> 4, ch = threadIdx.x & 15;
  const float4* xr = xs + cloud * ld4;
  const float4* wr = ws + ch * ld4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int s = 0; s < LT_STAGES; ++s) {
    __pipeline_wait_prior(LT_STAGES - 1 - s);
    __syncthreads();
    const int k0 = s * per, k1 = min(c4, k0 + per);
#pragma unroll 4
    for (int k = k0; k < k1; ++k) {
      const float4 a = xr[k], w = wr[k];
      acc.x = fmaf(a.x, w.x, acc.x);
      acc.y = fmaf(a.y, w.y, acc.y);
      acc.z = fmaf(a.z, w.z, acc.z);
      acc.w = fmaf(a.w, w.w, acc.w);
    }
  }
  const int b = b0 + cloud, co = co0 + ch;
  if (b < B && co < Cout) {
    const float v = (acc.x + acc.y) + (acc.z + acc.w);
    const float t = fmaf(v, scale ? __ldg(scale + co) : 1.f, shift ? __ldg(shift + co) : 0.f);
    out[static_cast<size_t>(b) * Cout + co] = ELU ? elu1(t) : (relu ? fmax_nan(t, 0.f) : t);
  }
}

// ---- row max, L = 4*G with G a power of two <= 32: G lanes per row, one 128-bit load per lane,
// four row groups in flight per warp ----
__global__ void __launch_bounds__(256)
    rowmax_vec_kernel(const float4* __restrict__ in, long long R, int G, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp_id = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int rpw = 32 / G;                       // rows per warp and pass
  const int sub = lane / G;
  const long long row0 = warp_id * (4LL * rpw) + sub;
  float m[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const long long r = row0 + static_cast<long long>(u) * rpw;
    if (r < R) {
      const float4 v = __ldg(in + r * G + (lane - sub * G));
      m[u] = fmax_nan(fmax_nan(v.x, v.y), fmax_nan(v.z, v.w));
    } else {
      m[u] = -__int_as_float(0x7f800000);
    }
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    for (int o = G >> 1; o > 0; o >>= 1) m[u] = fmax_nan(m[u], __shfl_xor_sync(0xffffffffu, m[u], o));
    const long long r = row0 + static_cast<long long>(u) * rpw;
    if (lane == sub * G && r < R) out[r] = m[u];
  }
}

// ---- row max: in [R, L] -> out [R] --------------------------------------------------------------------
// L <= 32: one thread per row group (lanes cover consecutive rows); else one warp per row.
__global__ void __launch_bounds__(256)
    rowmax_small_kernel(const float* __restrict__ in, long long R, int L, float* __restrict__ out) {
  const long long r = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float* p = in + r * L;
  float m = p[0];
  for (int i = 1; i < L; ++i) m = fmax_nan(m, p[i]);
  out[r] = m;
}
__global__ void __launch_bounds__(256)
    rowmax_warp_kernel(const float* __restrict__ in, long long R, int L, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long r = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (r >= R) return;
  const float* p = in + r * L;
  float m = -__int_as_float(0x7f800000);
  for (int i = lane; i < L; i += 32) m = fmax_nan(m, p[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax_nan(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) out[r] = m;
}

// ---- gathers -----------------------------------------------------------------------------------------
__device__ __forceinline__ int clamp_idx(int64_t v, int M) {
  const long long w = static_cast<long long>(v);
  return static_cast<int>(w < 0 ? 0 : (w > M - 1 ? M - 1 : w));
}
__global__ void __launch_bounds__(256)
    knn_gather_kernel(const float* __restrict__ src, const int64_t* __restrict__ idx, int C, int M,
                      int K, int Kstride, float* __restrict__ out, long long total) {
  // out[b,c,m,j] = src[b,c,idx[b,m,j]]
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(t % K);
    const long long r = t / K;
    const int m = static_cast<int>(r % M);
    const long long bc = r / M;
    const long long b = bc / C;
    const int id = clamp_idx(idx[(b * M + m) * Kstride + j], M);
    out[t] = __ldg(src + bc * M + id);
  }
}

// KNNModule input assembly (models/layers.py:346-361). One CTA per (b, m-chunk); channels strided.
__global__ void __launch_bounds__(256)
    knn_assemble_kernel(const float* __restrict__ coord, const float* __restrict__ feat,
                        const int64_t* __restrict__ idx, int C, int M, int K, int Kstride,
                        int center_type, float* __restrict__ center, float* __restrict__ x_aug) {
  const int b = blockIdx.y;
  const int MK = M * K;
  const int CA = 3 + C;
  const float* cb = coord + static_cast<size_t>(b) * 3 * M;
  const float* fb = feat + static_cast<size_t>(b) * C * M;
  float* ob = x_aug + static_cast<size_t>(b) * CA * MK;
  const int64_t* ib = idx + static_cast<size_t>(b) * M * Kstride;
  // coordinates: thread per (c, m)
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < 3 * M; t += gridDim.x * blockDim.x) {
    const int c = t / M, m = t % M;
    float ctr;
    if (center_type == 0) {  // 'avg': torch.mean over K = sum / K
      float s = 0.f;
      for (int j = 0; j < K; ++j) {
        int id = clamp_idx(ib[m * Kstride + j], M);
        s += cb[c * M + id];
      }
      ctr = __fdiv_rn(s, static_cast<float>(K));
    } else {
      ctr = cb[c * M + m];
    }
    center[(static_cast<size_t>(b) * 3 + c) * M + m] = ctr;
    if (x_aug == nullptr) continue;
    for (int j = 0; j < K; ++j) {
      int id = clamp_idx(ib[m * Kstride + j], M);
      ob[static_cast<size_t>(c) * MK + m * K + j] = __fsub_rn(cb[c * M + id], ctr);
    }
  }
  if (x_aug == nullptr) return;   // center only (the fused KNN MLP decentres on its own)
  // features: thread per (c, m, j); 32-bit index arithmetic (the launcher checks C*M*K < 2^31 — the
  // 64-bit division and modulo per element were what this loop spent its time on)
  const uint32_t total = static_cast<uint32_t>(C) * MK;
  const uint32_t uMK = static_cast<uint32_t>(MK), uK = static_cast<uint32_t>(K);
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
    const uint32_t c = t / uMK;
    const uint32_t mj = t - c * uMK;
    const uint32_t m = mj / uK, j = mj - m * uK;
    const int id = clamp_idx(ib[m * Kstride + j], M);
    ob[static_cast<size_t>(3 + c) * MK + mj] = __ldg(fb + static_cast<size_t>(c) * M + id);
  }
}

// Same assembly for the fused-pool path, reading the per-node maxima straight from the pool keys:
// pool_finalize (key -> value, empty node -> feature of copy 0, key reset) is folded in, so the
// [B,C,M] maxima are written once (first_pn_out_masked_max, an Encoder attribute) and gathered
// from shared memory. CTA = (channel group, cloud); threads run over the M*K output columns, so
// the inner loop has no divisions and its stores are coalesced.
constexpr int KA_CPB = 16;       // channels per CTA
__device__ __forceinline__ bool sonet_aligned16_ptr(const void* p) {
  return (reinterpret_cast<uintptr_t>(p) & 15u) == 0;
}
constexpr int KA_MAX_MK = 2304;  // M*K positions cached per CTA

// center [b,3,M] and, when ob is not null, the decentred coordinates = channels 0-2 of x_aug:
// thread per (c, m)
__device__ void knn_pool_center(const float* __restrict__ coord, int b, int M, int K, int center_type,
                                const uint16_t* sid, float* __restrict__ center, float* __restrict__ ob) {
  const float* cb = coord + static_cast<size_t>(b) * 3 * M;
  const int MK = M * K;
  for (int t = threadIdx.x; t < 3 * M; t += blockDim.x) {
    const int c = t / M, m = t - c * M;
    float ctr;
    if (center_type == 0) {  // 'avg': torch.mean over K = sum / K
      float s = 0.f;
      for (int j = 0; j < K; ++j) s += cb[c * M + sid[m * K + j]];
      ctr = __fdiv_rn(s, static_cast<float>(K));
    } else {
      ctr = cb[c * M + m];
    }
    center[(static_cast<size_t>(b) * 3 + c) * M + m] = ctr;
    if (ob == nullptr) continue;
    for (int j = 0; j < K; ++j)
      ob[static_cast<size_t>(c) * MK + m * K + j] = __fsub_rn(cb[c * M + sid[m * K + j]], ctr);
  }
}

__global__ void __launch_bounds__(256)
    knn_assemble_pool_kernel(const float* __restrict__ coord, int32_t* __restrict__ keys,
                             const float* __restrict__ p0, const int64_t* __restrict__ idx, int C,
                             int M, int K, int Kstride, int center_type,
                             float* __restrict__ masked_max, float* __restrict__ center,
                             float* __restrict__ x_aug) {
  __shared__ float vals[KA_CPB * 256];          // [KA_CPB][M], M <= 256
  __shared__ __align__(16) uint16_t sid[KA_MAX_MK];
  const int b = blockIdx.y;
  const int MK = M * K;
  const int c0 = blockIdx.x * KA_CPB;
  const int nc = min(KA_CPB, C - c0);
  const int64_t* ib = idx + static_cast<size_t>(b) * M * Kstride;
  for (int mj = threadIdx.x; mj < MK; mj += blockDim.x) {
    const int m = mj / K, j = mj - m * K;
    sid[mj] = static_cast<uint16_t>(clamp_idx(ib[m * Kstride + j], M));
  }
  for (int t = threadIdx.x; t < nc * M; t += blockDim.x) {
    const int cl = t / M, m = t - cl * M;
    const size_t g = (static_cast<size_t>(b) * C + c0 + cl) * M + m;
    const float v = pool_key_value(keys[g], __ldg(p0 + static_cast<size_t>(b) * C + c0 + cl));
    keys[g] = POOL_KEY_INIT;                      // ready for the next forward
    masked_max[g] = v;
    vals[cl * M + m] = v;
  }
  if (x_aug == nullptr) {   // the fused KNN MLP gathers and decentres on its own
    if (blockIdx.x == 0) {
      __syncthreads();         // sid
      knn_pool_center(coord, b, M, K, center_type, sid, center, nullptr);
    }
    return;
  }
  __syncthreads();
  float* ob = x_aug + static_cast<size_t>(b) * (3 + C) * MK;
  if ((MK & 3) == 0 && sonet_aligned16_ptr(ob)) {
    // four output columns per thread: one 8-byte read of the neighbour ids, one 16-byte store
    const int MK4 = MK >> 2;
    for (int t = threadIdx.x; t < nc * MK4; t += blockDim.x) {
      const int cl = t / MK4, q = t - cl * MK4;
      const float* vrow = vals + cl * M;
      const uint2 ids = *reinterpret_cast<const uint2*>(sid + 4 * q);
      float4 v;
      v.x = vrow[ids.x & 0xffffu];
      v.y = vrow[ids.x >> 16];
      v.z = vrow[ids.y & 0xffffu];
      v.w = vrow[ids.y >> 16];
      reinterpret_cast<float4*>(ob + static_cast<size_t>(3 + c0 + cl) * MK)[q] = v;
    }
  } else {
    for (int cl = 0; cl < nc; ++cl) {
      float* orow = ob + static_cast<size_t>(3 + c0 + cl) * MK;
      const float* vrow = vals + cl * M;
      for (int mj = threadIdx.x; mj < MK; mj += blockDim.x) orow[mj] = vrow[sid[mj]];
    }
  }
  if (blockIdx.x == 0) knn_pool_center(coord, b, M, K, center_type, sid, center, ob);
}

// exact K-NN among the M nodes (models/layers.py:334-337): thread per (b, m).
__global__ void __launch_bounds__(128)
    node_knn_kernel(const float* __restrict__ coord, int B, int M, int K,
                    int64_t* __restrict__ idx) {
  extern __shared__ float sc[];  // [3][M] of this cloud
  const int b = blockIdx.x;
  const float* cb = coord + static_cast<size_t>(b) * 3 * M;
  for (int i = threadIdx.x; i < 3 * M; i += blockDim.x) sc[i] = cb[i];
  __syncthreads();
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    int64_t* o = idx + (static_cast<size_t>(b) * M + m) * K;
    float last_d = -1.f;
    int last_i = -1;
    // K passes of "next smallest (d, i) greater than the last emitted" — K, M are tiny.
    for (int j = 0; j < K; ++j) {
      float bd = __int_as_float(0x7f800000);
      int bi = M;
      for (int q = 0; q < M; ++q) {
        const float dx = __fsub_rn(sc[m], sc[q]), dy = __fsub_rn(sc[M + m], sc[M + q]),
                    dz = __fsub_rn(sc[2 * M + m], sc[2 * M + q]);
        const float d =
            __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        const bool after = (d > last_d) || (d == last_d && q > last_i);
        if (after && (d < bd || (d == bd && q < bi))) {
          bd = d;
          bi = q;
        }
      }
      if (bi == M) bi = (last_i + 1 < M) ? last_i + 1 : M - 1;  // NaN coordinates: stay in range
      o[j] = bi;
      last_d = bd;
      last_i = bi;
    }
  }
}

__global__ void __launch_bounds__(256)
    gather_points_kernel(const float* __restrict__ src, const int32_t* __restrict__ gidx, int C,
                         int M, int P, float* __restrict__ out, long long total) {
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int p = static_cast<int>(t % P);
    const long long bc = t / P;
    const long long b = bc / C;
    const int g = min(max(__ldg(gidx + b * P + p), 0), M - 1);
    out[t] = __ldg(src + bc * M + g);
  }
}

__global__ void __launch_bounds__(256)
    kcopy_mean_kernel(const float* __restrict__ in, long long rows, int N, int k,
                      float* __restrict__ out) {
  const long long total = rows * N;
  const float w = (k == 2) ? 0.5f : (k == 3 ? (1.0f / 3.0f) : __fdiv_rn(1.0f, (float)k));
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = t / N;
    const int n = static_cast<int>(t - r * N);
    const float* p = in + r * k * N + n;
    float s = p[0];
    for (int i = 1; i < k; ++i) s = __fadd_rn(s, p[static_cast<size_t>(i) * N]);
    out[t] = __fmul_rn(w, s);
  }
}

// N % 4 == 0 and 16-byte aligned rows: one float4 of k copies per thread, 32-bit indexing per row
__global__ void __launch_bounds__(256)
    kcopy_mean_vec4_kernel(const float4* __restrict__ in, long long rows, int n4, int k,
                           float4* __restrict__ out) {
  const float w = (k == 2) ? 0.5f : (k == 3 ? (1.0f / 3.0f) : __fdiv_rn(1.0f, (float)k));
  const long long total = rows * n4;
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = t / n4;
    const int n = static_cast<int>(t - r * n4);
    const float4* p = in + r * k * n4 + n;
    float4 s = ldg_stream_f4(p);
    for (int i = 1; i < k; ++i) {
      const float4 v = ldg_stream_f4(p + static_cast<size_t>(i) * n4);
      s.x = __fadd_rn(s.x, v.x);
      s.y = __fadd_rn(s.y, v.y);
      s.z = __fadd_rn(s.z, v.z);
      s.w = __fadd_rn(s.w, v.w);
    }
    out[t] = make_float4(__fmul_rn(w, s.x), __fmul_rn(w, s.y), __fmul_rn(w, s.z), __fmul_rn(w, s.w));
  }
}

static inline int grid_for(long long total, int threads, int sms) {
  return static_cast<int>(std::max<long long>(
      1, std::min<long long>((total + threads - 1) / threads, 32LL * sms)));
}

}  // namespace sonet

extern "C" int sonet_pointwise_layer_f32(const float* x0, int C0, const float* x1, int C1, int B,
                                         int P, const float* Wt, const float* scale,
                                         const float* shift, int Cout, int relu,
                                         const float* addend, const int32_t* gidx, int G,
                                         float* out, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE_ACT(relu, "pointwise");
  SONET_REQUIRE(B >= 0 && P >= 0 && C0 >= 1 && C1 >= 0 && Cout >= 1, "pointwise: bad dimension");
  SONET_REQUIRE(B <= 65535, "pointwise: B=%d exceeds grid limit", B);
  if (B == 0 || P == 0) return SONET_OK;
  SONET_REQUIRE(x0 && Wt && out, "pointwise: null pointer");
  SONET_REQUIRE(C1 == 0 || x1 != nullptr, "pointwise: x1 null with C1=%d", C1);
  SONET_REQUIRE(!addend || (gidx && G >= 1), "pointwise: addend needs gidx and G");
  // 128-bit loads: of the activation rows and the output (vecp), of the weight rows (wvec)
  const bool vecp = (P % 4 == 0) && aligned16(x0) && aligned16(out) && (C1 == 0 || aligned16(x1));
  const int wvec = (Cout % 4 == 0) && aligned16(Wt);
  cudaStream_t st = as_stream(stream);
  if (P >= 1024 && Cout >= 128) {
    dim3 grid((P + 127) / 128, (Cout + 127) / 128, B);
    SONET_REQUIRE(grid.y <= 65535, "pointwise: Cout too large");
    launch_pointwise<128, 128, 8, 8>(vecp, grid, st, x0, C0, x1, C1, P, Wt, wvec, scale, shift, Cout,
                                     relu, addend, gidx, G, out);
  } else {
    dim3 grid((P + 63) / 64, (Cout + 63) / 64, B);
    SONET_REQUIRE(grid.y <= 65535, "pointwise: Cout too large");
    launch_pointwise<64, 64, 4, 4>(vecp, grid, st, x0, C0, x1, C1, P, Wt, wvec, scale, shift, Cout,
                                   relu, addend, gidx, G, out);
  }
  return check_launch("pointwise_layer");
}

namespace sonet {
template <bool ELU>
static int launch_linear(const float* x, int B, int Cin, const float* W, const float* scale,
                         const float* shift, int Cout, int relu, float* out, cudaStream_t st) {
  const size_t tile_smem = static_cast<size_t>(LT_B + LT_C) * (Cin / 4 + 1) * sizeof(float4);
  if (Cin % 4 == 0 && aligned16(x) && aligned16(W) && tile_smem <= static_cast<size_t>(max_smem_optin())) {
    cudaFuncSetAttribute(linear_tile_kernel<ELU>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         static_cast<int>(tile_smem));
    dim3 grid((Cout + LT_C - 1) / LT_C, (B + LT_B - 1) / LT_B);
    if (grid.y <= 65535) {
      linear_tile_kernel<ELU><<<grid, 256, tile_smem, st>>>(x, B, Cin, W, scale, shift, Cout, relu, out);
      return check_launch("linear");
    }
  }
  if (Cin % 4 == 0 && aligned16(x) && aligned16(W)) {
    // the widest channel tile that still fills the SMs and fits 48 KB of shared memory
    const int sms = sm_count();
    int ct = 4;
    while (ct > 1 && ((Cout + ct - 1) / ct < (sms * 3) / 4 || static_cast<size_t>(ct) * Cin * 4 > 48 * 1024))
      ct >>= 1;
    const size_t smem = static_cast<size_t>(ct) * Cin * sizeof(float);
    if (smem <= 48 * 1024) {
      const int grid = (Cout + ct - 1) / ct;
      if (ct == 4)
        linear_block_kernel<4, ELU><<<grid, 256, smem, st>>>(x, B, Cin, W, scale, shift, Cout, relu, out);
      else if (ct == 2)
        linear_block_kernel<2, ELU><<<grid, 256, smem, st>>>(x, B, Cin, W, scale, shift, Cout, relu, out);
      else
        linear_block_kernel<1, ELU><<<grid, 256, smem, st>>>(x, B, Cin, W, scale, shift, Cout, relu, out);
      return check_launch("linear");
    }
  }
  const long long total = static_cast<long long>(B) * Cout;
  const int grid = static_cast<int>((total * 32 + 255) / 256);
  linear_kernel<ELU><<<grid, 256, 0, st>>>(x, B, Cin, W, scale, shift, Cout, relu, out);
  return check_launch("linear");
}
}  // namespace sonet

extern "C" int sonet_linear_f32(const float* x, int B, int Cin, const float* W, const float* scale,
                                const float* shift, int Cout, int relu, float* out,
                                sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE_ACT(relu, "linear");
  SONET_REQUIRE(B >= 0 && Cin >= 1 && Cout >= 1, "linear: bad dimension");
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(x && W && out, "linear: null pointer");
  if (relu == SONET_ACT_ELU)
    return launch_linear<true>(x, B, Cin, W, scale, shift, Cout, 0, out, as_stream(stream));
  return launch_linear<false>(x, B, Cin, W, scale, shift, Cout, relu, out, as_stream(stream));
}

extern "C" int sonet_rowmax_f32(const float* in, int R, int L, float* out, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(R >= 0 && L >= 1, "rowmax: bad dimension");
  if (R == 0) return SONET_OK;
  SONET_REQUIRE(in && out, "rowmax: null pointer");
  const int G = L / 4;
  if (L % 4 == 0 && G >= 1 && G <= 32 && (G & (G - 1)) == 0 && L > 32 && aligned16(in)) {
    const long long warps = (static_cast<long long>(R) + 4 * (32 / G) - 1) / (4 * (32 / G));
    rowmax_vec_kernel<<<static_cast<int>((warps * 32 + 255) / 256), 256, 0, as_stream(stream)>>>(
        reinterpret_cast<const float4*>(in), R, G, out);
  } else if (L <= 32) {
    rowmax_small_kernel<<<(R + 255) / 256, 256, 0, as_stream(stream)>>>(in, R, L, out);
  } else {
    const long long threads = static_cast<long long>(R) * 32;
    rowmax_warp_kernel<<<static_cast<int>((threads + 255) / 256), 256, 0, as_stream(stream)>>>(
        in, R, L, out);
  }
  return check_launch("rowmax");
}

extern "C" int sonet_knn_gather_f32(const float* src, const int64_t* idx, int B, int C, int M, int K,
                                    int Kstride, float* out, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 0 && M >= 1 && K >= 1 && Kstride >= K, "knn_gather: bad dimension");
  const long long total = static_cast<long long>(B) * C * M * K;
  if (total == 0) return SONET_OK;
  SONET_REQUIRE(src && idx && out, "knn_gather: null pointer");
  knn_gather_kernel<<<grid_for(total, 256, sm_count()), 256, 0, as_stream(stream)>>>(
      src, idx, C, M, K, Kstride, out, total);
  return check_launch("knn_gather");
}

extern "C" int sonet_knn_assemble_f32(const float* coord, const float* feat, const int64_t* idx,
                                      int B, int C, int M, int K, int Kstride, int center_type,
                                      float* center, float* x_aug, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 0 && M >= 1 && K >= 1 && Kstride >= K, "knn_assemble: bad dimension");
  SONET_REQUIRE(center_type == 0 || center_type == 1, "knn_assemble: center_type must be 0|1");
  SONET_REQUIRE(B <= 65535, "knn_assemble: B=%d exceeds grid limit", B);
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(coord && (feat || C == 0 || !x_aug) && idx && center, "knn_assemble: null pointer");
  const long long per_b = x_aug ? static_cast<long long>(C + 3) * M * K : 3LL * M;
  SONET_REQUIRE(per_b < (1LL << 31), "knn_assemble: C*M*K = %lld exceeds the 32-bit index range", per_b);
  dim3 grid(static_cast<unsigned>(std::max<long long>(1, std::min<long long>((per_b + 255) / 256, 64))), B);
  knn_assemble_kernel<<<grid, 256, 0, as_stream(stream)>>>(coord, feat, idx, C, M, K, Kstride,
                                                           center_type, center, x_aug);
  return check_launch("knn_assemble");
}

extern "C" int sonet_knn_assemble_pool_f32(const float* coord, int32_t* pool_keys, const float* p0,
                                           const int64_t* idx, int B, int C, int M, int K,
                                           int Kstride, int center_type, float* masked_max,
                                           float* center, float* x_aug, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 1 && M >= 1 && K >= 1 && Kstride >= K,
                "knn_assemble_pool: bad dimension");
  SONET_REQUIRE(center_type == 0 || center_type == 1, "knn_assemble_pool: center_type %d", center_type);
  SONET_REQUIRE(M <= 256 && static_cast<long long>(M) * K <= KA_MAX_MK,
                "knn_assemble_pool: M=%d, K=%d exceed the per-CTA cache (finalize the pool and use "
                "sonet_knn_assemble_f32)", M, K);
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(coord && pool_keys && p0 && idx && masked_max && center,
                "knn_assemble_pool: null pointer");
  dim3 grid(static_cast<unsigned>((C + KA_CPB - 1) / KA_CPB), B);
  knn_assemble_pool_kernel<<<grid, 256, 0, as_stream(stream)>>>(
      coord, pool_keys, p0, idx, C, M, K, Kstride, center_type, masked_max, center, x_aug);
  return check_launch("knn_assemble_pool");
}

extern "C" int sonet_node_knn(const float* coord, int B, int M, int K, int64_t* idx,
                              sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && M >= 1 && K >= 1 && K <= M, "node_knn: bad dimension");
  SONET_REQUIRE(M <= 4096, "node_knn: M=%d too large", M);
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(coord && idx, "node_knn: null pointer");
  node_knn_kernel<<<B, 128, 3 * M * sizeof(float), as_stream(stream)>>>(coord, B, M, K, idx);
  return check_launch("node_knn");
}

extern "C" int sonet_gather_points_f32(const float* src, const int32_t* gidx, int B, int C, int M,
                                       int P, float* out, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 0 && M >= 1 && P >= 0, "gather_points: bad dimension");
  const long long total = static_cast<long long>(B) * C * P;
  if (total == 0) return SONET_OK;
  SONET_REQUIRE(src && gidx && out, "gather_points: null pointer");
  gather_points_kernel<<<grid_for(total, 256, sm_count()), 256, 0, as_stream(stream)>>>(
      src, gidx, C, M, P, out, total);
  return check_launch("gather_points");
}

extern "C" int sonet_kcopy_mean_f32(const float* in, int B, int C, int N, int k, float* out,
                                    sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && C >= 0 && N >= 0 && k >= 1, "kcopy_mean: bad dimension");
  const long long rows = static_cast<long long>(B) * C;
  if (rows * N == 0) return SONET_OK;
  SONET_REQUIRE(in && out, "kcopy_mean: null pointer");
  if (N % 4 == 0 && aligned16(in) && aligned16(out)) {
    const int n4 = N / 4;
    kcopy_mean_vec4_kernel<<<grid_for(rows * n4, 256, sm_count()), 256, 0, as_stream(stream)>>>(
        reinterpret_cast<const float4*>(in), rows, n4, k, reinterpret_cast<float4*>(out));
    return check_launch("kcopy_mean");
  }
  kcopy_mean_kernel<<<grid_for(rows * N, 256, sm_count()), 256, 0, as_stream(stream)>>>(in, rows, N, k,
                                                                                       out);
  return check_launch("kcopy_mean");
}
