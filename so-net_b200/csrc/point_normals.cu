// point_normals.cu — exact k nearest neighbours within each cloud of a ragged batch, and surface
// normals estimated from them (sm_90a): the normals SO-Net reads, for point clouds that have none.
//
// Layout (include/sonet_b200.h): data [T, stride] f32 point-major with xyz in columns 0..2; cloud s
// is rows offsets[s] .. offsets[s+1], clamped as common.cuh's ragged_range states.
//
// k-NN: d = ((dx*dx + dy*dy) + dz*dz), dx = q.x - p.x, every operation explicitly rounded (no FMA
// contraction), the convention of the SOM assignment and sonet_node_knn. Each thread owns one query
// and keeps its sorted top-K in registers; candidates stream through shared memory in ascending index
// order, so a strict `<` against the current K-th distance keeps the lower index first on ties. A
// distance enters only when it is below the K-th, so +inf and NaN never enter on that pass; a query
// left with empty slots (fewer than K finite distances) gets them filled by one more pass over the
// cloud with the +inf candidates, then the NaN ones, each in index order. Work is (cloud, 128-query
// tile) on a 2-D grid: blockIdx.y strides the clouds, blockIdx.x the tiles of a cloud, so a cloud's
// bits never depend on the rest of the batch.
//
// Normals: per point, the valid neighbours' mean and centred covariance in fp64 (two passes in slot
// order, explicitly rounded), cyclic Jacobi for the eigenvector of the smallest eigenvalue, fp64
// normalisation, one rounding to f32, then the sign rule (canonical, then the orientation code).
#include <math.h>

#include "common.cuh"

namespace sonet {

constexpr int PK_QTILE = 128;                   // queries per work item (one per thread)
constexpr int PK_CTILE = 1024;                  // candidates staged per shared-memory tile
constexpr long long PK_MAX_CLOUD = 2147483647LL;  // cloud-local indices are int32
constexpr int PN_THREADS = 128;
constexpr int PC_THREADS = 256;                 // centroid: one CTA per cloud, fixed reduction tree

// A cloud's first row and row count (common.cuh's ragged_range); the count is at most 2^31-1 (the
// rest of a longer range is not part of the cloud).
__device__ __forceinline__ void pk_range(const int64_t* off, int s, long long T, long long& begin,
                                         int& count) {
  long long end;
  ragged_range(off, s, T, begin, end);
  count = static_cast<int>(end - begin > PK_MAX_CLOUD ? PK_MAX_CLOUD : end - begin);
}

__device__ __forceinline__ float pk_dist(float qx, float qy, float qz, float px, float py, float pz) {
  const float dx = __fsub_rn(qx, px), dy = __fsub_rn(qy, py), dz = __fsub_rn(qz, pz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// KK register slots, ascending; the first KK-K hold (-inf, -1) and never move, so the K-th distance
// is always bd[KK-1] (a static index) whatever K is.
template <int KK>
__device__ __forceinline__ void pk_insert(float (&bd)[KK], int (&bi)[KK], float d, int j) {
#pragma unroll
  for (int s = KK - 1; s > 0; --s) {
    const bool shift = bd[s - 1] > d;   // stays false at the -inf slots
    const bool here = !shift && bd[s] > d;
    if (here) {
      bd[s] = d;
      bi[s] = j;
    } else if (shift) {
      bd[s] = bd[s - 1];
      bi[s] = bi[s - 1];
    }
  }
  if (bd[0] > d) {   // still the old slot 0 (moved to slot 1): d is the new smallest
    bd[0] = d;
    bi[0] = j;
  }
}

template <int KK>
__global__ void __launch_bounds__(PK_QTILE) point_knn_kernel(const float* __restrict__ data, long long T,
                                                             int stride, const int64_t* __restrict__ off,
                                                             int S, int K, int32_t* __restrict__ idx,
                                                             float* __restrict__ dist) {
  __shared__ float4 cand[PK_CTILE];
  const float NEG_INF = __int_as_float(0xff800000), POS_INF = __int_as_float(0x7f800000);
  for (int s = blockIdx.y; s < S; s += gridDim.y) {
    long long r0;
    int P;
    pk_range(off, s, T, r0, P);
    const int tiles = (P + PK_QTILE - 1) / PK_QTILE;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
      const int q = t * PK_QTILE + threadIdx.x;
      const bool active = q < P;
      float qx = 0.f, qy = 0.f, qz = 0.f;
      if (active) {
        const float* p = data + (r0 + q) * stride;
        qx = p[0];
        qy = p[1];
        qz = p[2];
      }
      float bd[KK];
      int bi[KK];
#pragma unroll
      for (int i = 0; i < KK; ++i) {
        bd[i] = i < KK - K ? NEG_INF : POS_INF;
        bi[i] = -1;
      }
      for (int c0 = 0; c0 < P; c0 += PK_CTILE) {
        const int n = P - c0 < PK_CTILE ? P - c0 : PK_CTILE;
        __syncthreads();   // the previous tile is consumed
        for (int i = threadIdx.x; i < n; i += PK_QTILE) {
          const float* p = data + (r0 + c0 + i) * stride;
          cand[i] = make_float4(p[0], p[1], p[2], 0.f);
        }
        __syncthreads();
        if (active) {
          int i = 0;
          for (; i + 4 <= n; i += 4) {
            const float4 a = cand[i], b = cand[i + 1], c = cand[i + 2], e = cand[i + 3];
            const float d0 = pk_dist(qx, qy, qz, a.x, a.y, a.z);
            const float d1 = pk_dist(qx, qy, qz, b.x, b.y, b.z);
            const float d2 = pk_dist(qx, qy, qz, c.x, c.y, c.z);
            const float d3 = pk_dist(qx, qy, qz, e.x, e.y, e.z);
            // fminf drops NaN, which never enters on this pass anyway
            if (fminf(fminf(d0, d1), fminf(d2, d3)) < bd[KK - 1]) {
              if (d0 < bd[KK - 1]) pk_insert(bd, bi, d0, c0 + i);
              if (d1 < bd[KK - 1]) pk_insert(bd, bi, d1, c0 + i + 1);
              if (d2 < bd[KK - 1]) pk_insert(bd, bi, d2, c0 + i + 2);
              if (d3 < bd[KK - 1]) pk_insert(bd, bi, d3, c0 + i + 3);
            }
          }
          for (; i < n; ++i) {
            const float4 a = cand[i];
            const float d = pk_dist(qx, qy, qz, a.x, a.y, a.z);
            if (d < bd[KK - 1]) pk_insert(bd, bi, d, c0 + i);
          }
        }
      }
      if (!active) continue;
      // fill: the +inf candidates, then the NaN ones, in index order, up to min(P, K) slots
      int filled = 0;
#pragma unroll
      for (int i = 0; i < KK; ++i) filled += bi[i] >= 0;
      const int want = P < K ? P : K;
      for (int pass = 0; pass < 2 && filled < want; ++pass) {
        for (int j = 0; j < P && filled < want; ++j) {
          const float* p = data + (r0 + j) * stride;
          const float d = pk_dist(qx, qy, qz, p[0], p[1], p[2]);
          if (pass == 0 ? d == POS_INF : d != d) {
            const int slot = KK - K + filled;
#pragma unroll
            for (int i = 0; i < KK; ++i)   // register slots: no dynamic index
              if (i == slot) {
                bd[i] = d;
                bi[i] = j;
              }
            ++filled;
          }
        }
      }
      int32_t* io = idx + (r0 + q) * K;
      float* dout = dist ? dist + (r0 + q) * K : nullptr;
#pragma unroll
      for (int i = 0; i < KK; ++i) {
        if (i < KK - K) continue;
        io[i - (KK - K)] = bi[i];
        if (dout) dout[i - (KK - K)] = bi[i] < 0 ? POS_INF : bd[i];
      }
    }
  }
}

// ---- normals ----------------------------------------------------------------------------------------
// Cloud centroid in fp64, in a fixed order: thread t of the CTA sums rows t, t+256, t+512, ...
// sequentially from +0, then s[i] += s[i+h] for h = 128, 64, .., 1; c = s[0] / P (NaN when P == 0).
__global__ void __launch_bounds__(PC_THREADS) point_centroid_kernel(const float* __restrict__ data, long long T,
                                                                   int stride, const int64_t* __restrict__ off,
                                                                   int S, double* __restrict__ cen) {
  __shared__ double acc[3][PC_THREADS];
  for (int s = blockIdx.x; s < S; s += gridDim.x) {
    long long r0;
    int P;
    pk_range(off, s, T, r0, P);
    double x = 0.0, y = 0.0, z = 0.0;
    for (int i = threadIdx.x; i < P; i += PC_THREADS) {
      const float* p = data + (r0 + i) * stride;
      x = __dadd_rn(x, static_cast<double>(p[0]));
      y = __dadd_rn(y, static_cast<double>(p[1]));
      z = __dadd_rn(z, static_cast<double>(p[2]));
    }
    acc[0][threadIdx.x] = x;
    acc[1][threadIdx.x] = y;
    acc[2][threadIdx.x] = z;
    __syncthreads();
    for (int h = PC_THREADS / 2; h > 0; h >>= 1) {
      if (threadIdx.x < h)
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c][threadIdx.x] = __dadd_rn(acc[c][threadIdx.x], acc[c][threadIdx.x + h]);
      __syncthreads();
    }
    if (threadIdx.x < 3) cen[3 * s + threadIdx.x] = __ddiv_rn(acc[threadIdx.x][0], static_cast<double>(P));
    __syncthreads();   // acc is reused by the next cloud of this CTA
  }
}

// Eigen-decomposition of the symmetric 3x3 a (upper triangle used, destroyed) by cyclic Jacobi:
// w the eigenvalues, v the eigenvectors as columns.
__device__ __forceinline__ void jacobi3(double a[3][3], double w[3], double v[3][3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) v[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 32; ++sweep) {
    const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
    const double diag = fabs(a[0][0]) + fabs(a[1][1]) + fabs(a[2][2]);
    if (off == 0.0 || off <= 0x1.0p-60 * diag) break;
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      const double apq = a[p][q];
      if (apq == 0.0) continue;
      const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
      const double at = fabs(theta);
      // tan of the rotation angle, the smaller root; 1/(2 theta) where theta^2 would overflow
      double t = at > 1e150 ? 0.5 / at : 1.0 / (at + sqrt(at * at + 1.0));
      if (theta < 0.0) t = -t;
      const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c, tau = sn / (1.0 + c);
      a[p][p] -= t * apq;
      a[q][q] += t * apq;
      a[p][q] = 0.0;
      const int r = 3 - p - q;   // the third index
      const double arp = p < r ? a[p][r] : a[r][p], arq = q < r ? a[q][r] : a[r][q];
      const double nrp = arp - sn * (arq + tau * arp), nrq = arq + sn * (arp - tau * arq);
      if (p < r) a[p][r] = nrp; else a[r][p] = nrp;
      if (q < r) a[q][r] = nrq; else a[r][q] = nrq;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double vp = v[k][p], vq = v[k][q];
        v[k][p] = vp - sn * (vq + tau * vp);
        v[k][q] = vq + sn * (vp - tau * vq);
      }
    }
  }
  w[0] = a[0][0];
  w[1] = a[1][1];
  w[2] = a[2][2];
}

struct NormalArgs {
  const float* data;
  const int64_t* off;
  const int32_t* idx;
  const float* view;
  const double* cen;
  float* normals;
  float* curv;
  long long T;
  int stride, nstride, S, K, orient;
};

__global__ void __launch_bounds__(PN_THREADS) point_normals_kernel(NormalArgs a) {
  const float QNAN = __int_as_float(0x7fc00000);
  for (int s = blockIdx.y; s < a.S; s += gridDim.y) {
    long long r0;
    int P;
    pk_range(a.off, s, a.T, r0, P);
    const int tiles = (P + PN_THREADS - 1) / PN_THREADS;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
      const int q = t * PN_THREADS + threadIdx.x;
      if (q >= P) continue;
      const long long row = r0 + q;
      const int32_t* nb = a.idx + row * a.K;
      // pass 1: the mean of the valid neighbours (indices in [0, P)), in slot order
      int n = 0;
      bool finite = true;
      double mx = 0.0, my = 0.0, mz = 0.0;
      for (int k = 0; k < a.K; ++k) {
        const int j = nb[k];
        if (j < 0 || j >= P) continue;
        const float* p = a.data + (r0 + j) * a.stride;
        const float x = p[0], y = p[1], z = p[2];
        finite &= isfinite(x) && isfinite(y) && isfinite(z);
        mx = __dadd_rn(mx, static_cast<double>(x));
        my = __dadd_rn(my, static_cast<double>(y));
        mz = __dadd_rn(mz, static_cast<double>(z));
        ++n;
      }
      float nrm[3] = {0.f, 0.f, 0.f};
      float curv = QNAN;
      if (n >= 3 && finite) {
        const double dn = static_cast<double>(n);
        mx = __ddiv_rn(mx, dn);
        my = __ddiv_rn(my, dn);
        mz = __ddiv_rn(mz, dn);
        // pass 2: the centred covariance, in slot order
        double cxx = 0.0, cxy = 0.0, cxz = 0.0, cyy = 0.0, cyz = 0.0, czz = 0.0;
        for (int k = 0; k < a.K; ++k) {
          const int j = nb[k];
          if (j < 0 || j >= P) continue;
          const float* p = a.data + (r0 + j) * a.stride;
          const double dx = __dsub_rn(p[0], mx), dy = __dsub_rn(p[1], my), dz = __dsub_rn(p[2], mz);
          cxx = __dadd_rn(cxx, __dmul_rn(dx, dx));
          cxy = __dadd_rn(cxy, __dmul_rn(dx, dy));
          cxz = __dadd_rn(cxz, __dmul_rn(dx, dz));
          cyy = __dadd_rn(cyy, __dmul_rn(dy, dy));
          cyz = __dadd_rn(cyz, __dmul_rn(dy, dz));
          czz = __dadd_rn(czz, __dmul_rn(dz, dz));
        }
        double m[3][3] = {{__ddiv_rn(cxx, dn), __ddiv_rn(cxy, dn), __ddiv_rn(cxz, dn)},
                          {0.0, __ddiv_rn(cyy, dn), __ddiv_rn(cyz, dn)},
                          {0.0, 0.0, __ddiv_rn(czz, dn)}};
        const double trace = __dadd_rn(__dadd_rn(m[0][0], m[1][1]), m[2][2]);
        if (trace > 0.0 && isfinite(trace)) {
          double w[3], v[3][3];
          jacobi3(m, w, v);
          // smallest eigenvalue, lowest column on ties (selects, not dynamic register indices)
          const int i0 = w[1] < w[0] ? (w[2] < w[1] ? 2 : 1) : (w[2] < w[0] ? 2 : 0);
          const double wa = i0 == 0 ? w[1] : w[0], wb = i0 == 2 ? w[1] : w[2];   // the other two
          const double l0 = fmax(i0 == 0 ? w[0] : (i0 == 1 ? w[1] : w[2]), 0.0);
          const double l1 = fmax(fmin(wa, wb), 0.0), l2 = fmax(fmax(wa, wb), 0.0);
          const double sum = (l0 + l1) + l2;
          // collinear (or coincident) neighbours: the second-smallest eigenvalue vanishes against
          // the spread, and the plane is not defined
          if (l1 > 0x1.0p-40 * sum) {
            const double ex = i0 == 0 ? v[0][0] : (i0 == 1 ? v[0][1] : v[0][2]);
            const double ey = i0 == 0 ? v[1][0] : (i0 == 1 ? v[1][1] : v[1][2]);
            const double ez = i0 == 0 ? v[2][0] : (i0 == 1 ? v[2][1] : v[2][2]);
            const double len = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)),
                                                    __dmul_rn(ez, ez)));
            nrm[0] = __double2float_rn(__ddiv_rn(ex, len));
            nrm[1] = __double2float_rn(__ddiv_rn(ey, len));
            nrm[2] = __double2float_rn(__ddiv_rn(ez, len));
            curv = static_cast<float>(l0 / sum);
            // canonical sign: the first component of largest magnitude is positive
            int c = 0;
            if (fabsf(nrm[1]) > fabsf(nrm[c])) c = 1;
            if (fabsf(nrm[2]) > fabsf(nrm[c])) c = 2;
            bool flip = nrm[c] < 0.f;
            if (a.orient != SONET_NORMALS_CANONICAL) {
              const float* p = a.data + row * a.stride;
              double rx, ry, rz;
              if (a.orient == SONET_NORMALS_AWAY_FROM_CENTROID) {
                const double* cc = a.cen + 3 * s;
                rx = __dsub_rn(p[0], cc[0]);
                ry = __dsub_rn(p[1], cc[1]);
                rz = __dsub_rn(p[2], cc[2]);
              } else {
                const float* vp = a.view + 3 * s;
                rx = __dsub_rn(vp[0], p[0]);
                ry = __dsub_rn(vp[1], p[1]);
                rz = __dsub_rn(vp[2], p[2]);
              }
              const double sg = flip ? -1.0 : 1.0;   // the dot with the canonical normal
              const double dot = __dadd_rn(__dadd_rn(__dmul_rn(sg * nrm[0], rx), __dmul_rn(sg * nrm[1], ry)),
                                           __dmul_rn(sg * nrm[2], rz));
              if (dot < 0.0) flip = !flip;
            }
            if (flip) {
              nrm[0] = -nrm[0];
              nrm[1] = -nrm[1];
              nrm[2] = -nrm[2];
            }
          }
        }
      }
      float* o = a.normals + row * a.nstride;
      o[0] = nrm[0];
      o[1] = nrm[1];
      o[2] = nrm[2];
      if (a.curv) a.curv[row] = curv;
    }
  }
}

// 2-D grid over (tiles of a cloud, clouds): about twice the mean tile count per cloud along x (idle
// blocks of short clouds exit at once), every cloud its own row of blocks along y.
static dim3 pk_grid(long long T, int S, int tile) {
  const long long mean = (T + static_cast<long long>(tile) * S - 1) / (static_cast<long long>(tile) * S);
  long long x = 2 * mean;
  x = x < 1 ? 1 : (x > 65535 ? 65535 : x);
  const long long y = S < 65535 ? S : 65535;
  return dim3(static_cast<unsigned>(x), static_cast<unsigned>(y));
}

static size_t pn_scratch(int S) { return (sizeof(double) * 3 * static_cast<size_t>(S) + 255) & ~static_cast<size_t>(255); }

// ---- orientation: signs propagated along each component's minimum spanning tree ------------------
// Borůvka over the k-NN graph of every cloud at once, the parity carried through the union. Per
// vertex, node = (root row << 1) | parity of its sign relative to the root. A round: every directed
// entry (u -> v) across two components offers its key to both roots, first the ordered weight bits
// (atomicMin), then the cloud-local pair (lo << 24) | hi among the entries that reach that weight;
// every root hooks to the root at the other end of its least edge (a mutual pair keeps the lower
// row), the hooked roots pointer-jump to their tree's root XOR-ing the parities, and every vertex
// rebases onto it. Edges are strictly ordered, so the least edges form a forest: each component with
// an outgoing edge merges, and ceil(log2(max_points)) rounds join every connected component. Then
// each component takes its anchor (least distance key, then least cloud-local index) and every
// vertex's sign is its anchor's flip XOR its parity relative to the anchor.
constexpr int PO_THREADS = 256;
constexpr int PO_MAX_ROUNDS = SONET_POINT_ORIENT_MAX_ROUNDS;   // ceil(log2(max_points)), max_points < 2^24
constexpr unsigned long long PO_NONE = ~0ull;

struct OrientArgs {
  const float* data;
  const int64_t* off;
  const int32_t* idx;
  const float* view;
  const double* cen;
  float* normals;
  int32_t* comp;
  int* merged;                 // [PO_MAX_ROUNDS]: round r hooked at least one root
  int32_t* cid;                // [T] the cloud of a vertex, -1 for a non-vertex
  unsigned long long* node;    // [T] (root row << 1) | parity relative to the root
  unsigned long long* link;    // [T] a root's (parent row << 1) | parity within a round
  unsigned int* bw;            // [T] a root's least ordered weight key offered this round
  unsigned long long* be;      // [T] a root's least (lo << 24) | hi among the entries at bw
  unsigned long long* ak;      // [T] a root's least anchor distance key
  unsigned int* ai;            // [T] a root's least (local << 1) | flip among the vertices at ak
  long long T;
  int stride, nstride, S, K, max_points, anchor;
};

// The pointer jumps read links other threads are rewriting: one 64-bit word holds parent and parity,
// so any value read is a consistent ancestor, and relaxed device-scope accesses keep them uncached.
__device__ __forceinline__ unsigned long long po_load(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void po_store(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ bool po_active(const int* merged, int round) {
  return round == 0 || *reinterpret_cast<const volatile int*>(merged + round - 1) != 0;
}

// (nx_u*nx_v + ny_u*ny_v) + nz_u*nz_v in fp64, explicitly rounded
__device__ __forceinline__ double po_dot(const float* a, const float* b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

// w = fp32(1 - |dot|) as an unsigned key in float order (-0 made +0 first; w is never NaN)
__device__ __forceinline__ unsigned po_wkey(double dot) {
  const unsigned b = __float_as_uint(__fadd_rn(__double2float_rn(__dsub_rn(1.0, fabs(dot))), 0.f));
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// The anchor's distance key of vertex g (least wins) and its reference vector: the squared fp64
// distance to the centroid (farthest first) or to view[s] (nearest first); NaN last.
__device__ __forceinline__ unsigned long long po_akey(const OrientArgs& a, long long g, int s, double& rx,
                                                      double& ry, double& rz) {
  const float* p = a.data + g * a.stride;
  if (a.anchor == SONET_NORMALS_AWAY_FROM_CENTROID) {
    const double* c = a.cen + 3 * s;
    rx = __dsub_rn(p[0], c[0]);
    ry = __dsub_rn(p[1], c[1]);
    rz = __dsub_rn(p[2], c[2]);
  } else {
    const float* v = a.view + 3 * s;
    rx = __dsub_rn(v[0], p[0]);
    ry = __dsub_rn(v[1], p[1]);
    rz = __dsub_rn(v[2], p[2]);
  }
  const double d = __dadd_rn(__dadd_rn(__dmul_rn(rx, rx), __dmul_rn(ry, ry)), __dmul_rn(rz, rz));
  const unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(d));   // d >= +0
  if (d != d) return PO_NONE;
  return a.anchor == SONET_NORMALS_AWAY_FROM_CENTROID ? 0x7ff0000000000000ull - bits : bits;
}

#define PO_ROWS(g, n)                                                                   \
  for (long long g = static_cast<long long>(blockIdx.x) * PO_THREADS + threadIdx.x; g < (n); \
       g += static_cast<long long>(gridDim.x) * PO_THREADS)

// Each row's cloud (ragged_find) and vertex test; every root starts alone with parity 0.
__global__ void __launch_bounds__(PO_THREADS) orient_init_kernel(OrientArgs a) {
  if (blockIdx.x == 0 && threadIdx.x < PO_MAX_ROUNDS) a.merged[threadIdx.x] = 0;
  PO_ROWS(g, a.T) {
    long long lo, hi;
    const int s = ragged_find(a.off, a.S, a.T, g, lo, hi);
    bool vert = g >= lo && g < hi && g - lo < a.max_points;
    if (vert) {
      const float* p = a.data + g * a.stride;
      const float* n = a.normals + g * a.nstride;
      vert = isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]) && isfinite(n[0]) && isfinite(n[1]) &&
             isfinite(n[2]) && (n[0] != 0.f || n[1] != 0.f || n[2] != 0.f);
    }
    a.cid[g] = vert ? s : -1;
    a.node[g] = static_cast<unsigned long long>(g) << 1;
    a.bw[g] = ~0u;
    a.be[g] = PO_NONE;
    a.ak[g] = PO_NONE;
    a.ai[g] = ~0u;
  }
}

// PASS 0 offers the weight keys, PASS 1 the pairs of the entries at their root's least weight.
template <int PASS>
__global__ void __launch_bounds__(PO_THREADS) orient_offer_kernel(OrientArgs a, int round) {
  if (!po_active(a.merged, round)) return;
  PO_ROWS(e, a.T * a.K) {
    const long long u = e / a.K;
    const int s = a.cid[u];
    if (s < 0) continue;
    const int j = a.idx[e];
    long long lo, hi;
    ragged_range(a.off, s, a.T, lo, hi);
    const long long ul = u - lo;
    if (j < 0 || j >= hi - lo || j == ul || a.cid[lo + j] != s) continue;
    const long long ru = static_cast<long long>(a.node[u] >> 1), rv = static_cast<long long>(a.node[lo + j] >> 1);
    if (ru == rv) continue;
    const unsigned key = po_wkey(po_dot(a.normals + u * a.nstride, a.normals + (lo + j) * a.nstride));
    if (PASS == 0) {
      atomicMin(a.bw + ru, key);
      atomicMin(a.bw + rv, key);
    } else {
      const unsigned long long uj = static_cast<unsigned long long>(j), uu = static_cast<unsigned long long>(ul);
      const unsigned long long pair = uu < uj ? (uu << 24) | uj : (uj << 24) | uu;
      if (a.bw[ru] == key) atomicMin(a.be + ru, pair);
      if (a.bw[rv] == key) atomicMin(a.be + rv, pair);
    }
  }
}

// Every root links to the root across its least edge, with its parity relative to that root.
__global__ void __launch_bounds__(PO_THREADS) orient_hook_kernel(OrientArgs a, int round) {
  if (!po_active(a.merged, round)) return;
  PO_ROWS(g, a.T) {
    const int s = a.cid[g];
    if (s < 0 || static_cast<long long>(a.node[g] >> 1) != g) continue;
    const unsigned long long e = a.be[g];
    unsigned long long l = static_cast<unsigned long long>(g) << 1;
    if (e != PO_NONE) {
      long long lo, hi;
      ragged_range(a.off, s, a.T, lo, hi);
      const long long x = lo + static_cast<long long>(e >> 24), y = lo + static_cast<long long>(e & 0xffffffull);
      const unsigned long long nx = a.node[x], ny = a.node[y];
      const long long other = static_cast<long long>((nx >> 1) == static_cast<unsigned long long>(g) ? ny >> 1 : nx >> 1);
      const unsigned long long flip = po_dot(a.normals + x * a.nstride, a.normals + y * a.nstride) < 0.0;
      if (!(g < other && a.be[other] == e)) {   // a mutual pair keeps the lower row as root
        l = (static_cast<unsigned long long>(other) << 1) | (((nx ^ ny) & 1ull) ^ flip);
        a.merged[round] = 1;
      }
    }
    a.link[g] = l;
  }
}

// Every hooked root walks to its tree's root. Each step moves at least one link closer, and a tree
// holds fewer than max_points roots, so max_points steps always reach it.
__global__ void __launch_bounds__(PO_THREADS) orient_jump_kernel(OrientArgs a, int round) {
  if (!po_active(a.merged, round + 1)) return;
  PO_ROWS(g, a.T) {
    if (a.cid[g] < 0 || static_cast<long long>(a.node[g] >> 1) != g) continue;
    unsigned long long l = po_load(a.link + g);
    for (int step = 0; step < a.max_points; ++step) {
      const unsigned long long p = l >> 1;
      if (p == static_cast<unsigned long long>(g)) break;
      const unsigned long long lp = po_load(a.link + p);
      if ((lp >> 1) == p) break;
      l = (lp & ~1ull) | ((l ^ lp) & 1ull);
      po_store(a.link + g, l);
    }
  }
}

// Every vertex moves onto its root's root; the per-root offers start over.
__global__ void __launch_bounds__(PO_THREADS) orient_rebase_kernel(OrientArgs a, int round) {
  if (!po_active(a.merged, round + 1)) return;
  PO_ROWS(g, a.T) {
    if (a.cid[g] < 0) continue;
    const unsigned long long nd = a.node[g], l = a.link[nd >> 1];
    a.node[g] = (l & ~1ull) | ((nd ^ l) & 1ull);
    a.bw[g] = ~0u;
    a.be[g] = PO_NONE;
  }
}

// PASS 0: each component's least distance key; PASS 1: among its vertices at that key, the least
// (local index << 1) | (anchor flip XOR parity relative to the root).
template <int PASS>
__global__ void __launch_bounds__(PO_THREADS) orient_anchor_kernel(OrientArgs a) {
  PO_ROWS(g, a.T) {
    const int s = a.cid[g];
    if (s < 0) continue;
    double rx, ry, rz;
    const unsigned long long key = po_akey(a, g, s, rx, ry, rz), nd = a.node[g];
    if (PASS == 0) {
      atomicMin(a.ak + (nd >> 1), key);
    } else if (a.ak[nd >> 1] == key) {
      const float* n = a.normals + g * a.nstride;
      const double dot = __dadd_rn(__dadd_rn(__dmul_rn(n[0], rx), __dmul_rn(n[1], ry)), __dmul_rn(n[2], rz));
      long long lo, hi;
      ragged_range(a.off, s, a.T, lo, hi);
      atomicMin(a.ai + (nd >> 1), (static_cast<unsigned>(g - lo) << 1) | ((dot < 0.0) ^ static_cast<unsigned>(nd & 1ull)));
    }
  }
}

__global__ void __launch_bounds__(PO_THREADS) orient_write_kernel(OrientArgs a) {
  PO_ROWS(g, a.T) {
    if (a.cid[g] < 0) {
      if (a.comp) a.comp[g] = -1;
      continue;
    }
    const unsigned long long nd = a.node[g];
    const unsigned w = a.ai[nd >> 1];
    if ((w ^ static_cast<unsigned>(nd)) & 1u) {
      float* n = a.normals + g * a.nstride;
      n[0] = -n[0];
      n[1] = -n[1];
      n[2] = -n[2];
    }
    if (a.comp) a.comp[g] = static_cast<int32_t>(w >> 1);
  }
}
#undef PO_ROWS

static int po_rounds(int max_points) { return max_points <= 1 ? 0 : 32 - __builtin_clz(static_cast<unsigned>(max_points - 1)); }

static size_t al256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }

// flags | centroids [S, 3] f64 | node, link, be, ak [T] u64 | cid, bw, ai [T] 32-bit
static size_t po_scratch(long long T, int S) {
  if (S == 0) return 0;
  const size_t t = static_cast<size_t>(T);
  return al256(sizeof(int) * PO_MAX_ROUNDS) + pn_scratch(S) + 4 * al256(8 * t) + 3 * al256(4 * t);
}

static unsigned po_blocks(long long n) {
  const long long cap = 16LL * sm_count(), b = (n + PO_THREADS - 1) / PO_THREADS;
  return static_cast<unsigned>(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace sonet

extern "C" int sonet_point_knn_f32(const float* data, long long T, int stride, const int64_t* offsets, int S,
                                   int K, int32_t* idx, float* dist, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(S >= 0, "point_knn: S=%d must be >= 0", S);
  SONET_REQUIRE(T >= 0, "point_knn: T=%lld must be >= 0", T);
  SONET_REQUIRE(stride >= 3, "point_knn: stride=%d must be >= 3", stride);
  SONET_REQUIRE(K >= 3 && K <= SONET_POINT_KNN_MAX_K, "point_knn: K=%d outside [3, %d]", K,
                SONET_POINT_KNN_MAX_K);
  SONET_REQUIRE(offsets && idx, "point_knn: offsets and idx must not be null");
  SONET_REQUIRE(data || T == 0, "point_knn: data must not be null (T=%lld)", T);
  if (S == 0) return SONET_OK;
  const dim3 grid = pk_grid(T, S, PK_QTILE);
  cudaStream_t st = as_stream(stream);
  if (K <= 4) point_knn_kernel<4><<<grid, PK_QTILE, 0, st>>>(data, T, stride, offsets, S, K, idx, dist);
  else if (K <= 8) point_knn_kernel<8><<<grid, PK_QTILE, 0, st>>>(data, T, stride, offsets, S, K, idx, dist);
  else if (K <= 16) point_knn_kernel<16><<<grid, PK_QTILE, 0, st>>>(data, T, stride, offsets, S, K, idx, dist);
  else point_knn_kernel<32><<<grid, PK_QTILE, 0, st>>>(data, T, stride, offsets, S, K, idx, dist);
  return check_launch("point_knn");
}

extern "C" long long sonet_point_normals_scratch_bytes(int S) {
  using namespace sonet;
  SONET_REQUIRE(S >= 0, "point_normals_scratch_bytes: S=%d must be >= 0", S);
  return static_cast<long long>(pn_scratch(S));
}

extern "C" int sonet_point_normals_f32(const float* data, long long T, int stride, const int64_t* offsets,
                                       int S, const int32_t* idx, int K, int orient, const float* view,
                                       void* scratch, long long scratch_bytes, float* normals,
                                       int normal_stride, float* curvature, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(S >= 0, "point_normals: S=%d must be >= 0", S);
  SONET_REQUIRE(T >= 0, "point_normals: T=%lld must be >= 0", T);
  SONET_REQUIRE(stride >= 3, "point_normals: stride=%d must be >= 3", stride);
  SONET_REQUIRE(normal_stride >= 3, "point_normals: normal_stride=%d must be >= 3", normal_stride);
  SONET_REQUIRE(K >= 3 && K <= SONET_POINT_KNN_MAX_K, "point_normals: K=%d outside [3, %d]", K,
                SONET_POINT_KNN_MAX_K);
  SONET_REQUIRE(orient == SONET_NORMALS_CANONICAL || orient == SONET_NORMALS_AWAY_FROM_CENTROID ||
                    orient == SONET_NORMALS_TOWARD_VIEWPOINT,
                "point_normals: orientation code %d is not SONET_NORMALS_CANONICAL (0), "
                "_AWAY_FROM_CENTROID (1) or _TOWARD_VIEWPOINT (2)", orient);
  SONET_REQUIRE(offsets && normals, "point_normals: offsets and normals must not be null");
  SONET_REQUIRE((data && idx) || T == 0, "point_normals: data and idx must not be null (T=%lld)", T);
  SONET_REQUIRE(view || orient != SONET_NORMALS_TOWARD_VIEWPOINT,
                "point_normals: view must not be null with SONET_NORMALS_TOWARD_VIEWPOINT");
  const bool need_cen = orient == SONET_NORMALS_AWAY_FROM_CENTROID;
  SONET_REQUIRE(!need_cen || (scratch && scratch_bytes >= static_cast<long long>(pn_scratch(S))),
                "point_normals: SONET_NORMALS_AWAY_FROM_CENTROID needs %lld bytes of scratch, got %lld%s",
                static_cast<long long>(pn_scratch(S)), scratch_bytes, scratch ? "" : " (null)");
  SONET_REQUIRE(!need_cen || (reinterpret_cast<uintptr_t>(scratch) & 255u) == 0,
                "point_normals: scratch must be 256-byte aligned");
  if (S == 0) return SONET_OK;
  cudaStream_t st = as_stream(stream);
  NormalArgs a;
  a.data = data;
  a.off = offsets;
  a.idx = idx;
  a.view = view;
  a.cen = static_cast<const double*>(scratch);
  a.normals = normals;
  a.curv = curvature;
  a.T = T;
  a.stride = stride;
  a.nstride = normal_stride;
  a.S = S;
  a.K = K;
  a.orient = orient;
  if (need_cen) {
    point_centroid_kernel<<<S < 65535 ? S : 65535, PC_THREADS, 0, st>>>(data, T, stride, offsets, S,
                                                                         static_cast<double*>(scratch));
    const int rc = check_launch("point_normals (centroids)");
    if (rc != SONET_OK) return rc;
  }
  point_normals_kernel<<<pk_grid(T, S, PN_THREADS), PN_THREADS, 0, st>>>(a);
  return check_launch("point_normals");
}

extern "C" long long sonet_point_normals_orient_scratch_bytes(long long T, int S) {
  using namespace sonet;
  SONET_REQUIRE(T >= 0 && S >= 0, "point_normals_orient_scratch_bytes: T=%lld and S=%d must be >= 0", T, S);
  return static_cast<long long>(po_scratch(T, S));
}

extern "C" int sonet_point_normals_orient_f32(const float* data, long long T, int stride, const int64_t* offsets,
                                              int S, int max_points, const int32_t* idx, int K, int anchor,
                                              const float* view, void* scratch, long long scratch_bytes,
                                              float* normals, int normal_stride, int32_t* component,
                                              sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(S >= 0, "point_normals_orient: S=%d must be >= 0", S);
  SONET_REQUIRE(T >= 0, "point_normals_orient: T=%lld must be >= 0", T);
  SONET_REQUIRE(stride >= 3, "point_normals_orient: stride=%d must be >= 3", stride);
  SONET_REQUIRE(normal_stride >= 3, "point_normals_orient: normal_stride=%d must be >= 3", normal_stride);
  SONET_REQUIRE(K >= 1 && K <= SONET_POINT_KNN_MAX_K, "point_normals_orient: K=%d outside [1, %d]", K,
                SONET_POINT_KNN_MAX_K);
  SONET_REQUIRE(max_points >= 0 && max_points < SONET_POINT_ORIENT_MAX_POINTS,
                "point_normals_orient: max_points=%d outside [0, %d)", max_points, SONET_POINT_ORIENT_MAX_POINTS);
  SONET_REQUIRE(anchor == SONET_NORMALS_AWAY_FROM_CENTROID || anchor == SONET_NORMALS_TOWARD_VIEWPOINT,
                "point_normals_orient: anchor code %d is not SONET_NORMALS_AWAY_FROM_CENTROID (1) or "
                "_TOWARD_VIEWPOINT (2)", anchor);
  SONET_REQUIRE(offsets && normals, "point_normals_orient: offsets and normals must not be null");
  SONET_REQUIRE((data && idx) || T == 0, "point_normals_orient: data and idx must not be null (T=%lld)", T);
  SONET_REQUIRE(view || anchor != SONET_NORMALS_TOWARD_VIEWPOINT,
                "point_normals_orient: view must not be null with SONET_NORMALS_TOWARD_VIEWPOINT");
  const long long need = static_cast<long long>(po_scratch(T, S));
  SONET_REQUIRE(need == 0 || (scratch && scratch_bytes >= need),
                "point_normals_orient: needs %lld bytes of scratch, got %lld%s", need, scratch_bytes,
                scratch ? "" : " (null)");
  SONET_REQUIRE(need == 0 || (reinterpret_cast<uintptr_t>(scratch) & 255u) == 0,
                "point_normals_orient: scratch must be 256-byte aligned");
  if (S == 0) return SONET_OK;
  cudaStream_t st = as_stream(stream);
  char* p = static_cast<char*>(scratch);
  const size_t t = static_cast<size_t>(T);
  auto take = [&](size_t bytes) {
    char* r = p;
    p += al256(bytes);
    return r;
  };
  OrientArgs a;
  a.merged = reinterpret_cast<int*>(take(sizeof(int) * PO_MAX_ROUNDS));
  double* cen = reinterpret_cast<double*>(take(sizeof(double) * 3 * static_cast<size_t>(S)));
  a.node = reinterpret_cast<unsigned long long*>(take(8 * t));
  a.link = reinterpret_cast<unsigned long long*>(take(8 * t));
  a.be = reinterpret_cast<unsigned long long*>(take(8 * t));
  a.ak = reinterpret_cast<unsigned long long*>(take(8 * t));
  a.cid = reinterpret_cast<int32_t*>(take(4 * t));
  a.bw = reinterpret_cast<unsigned int*>(take(4 * t));
  a.ai = reinterpret_cast<unsigned int*>(take(4 * t));
  a.data = data;
  a.off = offsets;
  a.idx = idx;
  a.view = view;
  a.cen = cen;
  a.normals = normals;
  a.comp = component;
  a.T = T;
  a.stride = stride;
  a.nstride = normal_stride;
  a.S = S;
  a.K = K;
  a.max_points = max_points;
  a.anchor = anchor;
  if (anchor == SONET_NORMALS_AWAY_FROM_CENTROID) {
    point_centroid_kernel<<<S < 65535 ? S : 65535, PC_THREADS, 0, st>>>(data, T, stride, offsets, S, cen);
    const int rc = check_launch("point_normals_orient (centroids)");
    if (rc != SONET_OK) return rc;
  }
  const unsigned rows = po_blocks(T), entries = po_blocks(T * K);
  orient_init_kernel<<<rows, PO_THREADS, 0, st>>>(a);
  int rc = check_launch("point_normals_orient (init)");
  for (int r = 0; r < po_rounds(max_points) && rc == SONET_OK; ++r) {
    orient_offer_kernel<0><<<entries, PO_THREADS, 0, st>>>(a, r);
    orient_offer_kernel<1><<<entries, PO_THREADS, 0, st>>>(a, r);
    orient_hook_kernel<<<rows, PO_THREADS, 0, st>>>(a, r);
    orient_jump_kernel<<<rows, PO_THREADS, 0, st>>>(a, r);
    orient_rebase_kernel<<<rows, PO_THREADS, 0, st>>>(a, r);
    rc = check_launch("point_normals_orient (round)");
  }
  if (rc != SONET_OK) return rc;
  orient_anchor_kernel<0><<<rows, PO_THREADS, 0, st>>>(a);
  orient_anchor_kernel<1><<<rows, PO_THREADS, 0, st>>>(a);
  orient_write_kernel<<<rows, PO_THREADS, 0, st>>>(a);
  return check_launch("point_normals_orient");
}
