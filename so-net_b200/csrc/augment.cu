// augment.cu — on-device training augmentation of a whole batch (SURVEY.md §8f-3) for sm_90a.
//
// Replaces the per-item numpy pipeline of the reference's loader
// (data/modelnet_shrec_loader.py:218-247 calling data/augmentation.py:52-144): rotation about the
// up axis, small-angle perturbation rotation, per-point jitter of points / normals / SOM nodes,
// random scale and random shift — for every cloud of the batch in ONE launch, instead of six
// numpy passes per item in the DataLoader workers.
//
// Numerics follow the loader: it computes in float64 (np.dot with a float64 matrix promotes the
// float32 cloud) and casts to float32 once at the end (loader :250-256). Every step here is fp64
// with separate multiply/add roundings in the reference's order, one final cvt.rn.f32.f64:
//     v  = v . R1            (rotate_point_cloud_with_normal_som, augmentation.py:52-76)
//     v  = v . R2            (rotate_perturbation_..._with_normal_som, :104-129)
//     v += clip(sigma * g, -clip, clip)          (jitter_point_cloud, :132-144)
//     v *= scale ; v += shift                    (loader :236-247; the shift skips the normals)
// The Gaussian draws g come either from the caller (host numpy draws: bit-for-bit the loader's
// stream, used by the parity tests) or from an in-kernel counter-based generator
// (Philox4x32-10 + Box-Muller, keyed by seed / cloud / array / point) for production loaders,
// where shipping 11 doubles per point from the host would cost more than the augmentation.
#include <algorithm>

#include "common.cuh"
#include "philox.cuh"

namespace sonet {

// three standard normals for (seed, cloud, array, point)
__device__ __forceinline__ void normal3(unsigned long long seed, uint32_t cloud, uint32_t array,
                                        uint32_t point, double (&g)[3]) {
  uint32_t c[4] = {point, cloud, array, 0x5eedu};
  philox4x32_10(c, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  // Box-Muller on two pairs of uniforms in (0,1]
  const double u0 = (static_cast<double>(c[0]) + 1.0) * (1.0 / 4294967296.0);
  const double u1 = (static_cast<double>(c[1]) + 0.5) * (1.0 / 4294967296.0);
  const double u2 = (static_cast<double>(c[2]) + 1.0) * (1.0 / 4294967296.0);
  const double u3 = (static_cast<double>(c[3]) + 0.5) * (1.0 / 4294967296.0);
  const double r0 = sqrt(-2.0 * log(u0)), r1 = sqrt(-2.0 * log(u2));
  double s0, c0, s1, c1;
  sincospi(2.0 * u1, &s0, &c0);
  sincospi(2.0 * u3, &s1, &c1);
  g[0] = r0 * c0;
  g[1] = r0 * s0;
  g[2] = r1 * c1;
}

struct AugArray {
  const float* in;      // [B,3,P]
  float* out;           // [B,3,P]
  const double* noise;  // [B,P,3] standard-normal draws (nullable)
  int P;
  double sigma, clip;   // jitter (sigma <= 0: none)
  int shift;            // apply the random shift to this array?
};

struct AugParams {
  AugArray a[3];        // points, normals, SOM nodes
  const double* rot1;   // [B,3,3] row-major, v' = v . R (nullable)
  const double* rot2;   // [B,3,3] (nullable)
  const double* scale;  // [B] (nullable)
  const double* shiftv; // [B,3] (nullable)
  unsigned long long seed;
};

__device__ __forceinline__ void rot_apply(const double* __restrict__ R, double (&v)[3]) {
  // (v0*R0j + v1*R1j) + v2*R2j — the k-ascending accumulation of a [N,3]x[3,3] product
  double o[3];
#pragma unroll
  for (int j = 0; j < 3; ++j)
    o[j] = __dadd_rn(__dadd_rn(__dmul_rn(v[0], R[j]), __dmul_rn(v[1], R[3 + j])),
                     __dmul_rn(v[2], R[6 + j]));
  v[0] = o[0]; v[1] = o[1]; v[2] = o[2];
}

// rotations, jitter, scale and shift of one 3-vector v: element n of array `which` of cloud b
__device__ __forceinline__ void augment_vec(const AugParams& p, const AugArray& a, const double (&sR)[2][9],
                                            const double (&sS)[4], int b, int which, int n,
                                            double (&v)[3]) {
  if (p.rot1) rot_apply(sR[0], v);
  if (p.rot2) rot_apply(sR[1], v);
  if (a.sigma > 0.0) {
    double g[3];
    if (a.noise) {
      const double* gp = a.noise + (static_cast<size_t>(b) * a.P + n) * 3;
      g[0] = gp[0]; g[1] = gp[1]; g[2] = gp[2];
    } else {
      normal3(p.seed, static_cast<uint32_t>(b), static_cast<uint32_t>(which),
              static_cast<uint32_t>(n), g);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double j = fmin(fmax(__dmul_rn(a.sigma, g[c]), -a.clip), a.clip);
      v[c] = __dadd_rn(j, v[c]);
    }
  }
  if (p.scale) {
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __dmul_rn(v[c], sS[3]);
  }
  if (p.shiftv && a.shift) {
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __dadd_rn(v[c], sS[c]);
  }
}

// Ragged clouds (sonet_augment_ragged_f32): arrays 0 and 1 are the columns 0-2 and 3-5 of the rows
// offsets[b] .. offsets[b+1] of points [T, ld], written to rows of 6; row n of cloud b is its point n
// (the Philox key's cloud-local index). The SOM nodes stay [B,3,M] planes.
struct AugRows {
  const long long* offsets;
  long long T;
  int ld;
};

// Rows: none, every array [B,3,P] planes; or one AugRows, the ragged points
template <class... Rows>
__global__ void __launch_bounds__(256) augment_kernel(AugParams p, Rows... rows) {
  const int b = blockIdx.y;
  const int which = blockIdx.z;
  const AugArray a = p.a[which];
  if (a.in == nullptr) return;
  __shared__ double sR[2][9];
  __shared__ double sS[4];
  if (threadIdx.x < 9) {
    sR[0][threadIdx.x] = p.rot1 ? p.rot1[static_cast<size_t>(b) * 9 + threadIdx.x] : 0.0;
    sR[1][threadIdx.x] = p.rot2 ? p.rot2[static_cast<size_t>(b) * 9 + threadIdx.x] : 0.0;
  } else if (threadIdx.x < 12) {
    sS[threadIdx.x - 9] = (p.shiftv && a.shift) ? p.shiftv[static_cast<size_t>(b) * 3 + threadIdx.x - 9] : 0.0;
  } else if (threadIdx.x == 12) {
    sS[3] = p.scale ? p.scale[b] : 1.0;
  }
  __syncthreads();
  if constexpr (sizeof...(Rows) == 1) {
    if (which < 2) {
      const AugRows r = (rows, ...);
      long long lo, hi;
      ragged_range(r.offsets, b, r.T, lo, hi);
      const int P = static_cast<int>(hi - lo);
      const float* in = a.in + lo * r.ld;
      float* out = a.out + lo * 6;
      for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < P; n += gridDim.x * blockDim.x) {
        const float* q = in + static_cast<long long>(n) * r.ld;
        double v[3] = {static_cast<double>(q[0]), static_cast<double>(q[1]), static_cast<double>(q[2])};
        augment_vec(p, a, sR, sS, b, which, n, v);
        float* o = out + static_cast<long long>(n) * 6;
        o[0] = static_cast<float>(v[0]);
        o[1] = static_cast<float>(v[1]);
        o[2] = static_cast<float>(v[2]);
      }
      return;
    }
  }
  const int P = a.P;
  const float* in = a.in + static_cast<size_t>(b) * 3 * P;
  float* out = a.out + static_cast<size_t>(b) * 3 * P;
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < P; n += gridDim.x * blockDim.x) {
    double v[3] = {static_cast<double>(in[n]), static_cast<double>(in[P + n]),
                   static_cast<double>(in[2 * P + n])};
    augment_vec(p, a, sR, sS, b, which, n, v);
    out[n] = static_cast<float>(v[0]);
    out[P + n] = static_cast<float>(v[1]);
    out[2 * P + n] = static_cast<float>(v[2]);
  }
}

}  // namespace sonet

extern "C" int sonet_augment_f32(const float* pc, const float* sn, const float* som, int B, int N,
                                 int M, const double* rot1, const double* rot2,
                                 const double* scale, const double* shift, double sigma_pc,
                                 double clip_pc, double sigma_sn, double clip_sn, double sigma_som,
                                 double clip_som, const double* noise_pc, const double* noise_sn,
                                 const double* noise_som, unsigned long long seed, float* pc_out,
                                 float* sn_out, float* som_out, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && N >= 0 && M >= 0, "augment: negative dimension");
  SONET_REQUIRE(B <= 65535, "augment: B=%d exceeds grid limit", B);
  if (B == 0) return SONET_OK;
  SONET_REQUIRE((pc == nullptr) == (pc_out == nullptr) && (sn == nullptr) == (sn_out == nullptr) &&
                    (som == nullptr) == (som_out == nullptr),
                "augment: every input array needs its output (and vice versa)");
  SONET_REQUIRE((sigma_pc <= 0 || clip_pc > 0) && (sigma_sn <= 0 || clip_sn > 0) &&
                    (sigma_som <= 0 || clip_som > 0),
                "augment: clip must be > 0 (data/augmentation.py:140)");
  AugParams p;
  p.a[0] = AugArray{pc, pc_out, noise_pc, N, sigma_pc, clip_pc, 1};
  p.a[1] = AugArray{sn, sn_out, noise_sn, N, sigma_sn, clip_sn, 0};
  p.a[2] = AugArray{som, som_out, noise_som, M, sigma_som, clip_som, 1};
  p.rot1 = rot1;
  p.rot2 = rot2;
  p.scale = scale;
  p.shiftv = shift;
  p.seed = seed;
  const int P = N > M ? N : M;
  if (P == 0) return SONET_OK;
  int gx = (P + 255) / 256;
  if (gx > 64) gx = 64;
  augment_kernel<<<dim3(gx, B, 3), 256, 0, as_stream(stream)>>>(p);
  return check_launch("augment");
}

extern "C" int sonet_augment_ragged_f32(const float* points, long long T, int ld, const long long* offsets,
                                        int B, const float* som, int M, const double* rot1,
                                        const double* rot2, const double* scale, const double* shift,
                                        double sigma_pc, double clip_pc, double sigma_sn, double clip_sn,
                                        double sigma_som, double clip_som, unsigned long long seed,
                                        float* points_out, float* som_out, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 1 && B <= 65535, "augment_ragged: B=%d outside [1, 65535]", B);
  SONET_REQUIRE(T >= 0 && T < (1LL << 31) && M >= 0, "augment_ragged: bad dimension T=%lld M=%d", T, M);
  SONET_REQUIRE(ld >= 6, "augment_ragged: row stride %d below the 6 columns (xyz | normal)", ld);
  SONET_REQUIRE(offsets && (T == 0 || (points && points_out)), "augment_ragged: null pointer");
  SONET_REQUIRE((som == nullptr) == (som_out == nullptr), "augment_ragged: som and som_out go together");
  SONET_REQUIRE(points != points_out || T == 0 || ld == 6,
                "augment_ragged: points_out may alias points only with ld = 6");
  SONET_REQUIRE((sigma_pc <= 0 || clip_pc > 0) && (sigma_sn <= 0 || clip_sn > 0) &&
                    (sigma_som <= 0 || clip_som > 0),
                "augment_ragged: clip must be > 0 (data/augmentation.py:140)");
  AugParams p;
  p.a[0] = AugArray{T ? points : nullptr, points_out, nullptr, 0, sigma_pc, clip_pc, 1};
  p.a[1] = AugArray{T ? points + 3 : nullptr, points_out + 3, nullptr, 0, sigma_sn, clip_sn, 0};
  p.a[2] = AugArray{M ? som : nullptr, som_out, nullptr, M, sigma_som, clip_som, 1};
  p.rot1 = rot1;
  p.rot2 = rot2;
  p.scale = scale;
  p.shiftv = shift;
  p.seed = seed;
  const long long rows = std::max<long long>((T + B - 1) / B, M);
  if (rows == 0) return SONET_OK;
  const int gx = static_cast<int>(std::min<long long>((rows + 255) / 256, 64));
  augment_kernel<<<dim3(gx, B, 3), 256, 0, as_stream(stream)>>>(p, AugRows{offsets, T, ld});
  return check_launch("augment_ragged");
}
