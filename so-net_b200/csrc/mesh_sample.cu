// mesh_sample.cu — area-weighted surface sampling of a batch of triangle meshes, with face normals
// (sm_90a): the point clouds SO-Net's datasets are made of, drawn on the device.
//
// Replaces the reference's MATLAB sampler (data/sampler_matlab/sampler.m): a face is chosen with
// probability proportional to its area, a point uniformly on that face, and the point carries the
// face's unit normal. Every quantity is float64 with explicitly rounded operations (no FMA
// contraction), rounded to float32 once on output, so a numpy float64 restatement that follows
// the order below reproduces the output bit for bit.
//
// Per face (a, b, c its vertices): e1 = b - a, e2 = c - a, n = cross(e1, e2) with each component a
// difference of two rounded products, |n| = sqrt((nx*nx + ny*ny) + nz*nz), area = 0.5 * |n|,
// normal = n / |n| per component. A face whose area is 0 or not finite has weight 0.
//
// CDF (per mesh, in float64, the blocking of SONET_MESH_RUN and SONET_MESH_TILE, include/sonet_b200.h):
// every summation is sequential, left to right, and starts from +0 (0 + x = x exactly), so each
// level is non-decreasing and so is the CDF.
//   run[f]  inclusive sum of the weights of f's run (SONET_MESH_RUN faces, starting at multiples of
//           the run length within the mesh) up to f
//   roff    exclusive sum of the run totals of the preceding runs of f's tile (SONET_MESH_TILE faces)
//   toff    exclusive sum of the tile totals (roff + run at a tile's last face) of the preceding tiles
//   cdf[f] = toff + (roff + run[f])
// Three launches build it for any mix of mesh sizes: the tile numbering (one CTA over the batch),
// one CTA per tile (runs and run offsets, the tile's total, its last face of positive weight and
// whether a face's area was not finite), and one thread per mesh (tile offsets, in place).
//
// Per sample, with draws (r, u, v) in [0,1): t = r * total; the face is the first f with
// cdf[f] > t (upper bound), clamped to the last face of positive weight; if u + v > 1 then
// u = 1 - u, v = 1 - v; the point is (a + u*e1) + v*e2. This is uniform on the triangle. The
// reference's sampler.m:35 computes a + u*b + v*c instead, which is not a point of the triangle; the
// README's description (uniform surface sampling) is what is implemented.
//
// The draws are given (DEVICE [B*N, 3] f64) or drawn from Philox4x32-10 (philox.cuh) keyed by
// (seed, mesh_ids[b], sample j) with stream tags 5 and 6: r and u from the first block's word pairs,
// v from the second's, 53 random bits each (32-bit draws would bias the choice among faces whose
// weights differ by less than 2^-32 of the total). The key is the mesh id, not the batch position, so
// a dataset built in chunks of any size and order has the same bits. Nothing synchronises, and no
// atomic operation decides a value.
#include <math.h>

#include "common.cuh"
#include "philox.cuh"

namespace sonet {

constexpr int MS_RUN = SONET_MESH_RUN;
constexpr int MS_TILE = SONET_MESH_TILE;
constexpr int MS_THREADS = MS_TILE / MS_RUN;       // one run per thread of the tile kernel
constexpr uint32_t MS_TAG_RU = 5u;                 // Philox stream tags (sample_points uses 3..4)
constexpr uint32_t MS_TAG_V = 6u;
constexpr long long MS_MAX_COUNT = 2147483647LL;   // per-mesh faces and vertices
constexpr long long MS_MAX_TOTAL = 1LL << 40;      // batch totals of faces and vertices
static_assert(MS_THREADS == 256 && MS_TILE % MS_RUN == 0, "tile kernel layout");

struct MeshScratch {
  size_t loc, tinc, tlast, tbad, tstart, mtotal, mlast, bytes;
  long long max_tiles;
};

static size_t ms_align256(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }

static MeshScratch mesh_scratch(int B, long long total_F) {
  MeshScratch s;
  // non-overlapping meshes cover at most total_F / tile full tiles plus one partial tile each
  s.max_tiles = total_F / MS_TILE + B;
  size_t o = 0;
  s.loc = o;    o = ms_align256(o + sizeof(double) * static_cast<size_t>(total_F));
  s.tinc = o;   o = ms_align256(o + sizeof(double) * static_cast<size_t>(s.max_tiles));
  s.tlast = o;  o = ms_align256(o + sizeof(int32_t) * static_cast<size_t>(s.max_tiles));
  s.tbad = o;   o = ms_align256(o + sizeof(int32_t) * static_cast<size_t>(s.max_tiles));
  s.tstart = o; o = ms_align256(o + sizeof(int64_t) * (static_cast<size_t>(B) + 1));
  s.mtotal = o; o = ms_align256(o + sizeof(double) * static_cast<size_t>(B));
  s.mlast = o;  o = ms_align256(o + sizeof(int32_t) * static_cast<size_t>(B));
  s.bytes = o;
  return s;
}

struct MeshArgs {
  const double* verts;      // [total_V, 3]
  const int64_t* v_off;     // [B+1]
  const int32_t* faces;     // [total_F, 3], vertex indices local to the mesh
  const int64_t* f_off;     // [B+1]
  const int64_t* mesh_ids;  // [B]
  const double* draws;      // [B*N, 3] (nullable: in-kernel draws)
  double* loc;              // [total_F] tile-local CDF (roff + run)
  double* tinc;             // [max_tiles] tile totals -> inclusive tile prefix of the mesh
  int32_t* tlast;           // [max_tiles] last face of positive weight in the tile (mesh-local), -1
  int32_t* tbad;            // [max_tiles] 1 when a face's area is not finite
  int64_t* tstart;          // [B+1] first tile of every mesh
  double* mtotal;           // [B] total weight, NaN for a mesh that cannot be sampled
  int32_t* mlast;           // [B] last face of positive weight
  float* out;               // [B*N, 6]
  int32_t* face_out;        // [B*N] (nullable)
  double* area_out;         // [B] (nullable)
  long long total_V, total_F, max_tiles;
  int B, N;
  uint32_t k0, k1;
};

// A mesh's [begin, end) rows of a ragged array, clamped into [0, total]; the count is 0 for a
// reversed range. Returns false when the count exceeds the per-mesh limit.
__device__ __forceinline__ bool mesh_range(const int64_t* off, int b, long long total, long long& begin,
                                           long long& count) {
  long long lo = off[b], hi = off[b + 1];
  lo = lo < 0 ? 0 : (lo > total ? total : lo);
  hi = hi < lo ? lo : (hi > total ? total : hi);
  begin = lo;
  count = hi - lo;
  return count <= MS_MAX_COUNT;
}

__device__ __forceinline__ long long mesh_tiles(const MeshArgs& a, int b) {
  long long f0, F, v0, V;
  const bool ok = mesh_range(a.f_off, b, a.total_F, f0, F) & mesh_range(a.v_off, b, a.total_V, v0, V);
  return ok ? (F + MS_TILE - 1) / MS_TILE : 0;
}

// The three vertices of face f of a mesh (indices clamped to [0, V-1]).
struct Tri {
  double ax, ay, az, e1x, e1y, e1z, e2x, e2y, e2z;
};

__device__ __forceinline__ Tri load_tri(const MeshArgs& a, long long f0, long long v0, long long V,
                                        long long f) {
  const int32_t* fi = a.faces + 3 * (f0 + f);
  long long idx[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const long long i = fi[k];
    idx[k] = v0 + (i < 0 ? 0 : (i >= V ? V - 1 : i));
  }
  const double* pa = a.verts + 3 * idx[0];
  const double* pb = a.verts + 3 * idx[1];
  const double* pc = a.verts + 3 * idx[2];
  Tri t;
  t.ax = pa[0];
  t.ay = pa[1];
  t.az = pa[2];
  t.e1x = __dsub_rn(pb[0], t.ax);
  t.e1y = __dsub_rn(pb[1], t.ay);
  t.e1z = __dsub_rn(pb[2], t.az);
  t.e2x = __dsub_rn(pc[0], t.ax);
  t.e2y = __dsub_rn(pc[1], t.ay);
  t.e2z = __dsub_rn(pc[2], t.az);
  return t;
}

// n = cross(e1, e2); returns |n|
__device__ __forceinline__ double tri_normal(const Tri& t, double& nx, double& ny, double& nz) {
  nx = __dsub_rn(__dmul_rn(t.e1y, t.e2z), __dmul_rn(t.e1z, t.e2y));
  ny = __dsub_rn(__dmul_rn(t.e1z, t.e2x), __dmul_rn(t.e1x, t.e2z));
  nz = __dsub_rn(__dmul_rn(t.e1x, t.e2y), __dmul_rn(t.e1y, t.e2x));
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz)));
}

// ---- launch 1: first tile of every mesh (one CTA, exact integer scan in chunks of its width) ----
constexpr int MS_SCAN_THREADS = 1024;

__global__ void __launch_bounds__(MS_SCAN_THREADS) mesh_tile_start_kernel(MeshArgs a) {
  __shared__ long long s[MS_SCAN_THREADS];
  __shared__ long long s_carry;
  const int tid = threadIdx.x;
  if (tid == 0) s_carry = 0;
  for (int base = 0; base < a.B; base += MS_SCAN_THREADS) {
    const int b = base + tid;
    const long long k = b < a.B ? mesh_tiles(a, b) : 0;
    s[tid] = k;
    __syncthreads();
    for (int o = 1; o < MS_SCAN_THREADS; o <<= 1) {
      const long long add = tid >= o ? s[tid - o] : 0;
      __syncthreads();
      s[tid] += add;
      __syncthreads();
    }
    const long long carry = s_carry;
    if (b < a.B) a.tstart[b] = carry + s[tid] - k;
    __syncthreads();
    if (tid == MS_SCAN_THREADS - 1) s_carry = carry + s[tid];
    __syncthreads();
  }
  if (tid == 0) a.tstart[a.B] = s_carry;
}

// ---- launch 2: one CTA per tile: run sums, run offsets, the tile's total, last face, flags ----
__global__ void __launch_bounds__(MS_THREADS) mesh_tile_kernel(MeshArgs a) {
  __shared__ double s_run[MS_THREADS];
  __shared__ int s_last[MS_THREADS / 32];
  const int tid = threadIdx.x;
  const long long ntiles = a.tstart[a.B] < a.max_tiles ? a.tstart[a.B] : a.max_tiles;
  for (long long g = blockIdx.x; g < ntiles; g += gridDim.x) {
    // the mesh owning global tile g: the last b with tstart[b] <= g (empty meshes own no tile)
    int lo = 0, hi = a.B - 1;
    while (lo < hi) {
      const int mid = lo + (hi - lo + 1) / 2;
      if (a.tstart[mid] <= g) lo = mid;
      else hi = mid - 1;
    }
    const int b = lo;
    long long f0, F, v0, V;
    mesh_range(a.f_off, b, a.total_F, f0, F);
    mesh_range(a.v_off, b, a.total_V, v0, V);
    const long long tile0 = (g - a.tstart[b]) * MS_TILE;
    const long long r0 = tile0 + static_cast<long long>(tid) * MS_RUN;
    double run[MS_RUN];
    double acc = 0.0;
    int last = -1;
    bool bad = false;
#pragma unroll
    for (int i = 0; i < MS_RUN; ++i) {
      const long long f = r0 + i;
      double w = 0.0;
      if (f < F && V > 0) {
        const Tri t = load_tri(a, f0, v0, V, f);
        double nx, ny, nz;
        const double area = __dmul_rn(0.5, tri_normal(t, nx, ny, nz));
        if (!isfinite(area)) bad = true;
        else if (area > 0.0) {
          w = area;
          last = static_cast<int>(f);
        }
      }
      acc = __dadd_rn(acc, w);
      run[i] = acc;
    }
    s_run[tid] = acc;
    const bool any_bad = __syncthreads_or(bad);
    if (tid == 0) {   // run offsets: sequential exclusive sum of the run totals
      double o = 0.0;
      for (int r = 0; r < MS_THREADS; ++r) {
        const double tot = s_run[r];
        s_run[r] = o;
        o = __dadd_rn(o, tot);
      }
    }
    last = __reduce_max_sync(0xffffffffu, last);
    if ((tid & 31) == 0) s_last[tid >> 5] = last;
    __syncthreads();
    const double roff = s_run[tid];
#pragma unroll
    for (int i = 0; i < MS_RUN; ++i)
      if (r0 + i < F) a.loc[f0 + r0 + i] = __dadd_rn(roff, run[i]);
    if (tid == MS_THREADS - 1) a.tinc[g] = __dadd_rn(roff, run[MS_RUN - 1]);  // the tile total
    if (tid == 0) {
      int m = s_last[0];
      for (int w = 1; w < MS_THREADS / 32; ++w) m = s_last[w] > m ? s_last[w] : m;
      a.tlast[g] = m;
      a.tbad[g] = any_bad ? 1 : 0;
    }
    __syncthreads();   // s_run and s_last are reused by the next tile of this CTA
  }
}

// ---- launch 3: one thread per mesh: tile offsets (in place), total, last face, area_out ----
__global__ void mesh_total_kernel(MeshArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;
  long long f0, F, v0, V;
  const bool ok = mesh_range(a.f_off, b, a.total_F, f0, F) & mesh_range(a.v_off, b, a.total_V, v0, V);
  const long long t0 = a.tstart[b], t1 = a.tstart[b + 1];
  double acc = 0.0;
  int last = -1;
  bool bad = !ok || t1 > a.max_tiles;   // too large a mesh, or offsets that overlap
  if (!bad) {
    for (long long g = t0; g < t1; ++g) {
      acc = __dadd_rn(acc, a.tinc[g]);
      a.tinc[g] = acc;
      last = a.tlast[g] > last ? a.tlast[g] : last;
      bad |= a.tbad[g] != 0;
    }
  }
  const double area = bad ? __longlong_as_double(0x7ff8000000000000LL) : acc;
  if (a.area_out) a.area_out[b] = area;
  const bool valid = !bad && acc > 0.0 && isfinite(acc) && last >= 0;
  a.mtotal[b] = valid ? acc : __longlong_as_double(0x7ff8000000000000LL);
  a.mlast[b] = last;
}

// ---- launch 4: one thread per sample ----
__device__ __forceinline__ double u53(uint32_t hi, uint32_t lo) {
  return static_cast<double>(((static_cast<uint64_t>(hi) << 32) | lo) >> 11) * 0x1.0p-53;
}

constexpr int MS_SAMPLE_THREADS = 256;

__global__ void __launch_bounds__(MS_SAMPLE_THREADS) mesh_sample_kernel(MeshArgs a) {
  const long long rows = static_cast<long long>(a.B) * a.N;
  for (long long i = static_cast<long long>(blockIdx.x) * MS_SAMPLE_THREADS + threadIdx.x; i < rows;
       i += static_cast<long long>(gridDim.x) * MS_SAMPLE_THREADS) {
    const int b = static_cast<int>(i / a.N);
    const uint32_t j = static_cast<uint32_t>(i - static_cast<long long>(b) * a.N);
    float* o = a.out + 6 * i;
    const double total = a.mtotal[b];
    if (!(total > 0.0)) {   // NaN: the mesh has no face to draw from
      const float nan = __int_as_float(0x7fc00000);
#pragma unroll
      for (int k = 0; k < 6; ++k) o[k] = nan;
      if (a.face_out) a.face_out[i] = -1;
      continue;
    }
    double r, u, v;
    if (a.draws) {
      r = a.draws[3 * i];
      u = a.draws[3 * i + 1];
      v = a.draws[3 * i + 2];
    } else {
      const uint64_t id = static_cast<uint64_t>(a.mesh_ids[b]);
      uint32_t c[4] = {j, static_cast<uint32_t>(id), MS_TAG_RU, static_cast<uint32_t>(id >> 32)};
      philox4x32_10(c, a.k0, a.k1);
      r = u53(c[0], c[1]);
      u = u53(c[2], c[3]);
      uint32_t d[4] = {j, static_cast<uint32_t>(id), MS_TAG_V, static_cast<uint32_t>(id >> 32)};
      philox4x32_10(d, a.k0, a.k1);
      v = u53(d[0], d[1]);
    }
    long long f0, F, v0, V;
    mesh_range(a.f_off, b, a.total_F, f0, F);
    mesh_range(a.v_off, b, a.total_V, v0, V);
    const double t = __dmul_rn(r, total);
    const double* loc = a.loc + f0;
    const double* tinc = a.tinc + a.tstart[b];
    long long lo = 0, hi = F;   // upper bound: the first f with cdf[f] > t
    while (lo < hi) {
      const long long mid = lo + ((hi - lo) >> 1);
      const long long k = mid / MS_TILE;
      const double cdf = __dadd_rn(k ? tinc[k - 1] : 0.0, loc[mid]);
      if (cdf > t) hi = mid;
      else lo = mid + 1;
    }
    const int last = a.mlast[b];
    const long long f = lo > last ? last : lo;
    if (__dadd_rn(u, v) > 1.0) {
      u = __dsub_rn(1.0, u);
      v = __dsub_rn(1.0, v);
    }
    const Tri tr = load_tri(a, f0, v0, V, f);
    double nx, ny, nz;
    const double len = tri_normal(tr, nx, ny, nz);
    o[0] = __double2float_rn(__dadd_rn(__dadd_rn(tr.ax, __dmul_rn(u, tr.e1x)), __dmul_rn(v, tr.e2x)));
    o[1] = __double2float_rn(__dadd_rn(__dadd_rn(tr.ay, __dmul_rn(u, tr.e1y)), __dmul_rn(v, tr.e2y)));
    o[2] = __double2float_rn(__dadd_rn(__dadd_rn(tr.az, __dmul_rn(u, tr.e1z)), __dmul_rn(v, tr.e2z)));
    o[3] = __double2float_rn(__ddiv_rn(nx, len));
    o[4] = __double2float_rn(__ddiv_rn(ny, len));
    o[5] = __double2float_rn(__ddiv_rn(nz, len));
    if (a.face_out) a.face_out[i] = static_cast<int32_t>(f);
  }
}

static int mesh_check(const char* what, int B, long long total_F) {
  SONET_REQUIRE(B >= 0, "%s: B=%d must be >= 0", what, B);
  SONET_REQUIRE(total_F >= 0 && total_F <= MS_MAX_TOTAL, "%s: total_F=%lld outside [0, 2^40]", what,
                total_F);
  return SONET_OK;
}

}  // namespace sonet

extern "C" long long sonet_mesh_sample_scratch_bytes(int B, long long total_F) {
  using namespace sonet;
  if (mesh_check("mesh_sample_scratch_bytes", B, total_F) != SONET_OK) return SONET_ERR_BAD_ARG;
  return static_cast<long long>(mesh_scratch(B, total_F).bytes);
}

extern "C" int sonet_mesh_sample_f32(const double* verts, const int64_t* v_off, long long total_V,
                                     const int32_t* faces, const int64_t* f_off, long long total_F,
                                     const int64_t* mesh_ids, int B, int N, const double* draws,
                                     unsigned long long seed, void* scratch, long long scratch_bytes,
                                     float* out, int32_t* face_out, double* area_out,
                                     sonet_stream_t stream) {
  using namespace sonet;
  if (mesh_check("mesh_sample", B, total_F) != SONET_OK) return SONET_ERR_BAD_ARG;
  SONET_REQUIRE(N >= 1 && N <= SONET_MESH_MAX_N, "mesh_sample: N=%d outside [1, %d]", N,
                SONET_MESH_MAX_N);
  SONET_REQUIRE(total_V >= 0 && total_V <= MS_MAX_TOTAL, "mesh_sample: total_V=%lld outside [0, 2^40]",
                total_V);
  SONET_REQUIRE(v_off && f_off && mesh_ids && scratch && out,
                "mesh_sample: v_off, f_off, mesh_ids, scratch and out must not be null");
  SONET_REQUIRE(verts || total_V == 0, "mesh_sample: verts must not be null (total_V=%lld)", total_V);
  SONET_REQUIRE(faces || total_F == 0, "mesh_sample: faces must not be null (total_F=%lld)", total_F);
  const MeshScratch S = mesh_scratch(B, total_F);
  SONET_REQUIRE(scratch_bytes >= static_cast<long long>(S.bytes),
                "mesh_sample: scratch of %lld bytes, %lld needed", scratch_bytes,
                static_cast<long long>(S.bytes));
  SONET_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 255u) == 0,
                "mesh_sample: scratch must be 256-byte aligned");
  if (B == 0) return SONET_OK;
  char* base = static_cast<char*>(scratch);
  MeshArgs a;
  a.verts = verts;
  a.v_off = v_off;
  a.faces = faces;
  a.f_off = f_off;
  a.mesh_ids = mesh_ids;
  a.draws = draws;
  a.loc = reinterpret_cast<double*>(base + S.loc);
  a.tinc = reinterpret_cast<double*>(base + S.tinc);
  a.tlast = reinterpret_cast<int32_t*>(base + S.tlast);
  a.tbad = reinterpret_cast<int32_t*>(base + S.tbad);
  a.tstart = reinterpret_cast<int64_t*>(base + S.tstart);
  a.mtotal = reinterpret_cast<double*>(base + S.mtotal);
  a.mlast = reinterpret_cast<int32_t*>(base + S.mlast);
  a.out = out;
  a.face_out = face_out;
  a.area_out = area_out;
  a.total_V = total_V;
  a.total_F = total_F;
  a.max_tiles = S.max_tiles;
  a.B = B;
  a.N = N;
  a.k0 = static_cast<uint32_t>(seed);
  a.k1 = static_cast<uint32_t>(seed >> 32);
  cudaStream_t st = as_stream(stream);
  mesh_tile_start_kernel<<<1, MS_SCAN_THREADS, 0, st>>>(a);
  int rc = check_launch("mesh_sample (tile numbering)");
  if (rc != SONET_OK) return rc;
  const long long tile_grid = S.max_tiles < 8LL * 65536 ? S.max_tiles : 8LL * 65536;
  if (tile_grid > 0) {
    mesh_tile_kernel<<<static_cast<unsigned>(tile_grid), MS_THREADS, 0, st>>>(a);
    rc = check_launch("mesh_sample (tile scan)");
    if (rc != SONET_OK) return rc;
  }
  mesh_total_kernel<<<(B + 127) / 128, 128, 0, st>>>(a);
  rc = check_launch("mesh_sample (mesh totals)");
  if (rc != SONET_OK) return rc;
  const long long rows = static_cast<long long>(B) * N;
  const long long blocks = (rows + MS_SAMPLE_THREADS - 1) / MS_SAMPLE_THREADS;
  mesh_sample_kernel<<<static_cast<unsigned>(blocks < (1LL << 20) ? blocks : (1LL << 20)),
                       MS_SAMPLE_THREADS, 0, st>>>(a);
  return check_launch("mesh_sample");
}
