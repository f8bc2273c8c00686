// pointwise_tc.cu — generic point-wise shared-MLP layer (1x1 conv + folded BN + ReLU) on Hopper
// warpgroup MMA (wgmma).
//
// Same contract as sonet_pointwise_layer_f32 (csrc/pointwise.cu; EquivariantLayer / MyConv2d 1x1 eval
// forward, models/layers.py:203-210, 282-296) for the layers that are dense enough for tensor
// cores: KNNModule's 387->512->512 (models/layers.py:362-364), the final PointNet 515->768->1024
// (models/networks.py:192) and the segmenter head (models/networks.py:326-341).
//
//   out[b,co,p] = act( inv * sum_ci Ws[co,ci] * X[b,ci,p] + shift[co] (+ addend[b,co,g(b,p)]) )
//
// Rows (b,p) are flattened and tiled by 128; an item is (row tile, 128-wide out-channel tile); K
// streams in 64-channel chunks:
//   * two consumer warpgroups, one per 64 rows of the tile (wgmma M = 64). Each thread fetches 32
//     channels of one row of the next chunk with coalesced loads (a warp instruction reads 32
//     consecutive points of one channel) while the current chunk's wgmmas run, splits them into
//     fp16 hi/lo and writes the K-major no-swizzle A images with one 128-bit shared store per 8
//     channels (conflict free), then issues 3 wgmma per 16-channel K step (hi*hi + lo*hi + hi*lo)
//     with fp32 accumulators in registers (64 per thread at N = 128). A 2-slot A ring: a slot is
//     rewritten once wgmma.wait_group shows the chunk that read it complete. The opt-in fp16
//     mode (the `_f16` entries, NPROD = 1) writes only the hi image and issues hi*hi alone;
//   * producer warp: streams the pre-packed fp16 hi/lo weight images (cp.async.bulk + mbarrier)
//     through a 4-stage ring shared by both warpgroups;
//   * epilogue in registers: fused scale/shift (+ gathered addend) + ReLU (one max against 0 or
//     -inf, so ReLU and no activation share a kernel) or, in the ELU build, ELU; eight lanes of a warp
//     hold eight consecutive points of one channel, so every store fills 32-byte sectors. The
//     point-major store mode (out [B,P,Cout]) writes each thread's column pair as one float2: four
//     lanes fill one 32-byte sector of a row.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>

#include "tc_common.cuh"

namespace sonet {
namespace pwt {
// the weight blob's n-tile width NT, K chunk KCH and stage K extent WK: tc::wblob
constexpr int TILE = 128, KCH = tc::wblob::KCH, NT = tc::wblob::NT, WK = tc::wblob::WK;
constexpr int NSUB = 128;                       // out channels per item (two per blob tile)
constexpr int A_HALF = TILE * KCH * 2;          // one fp16 image of an activation chunk, 16 KB
constexpr int A_BYTES = 2 * A_HALF;             // hi + lo
constexpr int WIMG = NSUB * WK * 2;             // one [128 x 32] fp16 weight image, 8 KB
constexpr int WS_BYTES = 4 * WIMG;              // one chunk in shared memory: [half][hi|lo], 32 KB
constexpr int NSTAGE = 2;                       // A ring
constexpr int NSTAGE_W = 4;                     // weight ring
constexpr int NUM_THREADS = 288;                // warps 0-7: two consumer warpgroups, warp 8: producer
constexpr int OFF_A = 0;
constexpr int OFF_W = OFF_A + NSTAGE * A_BYTES;
constexpr int OFF_BAR = OFF_W + NSTAGE_W * WS_BYTES;
constexpr int NBAR = 2 * NSTAGE_W;
constexpr int SMEM_BYTES = OFF_BAR + NBAR * 8;

struct Dims {
  int C0, C1, B, P, Cout, G;
  float floor_v; // the non-ELU epilogue's max: 0 (ReLU), -inf (no activation) or NaN (a raw K-split
                 // partial: fmaxf(y, NaN) == y for every y, NaN included)
  int kchunks;   // ceil(pad16(Cin) / 64)
  int ntiles;    // out-channel items of <= 128 (each a multiple of 64)
  int cin_pad;   // Cin rounded up to 16
  float inv;     // 1 / weight pre-scale
  // ---- grouped / split-K / scatter extensions (the up-convolution decoder, csrc/upconv.cu) ----
  int groups;    // independent GEMMs sharing shapes: x is [groups*B, C, P], one weight blob each
  int splits;    // K split: an item covers kchunks/splits chunks and writes a raw partial sum
  int kpi;       // k chunks per item (= kchunks / splits)
  int row_tiles; // 128-row tiles per group
  int scat_w;    // > 0: group g = (py, px) parity of a x2 up-convolution over a [*, scat_w] map;
                 //      row p = i*W + j is stored at (2i+py)*2W + 2j+px of a [B, Cout, P_out] map
  int P_out;     // point stride of `out` (= P unless scattering)
  int conv_w;    // > 0: up-convolution mode without im2col. x is [3*B, Cin, H*W] = the input shifted
                 //      horizontally by -1, 0, +1 (csrc/upconv.cu); K chunk kc = (tap t = a*2+c,
                 //      64-channel chunk): rows are read from block c-1+px+1 at point p + (a-1+py)*W
                 //      — vertical shifts are plain coordinate offsets, out of range reads zeros
  int cpt;       // 64-channel chunks per tap (= Cin / 64) in conv mode
  const float* inv_ptr;     // non-null: 1 / weight pre-scale lives in device memory (train mode:
                            // the weights are packed on the device every step, csrc/train.cu)
  const float* act_ptr;     // non-null: power-of-two pre-scale of the ACTIVATIONS (device memory),
                            // applied before the fp16 hi/lo split — gradients are far below the
                            // fp16 normal range; its inverse must be folded into *inv_ptr
  long long blob_gstride;   // bytes between the weight blobs of consecutive groups
  long long out_gstride;    // floats between the outputs of consecutive groups (0 when scattering)
  long long out_sstride;    // floats between the partial sums of consecutive K splits
  int rows_out;             // 1: out is point-major [B, P, Cout] (single group, no split or scatter)
};
struct Item {
  int g, tile, nt, sub, kc0;
};
__device__ __forceinline__ Item decode_item(const Dims& d, int item) {
  // n-tile fastest: the activation tile stays hot in L2; then K split, row tile, group
  Item r;
  const int s = item % d.ntiles;
  r.nt = s >> 1;
  r.sub = s & 1;
  int t = item / d.ntiles;
  const int sp = t % d.splits;
  t /= d.splits;
  r.tile = t % d.row_tiles;
  r.g = t / d.row_tiles;
  r.kc0 = sp * d.kpi;
  return r;
}
__device__ inline int item_width(int Cout, int nt, int sub) {
  return min(NSUB, tc::wblob::tile_width(Cout, nt) - sub * NSUB);
}
}  // namespace pwt

// NPROD: fp16 products per MAC, 3 (hi/lo split, the default) or 1 (hi only, the opt-in fp16 mode:
// the lo A image is never written and the producer copies only the hi image of each stage).
// ELU: the epilogue applies ELU instead of the max against d.floor_v
template <int NPROD, bool ELU>
__global__ void __launch_bounds__(pwt::NUM_THREADS, 1)
    pointwise_tc_kernel(const float* __restrict__ x0, const float* __restrict__ x1,
                        const unsigned char* __restrict__ blob, const float* __restrict__ shift,
                        const float* __restrict__ addend, const int32_t* __restrict__ gidx,
                        float* __restrict__ out, pwt::Dims d, long long* __restrict__ dbg) {
  using namespace pwt;
  if (dbg != nullptr && blockIdx.x == 0 && threadIdx.x == 0) dbg[127] = clock64();
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* full_w = reinterpret_cast<uint64_t*>(smem + OFF_BAR);   // [NSTAGE_W] producer -> MMA
  uint64_t* empty_w = full_w + NSTAGE_W;                             // [NSTAGE_W] MMA -> producer

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const long long rows = static_cast<long long>(d.B) * d.P;   // rows of ONE group
  const int items = d.groups * d.row_tiles * d.splits * d.ntiles;
  const int my_items =
      (static_cast<int>(blockIdx.x) < items) ? (items - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const int Cin = d.C0 + d.C1;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE_W; ++s) {
      mbar_init(&full_w[s], 1);
      mbar_init(&empty_w[s], 8);   // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ================= producer: weight chunk images =================
    if (lane == 0) {
      uint32_t q = 0;
      for (int it = 0; it < my_items; ++it) {
        const Item im = decode_item(d, blockIdx.x + it * gridDim.x);
        const int nw = tc::wblob::tile_width(d.Cout, im.nt);
        const int ns = item_width(d.Cout, im.nt, im.sub);
        // this item's rows are [128 sub, 128 sub + ns) of each image of n-tile nt
        const unsigned char* rows = blob + static_cast<size_t>(im.g) * d.blob_gstride +
                                    static_cast<size_t>(im.sub) * NSUB * WK * 2;
        const uint32_t bytes = static_cast<uint32_t>(ns) * WK * 2;
        for (int kc = im.kc0; kc < im.kc0 + d.kpi; ++kc, ++q) {
          const int halves = (d.cin_pad - kc * KCH > WK) ? 2 : 1;   // the consumers agree
          const uint32_t slot = q % NSTAGE_W, use = q / NSTAGE_W;
          if (use > 0) tc::mbar_wait_relaxed(&empty_w[slot], (use - 1) & 1, 200);
          mbar_arrive_expect_tx(&full_w[slot], (NPROD == 3 ? 2 : 1) * halves * bytes);
          unsigned char* dst = smem + OFF_W + slot * WS_BYTES;
          for (int hh = 0; hh < halves; ++hh) {
            const unsigned char* src = rows + tc::wblob::stage_off(d.Cout, d.kchunks, im.nt, kc, hh);
            bulk_g2s(dst + (2 * hh) * WIMG, src, bytes, &full_w[slot]);
            if (NPROD == 3)
              bulk_g2s(dst + (2 * hh + 1) * WIMG, src + static_cast<size_t>(nw) * WK * 2, bytes,
                       &full_w[slot]);
          }
        }
      }
    }
  } else {
    // ================= consumers: 64 rows each =================
    const int wg = warp >> 2;                 // which 64 rows of the tile
    const int tw = threadIdx.x & 127;
    const int m = tw & 63, half = tw >> 6;    // conversion: row m, channels [32 half, 32 half + 32)
    const float act_s = d.act_ptr != nullptr ? __ldg(d.act_ptr) : 1.f;
    const float floor_v = d.floor_v;   // ReLU, no activation or a raw partial as one max
    const float inv_w = d.inv_ptr != nullptr ? __ldg(d.inv_ptr) : d.inv;
    const uint32_t a_base = smem_u32(smem + OFF_A) + wg * (A_HALF / 2);
    const uint32_t w_base = smem_u32(smem + OFF_W);
    uint32_t qa = 0;   // chunks consumed by this CTA so far (A and weight ring position)

    // fetch 32 channels of row m of chunk kc of item im
    auto fetch = [&](const Item& im, int kc, float (&v)[32]) {
      const long long R = static_cast<long long>(im.tile) * TILE + wg * 64 + m;
      const bool valid = R < rows;
      const int bl = valid ? static_cast<int>(R / d.P) : 0;
      int p = valid ? static_cast<int>(R - static_cast<long long>(bl) * d.P) : 0;
      if (d.conv_w > 0) {
        const int tap = kc / d.cpt;
        const int cc = (kc - tap * d.cpt) * KCH + half * 32;
        const int py = im.g >> 1, px = im.g & 1;
        p += ((tap >> 1) - 1 + py) * d.conv_w;                 // vertical shift: out of range -> 0
        const int b = ((tap & 1) + px) * d.B + bl;             // horizontal-shift block 0..2
        const bool ok = valid && p >= 0 && p < d.P;
        const float* src = x0 + (static_cast<size_t>(b) * d.C0 + cc) * d.P + p;
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = ok ? __ldg(src + static_cast<size_t>(i) * d.P) : 0.f;
        return;
      }
      const int b = im.g * d.B + bl;
      const float* r0 = x0 + static_cast<size_t>(b) * d.C0 * d.P + p;
      const float* r1 = d.C1 ? x1 + static_cast<size_t>(bl) * d.C1 * d.P + p : x0;
      const int c_base = kc * KCH + half * 32;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int ci = c_base + i;
        const bool ok = valid && ci < Cin;
        const float* src = ci < d.C0 ? r0 + static_cast<size_t>(ci) * d.P
                                     : r1 + static_cast<size_t>(ci - d.C0) * d.P;
        v[i] = ok ? __ldg(src) : 0.f;
      }
    };

    for (int it = 0; it < my_items; ++it) {
      const Item im = decode_item(d, blockIdx.x + it * gridDim.x);
      const int ns = item_width(d.Cout, im.nt, im.sub);
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      float v[32];
      fetch(im, im.kc0, v);
      uint32_t prev_slot = 0;
      for (int i = 0; i < d.kpi; ++i, ++qa) {
        const int kc = im.kc0 + i;
        const uint32_t sa = qa % NSTAGE, sw = qa % NSTAGE_W;
        // convert into A slot sa (the chunk that read it last completed: wait_group<1> below)
        if (d.act_ptr != nullptr) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] *= act_s;
        }
        unsigned char* a_hi = smem + OFF_A + sa * A_BYTES + wg * (A_HALF / 2) + (m >> 3) * 1024 +
                              (m & 7) * 16;
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int j = 0; j < 4; ++j)
            tc::split_words<NPROD>(v[o * 8 + 2 * j], v[o * 8 + 2 * j + 1], hi[j], lo[j]);
          const int oct = half * 4 + o;
          *reinterpret_cast<uint4*>(a_hi + oct * 128) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
          if (NPROD == 3)
            *reinterpret_cast<uint4*>(a_hi + A_HALF + oct * 128) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
        tc::fence_proxy_async();
        tc::named_sync(1 + wg, 128);         // the warpgroup's 64 rows are written
        tc::mbar_wait_bounded(&full_w[sw], (qa / NSTAGE_W) & 1, 202);
        const int nks = min(4, (d.cin_pad - kc * KCH) / 16);
        const uint32_t as = a_base + sa * A_BYTES, ws = w_base + sw * WS_BYTES;
        tc::wg_fence();
#pragma unroll 1
        for (int ks = 0; ks < nks; ++ks) {
          // A: [64 x 64] rows of this warpgroup, SBO 1024; B: [ns x 32] image of half ks/2, SBO 512
          const uint64_t ah = tc::smem_desc(as + ks * 256, 128, 1024),
                         al = tc::smem_desc(as + A_HALF + ks * 256, 128, 1024);
          const uint32_t wb = ws + (ks >> 1) * 2 * WIMG + (ks & 1) * 256;
          const uint64_t bh = tc::smem_desc(wb, 128, 512), bl = tc::smem_desc(wb + WIMG, 128, 512);
          if (ns == NSUB) {
            tc::wgmma_f16_n128(acc, ah, bh, 1);
            if (NPROD == 3) {
              tc::wgmma_f16_n128(acc, al, bh, 1);
              tc::wgmma_f16_n128(acc, ah, bl, 1);
            }
          } else {
            float (&a32)[32] = *reinterpret_cast<float (*)[32]>(acc);
            tc::wgmma_f16_n64(a32, ah, bh, 1);
            if (NPROD == 3) {
              tc::wgmma_f16_n64(a32, al, bh, 1);
              tc::wgmma_f16_n64(a32, ah, bl, 1);
            }
          }
        }
        tc::wg_commit();
        if (i + 1 < d.kpi) fetch(im, kc + 1, v);   // global loads in flight during the wgmmas
        tc::wg_wait<1>();                          // the previous chunk is complete ...
        // ... for every warp of the warpgroup (wait_group covers only the executing warp's groups):
        // the next chunk rewrites A rows that other warps' wgmmas of that chunk read
        tc::named_sync(1 + wg, 128);
        if (i > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_w[prev_slot]);
        }
        prev_slot = sw;
      }
      tc::wg_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_w[prev_slot]);

      // ---- epilogue: thread holds rows r0 = 16*(warp%4) + lane/4 and r0 + 8, columns
      // 8j + 2*(lane%4) + {0,1} (accumulators 4j+{0,1} and 4j+{2,3}) ----
      const int col0 = im.nt * NT + im.sub * NSUB + 2 * (lane & 3);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const long long R = static_cast<long long>(im.tile) * TILE + wg * 64 + 16 * (warp & 3) +
                            (lane >> 2) + 8 * rr;
        if (R >= rows) continue;
        const int b = static_cast<int>(R / d.P);
        const int p = static_cast<int>(R - static_cast<long long>(b) * d.P);
        // where row (b, p) of this group / K split lands in `out`
        const size_t obase = static_cast<size_t>(im.g) * d.out_gstride +
                             static_cast<size_t>(im.kc0 / d.kpi) * d.out_sstride;
        int po = p;
        if (d.scat_w > 0) {   // x2 up-convolution: parity (py, px) = group
          const int i = p / d.scat_w, j = p - i * d.scat_w;
          po = (2 * i + (im.g >> 1)) * 2 * d.scat_w + 2 * j + (im.g & 1);
        }
        const float* arow = nullptr;
        if (addend != nullptr) {
          const int g = min(max(__ldg(gidx + static_cast<long long>(im.g) * rows + R), 0), d.G - 1);
          arow = addend + static_cast<size_t>(b) * d.Cout * d.G + g;
        }
        if (d.rows_out) {
          // point-major: out[R, co], columns (co, co+1) as one float2 when both exist and Cout is
          // even (8-byte aligned); same values as the channel-major store
          float* o = out + static_cast<size_t>(R) * d.Cout;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            if (8 * j >= ns) break;
            const int co = col0 + 8 * j;
            float y[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              y[e] = fmaf(acc[4 * j + 2 * rr + e], inv_w,
                          (shift != nullptr && co + e < d.Cout) ? __ldg(shift + co + e) : 0.f);
              if (arow != nullptr && co + e < d.Cout) y[e] += __ldg(arow + static_cast<size_t>(co + e) * d.G);
              y[e] = ELU ? elu1(y[e]) : fmaxf(y[e], floor_v);
            }
            if (co + 1 < d.Cout && (d.Cout & 1) == 0)
              *reinterpret_cast<float2*>(o + co) = make_float2(y[0], y[1]);
            else
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (co + e < d.Cout) o[co + e] = y[e];
          }
          continue;
        }
        float* o = out + obase + static_cast<size_t>(b) * d.Cout * d.P_out + po;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          if (8 * j >= ns) break;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int co = col0 + 8 * j + e;
            if (co < d.Cout) {
              float y = fmaf(acc[4 * j + 2 * rr + e], inv_w, shift != nullptr ? __ldg(shift + co) : 0.f);
              if (arow != nullptr) y += __ldg(arow + static_cast<size_t>(co) * d.G);
              o[static_cast<size_t>(co) * d.P_out] = ELU ? elu1(y) : fmaxf(y, floor_v);
            }
          }
        }
      }
    }
  }
  if (dbg != nullptr && blockIdx.x == 0 && threadIdx.x == 0) dbg[126] = clock64();
}

}  // namespace sonet

extern "C" long long sonet_pointwise_tc_blob_bytes(int Cout, int Cin) {
  if (Cout < 1 || Cin < 1) return -1;
  return sonet::tc::wblob::bytes(Cout, Cin);
}

// G matrices [G, Cout, Cin] packed back to back (sonet_pointwise_tc_blob_bytes each) with ONE
// common power-of-two pre-scale: the weight blobs of a grouped launch.
extern "C" int sonet_pointwise_tc_pack_groups(const float* W, int G, int Cout, int Cin,
                                              void* blob_host, float* inv_scale) {
  using namespace sonet;
  SONET_REQUIRE(W && blob_host && inv_scale && G >= 1 && Cout >= 1 && Cin >= 1,
                "pointwise_tc_pack: bad args");
  const size_t per = static_cast<size_t>(Cout) * Cin;
  const float scale = pow2_scale(W, per * G);
  *inv_scale = 1.f / scale;
  const long long bytes = tc::wblob::bytes(Cout, Cin);
  const int kch = tc::wblob::kchunks(Cin);
  unsigned char* blob = static_cast<unsigned char*>(blob_host);
  std::memset(blob, 0, static_cast<size_t>(bytes) * G);
  for (int g = 0; g < G; ++g)
    for (int n = 0; n < Cout; ++n)
      for (int k = 0; k < Cin; ++k) {
        long long hi, lo;
        tc::wblob::elem_off(Cout, kch, n, k, hi, lo);
        tc::put_weight(blob + g * bytes + hi, blob + g * bytes + lo,
                       W[g * per + static_cast<size_t>(n) * Cin + k] * scale);
      }
  return SONET_OK;
}

extern "C" int sonet_pointwise_tc_pack(const float* W, int Cout, int Cin, void* blob_host,
                                       float* inv_scale) {
  return sonet_pointwise_tc_pack_groups(W, 1, Cout, Cin, blob_host, inv_scale);
}

struct TcExt {   // grouped / split-K / scatter / point-major launch options (defaults = the plain layer)
  int groups = 1, splits = 1, scat_w = 0, P_out = 0, conv_w = 0, rows_out = 0;
  int nprod = 3;   // fp16 products per MAC: 3 (hi/lo split) or 1 (the opt-in fp16 mode)
  int raw = 0;     // 1: store acc * inv (+ shift) with no activation, NaN kept (K-split partials)
  const float* inv_ptr = nullptr;
  const float* act_ptr = nullptr;
  long long blob_gstride = 0, out_gstride = 0, out_sstride = 0;
};

// relu: activation code (SONET_ACT_*), validated by the entry points
static int launch_pointwise_tc(const float* x0, int C0, const float* x1, int C1, int B,
                                          int P, const void* blob, float inv_scale,
                                          const float* shift, int Cout, int relu,
                                          const float* addend, const int32_t* gidx, int G,
                                          float* out, long long* dbg, sonet_stream_t stream,
                                          const TcExt& ext = TcExt()) {
  using namespace sonet;
  using namespace sonet::pwt;
  SONET_REQUIRE(B >= 0 && P >= 0 && C0 >= 1 && C1 >= 0 && Cout >= 1, "pointwise_tc: bad dimension");
  if (B == 0 || P == 0) return SONET_OK;
  SONET_REQUIRE(x0 && blob && out, "pointwise_tc: null pointer");
  SONET_REQUIRE(C1 == 0 || x1 != nullptr, "pointwise_tc: x1 null with C1=%d", C1);
  SONET_REQUIRE(C1 == 0 || ext.groups == 1, "pointwise_tc: two sources need groups == 1");
  SONET_REQUIRE(!addend || (gidx && G >= 1), "pointwise_tc: addend needs gidx and G");
  SONET_REQUIRE(aligned16(blob), "pointwise_tc: weight blob must be 16-byte aligned");
  Dims d;
  d.C0 = C0; d.C1 = C1; d.B = B; d.P = P; d.Cout = Cout; d.G = G;
  d.floor_v = ext.raw ? std::numeric_limits<float>::quiet_NaN()
                      : (relu == SONET_ACT_RELU ? 0.f : -std::numeric_limits<float>::infinity());
  d.conv_w = ext.conv_w;
  d.cpt = 1;
  if (ext.conv_w > 0) {
    SONET_REQUIRE(C1 == 0 && C0 % KCH == 0 && P % 64 == 0 && P % ext.conv_w == 0 && ext.groups == 4,
                  "pointwise_tc: conv mode needs Cin %% 64 == 0, H*W %% 64 == 0 and the 4 parity groups");
    d.cpt = C0 / KCH;
  }
  d.cin_pad = ext.conv_w > 0 ? 4 * C0 : (C0 + C1 + 15) / 16 * 16;
  d.kchunks = (d.cin_pad + KCH - 1) / KCH;
  d.ntiles = ((Cout + 63) / 64 * 64 + NSUB - 1) / NSUB;
  d.inv = inv_scale;
  SONET_REQUIRE(ext.groups >= 1 && ext.splits >= 1 && d.kchunks % ext.splits == 0,
                "pointwise_tc: %d K chunks cannot be split %d ways", d.kchunks, ext.splits);
  d.groups = ext.groups;
  d.splits = ext.splits;
  d.kpi = d.kchunks / ext.splits;
  d.scat_w = ext.scat_w;
  d.P_out = ext.P_out > 0 ? ext.P_out : P;
  d.inv_ptr = ext.inv_ptr;
  d.act_ptr = ext.act_ptr;
  d.blob_gstride = ext.blob_gstride;
  d.out_gstride = ext.out_gstride;
  d.out_sstride = ext.out_sstride;
  d.rows_out = ext.rows_out;
  SONET_REQUIRE(!ext.rows_out || (ext.groups == 1 && ext.splits == 1 && ext.scat_w == 0 &&
                                  ext.conv_w == 0),
                "pointwise_tc: the point-major store needs one group, no split and no scatter");
  const long long rows = static_cast<long long>(B) * P;
  d.row_tiles = static_cast<int>((rows + TILE - 1) / TILE);
  const long long items = static_cast<long long>(d.row_tiles) * d.ntiles * ext.groups * ext.splits;
  SONET_REQUIRE(items < (1LL << 31), "pointwise_tc: too many tiles");
  SONET_REQUIRE(SMEM_BYTES <= max_smem_optin(), "pointwise_tc: needs %d B of shared memory", SMEM_BYTES);
  SONET_REQUIRE(ext.nprod == 3 || ext.nprod == 1, "pointwise_tc: %d products per MAC", ext.nprod);
  auto kern = relu == SONET_ACT_ELU ? (ext.nprod == 1 ? pointwise_tc_kernel<1, true> : pointwise_tc_kernel<3, true>)
                                    : (ext.nprod == 1 ? pointwise_tc_kernel<1, false> : pointwise_tc_kernel<3, false>);
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  const int grid = static_cast<int>(std::min<long long>(items, sm_count()));
  kern<<<grid, NUM_THREADS, SMEM_BYTES, as_stream(stream)>>>(
      x0, x1, static_cast<const unsigned char*>(blob), shift, addend, gidx, out, d, dbg);
  return check_launch("pointwise_tc");
}

static TcExt with_nprod(int nprod) {
  TcExt e;
  e.nprod = nprod;
  return e;
}

extern "C" int sonet_pointwise_tc_forward(const float* x0, int C0, const float* x1, int C1, int B,
                                          int P, const void* blob, float inv_scale,
                                          const float* shift, int Cout, int relu,
                                          const float* addend, const int32_t* gidx, int G,
                                          float* out, sonet_stream_t stream) {
  SONET_REQUIRE_ACT(relu, "pointwise_tc_forward");
  return launch_pointwise_tc(x0, C0, x1, C1, B, P, blob, inv_scale, shift, Cout, relu, addend, gidx, G,
                             out, nullptr, stream);
}

// the opt-in fp16 mode: one product hi(x)*hi(w) per MAC, same blob and arguments
extern "C" int sonet_pointwise_tc_forward_f16(const float* x0, int C0, const float* x1, int C1, int B,
                                              int P, const void* blob, float inv_scale,
                                              const float* shift, int Cout, int relu,
                                              const float* addend, const int32_t* gidx, int G,
                                              float* out, sonet_stream_t stream) {
  SONET_REQUIRE_ACT(relu, "pointwise_tc_forward_f16");
  return launch_pointwise_tc(x0, C0, x1, C1, B, P, blob, inv_scale, shift, Cout, relu, addend, gidx, G,
                             out, nullptr, stream, with_nprod(1));
}

static int pointwise_tc_rows(const float* x0, int C0, const float* x1, int C1, int B, int P,
                             const void* blob, float inv_scale, const float* shift, int Cout, int relu,
                             const float* addend, const int32_t* gidx, int G, float* out,
                             sonet_stream_t stream, int nprod) {
  TcExt e = with_nprod(nprod);
  e.rows_out = 1;
  return launch_pointwise_tc(x0, C0, x1, C1, B, P, blob, inv_scale, shift, Cout, relu, addend, gidx, G,
                             out, nullptr, stream, e);
}

extern "C" int sonet_pointwise_tc_forward_rows(const float* x0, int C0, const float* x1, int C1,
                                               int B, int P, const void* blob, float inv_scale,
                                               const float* shift, int Cout, int relu,
                                               const float* addend, const int32_t* gidx, int G,
                                               float* out, sonet_stream_t stream) {
  SONET_REQUIRE_ACT(relu, "pointwise_tc_forward_rows");
  return pointwise_tc_rows(x0, C0, x1, C1, B, P, blob, inv_scale, shift, Cout, relu, addend, gidx, G,
                           out, stream, 3);
}

extern "C" int sonet_pointwise_tc_forward_rows_f16(const float* x0, int C0, const float* x1, int C1,
                                                   int B, int P, const void* blob, float inv_scale,
                                                   const float* shift, int Cout, int relu,
                                                   const float* addend, const int32_t* gidx, int G,
                                                   float* out, sonet_stream_t stream) {
  SONET_REQUIRE_ACT(relu, "pointwise_tc_forward_rows_f16");
  return pointwise_tc_rows(x0, C0, x1, C1, B, P, blob, inv_scale, shift, Cout, relu, addend, gidx, G,
                           out, stream, 1);
}

namespace sonet {
// partial [G][S][B][Cout][P] (raw K-split sums) -> out: sum over S in ascending order (fixed ->
// deterministic), + shift, the activation as the main epilogue applies it (a max against 0 or
// -inf, or in the ELU build ELU), and the up-convolution parity scatter.
// IT = uint32_t when every index fits 32 bits (always, in practice): the three divisions per element
// were 64-bit ones, and the kernel was bound by them (17 us for 2.1 M outputs), not by its 40 MB.
template <typename IT, bool ELU>
__global__ void __launch_bounds__(256)
    splitk_reduce_kernel(const float* __restrict__ part, int G, int S, int B, int Cout, int P,
                         const float* __restrict__ shift, int relu, int scat_w, int P_out,
                         long long out_gstride, float* __restrict__ out) {
  const IT per_split = static_cast<IT>(B) * Cout * P;
  const IT total = per_split * G;
  const IT uP = static_cast<IT>(P), uC = static_cast<IT>(Cout);
  for (IT t = static_cast<IT>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<IT>(gridDim.x) * blockDim.x) {
    const IT g = t / per_split;
    const IT r = t - g * per_split;
    const IT bc = r / uP;                          // b * Cout + co
    const int p = static_cast<int>(r - bc * uP);
    const int co = static_cast<int>(bc % uC);
    const float* src = part + static_cast<size_t>(g) * S * per_split + r;
    float acc = src[0];
    for (int s = 1; s < S; ++s) acc += src[static_cast<size_t>(s) * per_split];
    if (shift != nullptr) acc += __ldg(shift + co);
    // the main epilogue's last step, so a split layer gives the unsplit layer's result for every
    // input: the partials are raw, a NaN among them reaches this point as NaN
    acc = ELU ? elu1(acc) : fmaxf(acc, relu ? 0.f : -__int_as_float(0x7f800000));
    int po = p;
    if (scat_w > 0) {
      const int i = p / scat_w, j = p - i * scat_w;
      po = (2 * i + static_cast<int>(g >> 1)) * 2 * scat_w + 2 * j + static_cast<int>(g & 1);
    }
    out[static_cast<long long>(g) * out_gstride + static_cast<size_t>(bc) * P_out + po] = acc;
  }
}

template <bool ELU>
static void launch_splitk_reduce_act(const float* part, int G, int S, int B, int Cout, int P,
                                     const float* shift, int relu, int scat_w, int P_out,
                                     long long out_gstride, float* out, cudaStream_t st) {
  const long long total = static_cast<long long>(B) * Cout * P * G;
  const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, 8LL * sm_count()));
  if (total * std::max(S, 1) < (1LL << 32))
    splitk_reduce_kernel<uint32_t, ELU><<<grid, 256, 0, st>>>(part, G, S, B, Cout, P, shift, relu,
                                                               scat_w, P_out, out_gstride, out);
  else
    splitk_reduce_kernel<unsigned long long, ELU><<<grid, 256, 0, st>>>(part, G, S, B, Cout, P, shift,
                                                                         relu, scat_w, P_out,
                                                                         out_gstride, out);
}

// act: activation code (SONET_ACT_*)
static void launch_splitk_reduce(const float* part, int G, int S, int B, int Cout, int P,
                                 const float* shift, int act, int scat_w, int P_out,
                                 long long out_gstride, float* out, cudaStream_t st) {
  if (act == SONET_ACT_ELU)
    launch_splitk_reduce_act<true>(part, G, S, B, Cout, P, shift, 0, scat_w, P_out, out_gstride, out, st);
  else
    launch_splitk_reduce_act<false>(part, G, S, B, Cout, P, shift, act == SONET_ACT_RELU, scat_w, P_out,
                                    out_gstride, out, st);
}
}  // namespace sonet

static int pointwise_tc_grouped(const float* x, int C, int B, int P, const void* blob,
                                long long blob_gstride, float inv_scale, const float* shift, int Cout,
                                int relu, int groups, int splits, int scat_w, int conv_w, int P_out,
                                long long out_gstride, float* out, float* scratch,
                                sonet_stream_t stream, int nprod, const float* inv_ptr = nullptr,
                                const float* act_ptr = nullptr) {
  using namespace sonet;
  SONET_REQUIRE(groups >= 1 && splits >= 1 && scat_w >= 0, "pointwise_tc_grouped: bad group/split");
  SONET_REQUIRE(scat_w == 0 || (groups == 4 && P % scat_w == 0 && P_out == 4 * P && out_gstride == 0),
                "pointwise_tc_grouped: the x2 scatter needs 4 parity groups, P = H*W, P_out = 4P");
  SONET_REQUIRE(splits == 1 || scratch != nullptr, "pointwise_tc_grouped: split-K needs scratch");
  if (B == 0 || P == 0) return SONET_OK;
  if (P_out <= 0) P_out = P;
  SONET_REQUIRE(conv_w == 0 || conv_w == scat_w, "pointwise_tc_grouped: conv_w must equal scat_w");
  TcExt e = with_nprod(nprod);
  e.inv_ptr = inv_ptr;
  e.act_ptr = act_ptr;
  e.groups = groups;
  e.splits = splits;
  e.blob_gstride = blob_gstride;
  e.conv_w = conv_w;
  if (splits == 1) {
    e.scat_w = scat_w;
    e.P_out = P_out;
    e.out_gstride = out_gstride;
    return launch_pointwise_tc(x, C, nullptr, 0, B, P, blob, inv_scale, shift, Cout, relu, nullptr,
                               nullptr, 0, out, nullptr, stream, e);
  }
  const long long per_split = static_cast<long long>(B) * Cout * P;
  e.out_sstride = per_split;
  e.out_gstride = per_split * splits;
  e.raw = 1;
  int rc = launch_pointwise_tc(x, C, nullptr, 0, B, P, blob, inv_scale, nullptr, Cout, 0, nullptr,
                               nullptr, 0, scratch, nullptr, stream, e);
  if (rc) return rc;
  launch_splitk_reduce(scratch, groups, splits, B, Cout, P, shift, relu, scat_w, P_out, out_gstride, out,
                       as_stream(stream));
  return check_launch("splitk_reduce");
}

extern "C" int sonet_pointwise_tc_grouped_forward(const float* x, int C, int B, int P,
                                                  const void* blob, long long blob_gstride,
                                                  float inv_scale, const float* shift, int Cout,
                                                  int relu, int groups, int splits, int scat_w,
                                                  int conv_w, int P_out, long long out_gstride,
                                                  float* out, float* scratch,
                                                  sonet_stream_t stream) {
  SONET_REQUIRE_ACT(relu, "pointwise_tc_grouped_forward");
  return pointwise_tc_grouped(x, C, B, P, blob, blob_gstride, inv_scale, shift, Cout, relu, groups,
                              splits, scat_w, conv_w, P_out, out_gstride, out, scratch, stream, 3);
}

extern "C" int sonet_pointwise_tc_grouped_forward_f16(const float* x, int C, int B, int P,
                                                      const void* blob, long long blob_gstride,
                                                      float inv_scale, const float* shift, int Cout,
                                                      int relu, int groups, int splits, int scat_w,
                                                      int conv_w, int P_out, long long out_gstride,
                                                      float* out, float* scratch,
                                                      sonet_stream_t stream) {
  SONET_REQUIRE_ACT(relu, "pointwise_tc_grouped_forward_f16");
  return pointwise_tc_grouped(x, C, B, P, blob, blob_gstride, inv_scale, shift, Cout, relu, groups,
                              splits, scat_w, conv_w, P_out, out_gstride, out, scratch, stream, 1);
}

// Train-mode grouped launch (the up-convolution's parity GEMMs): the blobs were packed on the device
// this step (sonet_pointwise_tc_pack_groups_device) and their common 1/pre-scale is read from device
// memory; everything else as sonet_pointwise_tc_grouped_forward.
extern "C" int sonet_pointwise_tc_grouped_forward_dev(const float* x, int C, int B, int P,
                                                      const void* blob, long long blob_gstride,
                                                      const float* inv_scale_dev, const float* shift,
                                                      int Cout, int relu, int groups, int splits,
                                                      int scat_w, int conv_w, int P_out,
                                                      long long out_gstride, float* out, float* scratch,
                                                      sonet_stream_t stream) {
  SONET_REQUIRE_ACT(relu, "pointwise_tc_grouped_forward_dev");
  SONET_REQUIRE(inv_scale_dev != nullptr, "pointwise_tc_grouped_forward_dev: null inv_scale pointer");
  return pointwise_tc_grouped(x, C, B, P, blob, blob_gstride, 1.f, shift, Cout, relu, groups, splits,
                              scat_w, conv_w, P_out, out_gstride, out, scratch, stream, 3, inv_scale_dev);
}

// The one-product twin (SONET_TRAIN_TC=fp16): act_scale_dev, when given, pre-scales the activations
// before their fp16 rounding as in the split entry, so the operand keeps fp16's relative precision
// whatever its fp32 magnitude.
extern "C" int sonet_pointwise_tc_grouped_forward_dev_f16(const float* x, int C, int B, int P,
                                                          const void* blob, long long blob_gstride,
                                                          const float* inv_scale_dev,
                                                          const float* act_scale_dev,
                                                          const float* shift, int Cout, int relu,
                                                          int groups, int splits, int scat_w,
                                                          int conv_w, int P_out, long long out_gstride,
                                                          float* out, float* scratch,
                                                          sonet_stream_t stream) {
  SONET_REQUIRE_ACT(relu, "pointwise_tc_grouped_forward_dev_f16");
  SONET_REQUIRE(inv_scale_dev != nullptr, "pointwise_tc_grouped_forward_dev_f16: null inv_scale pointer");
  return pointwise_tc_grouped(x, C, B, P, blob, blob_gstride, 1.f, shift, Cout, relu, groups, splits,
                              scat_w, conv_w, P_out, out_gstride, out, scratch, stream, 1, inv_scale_dev,
                              act_scale_dev);
}

static int pointwise_tc_dev(const float* x0, int C0, int B, int P, const void* blob,
                            const float* inv_scale_dev, const float* act_scale_dev, const float* shift,
                            int Cout, int relu, int splits, float* out, float* scratch,
                            sonet_stream_t stream, int nprod) {
  using namespace sonet;
  SONET_REQUIRE(inv_scale_dev != nullptr, "pointwise_tc_forward_dev: null inv_scale pointer");
  SONET_REQUIRE(splits >= 1 && (splits == 1 || scratch != nullptr),
                "pointwise_tc_forward_dev: split-K needs scratch");
  TcExt e = with_nprod(nprod);
  e.inv_ptr = inv_scale_dev;
  e.act_ptr = act_scale_dev;
  if (splits == 1)
    return launch_pointwise_tc(x0, C0, nullptr, 0, B, P, blob, 1.f, shift, Cout, relu, nullptr,
                               nullptr, 0, out, nullptr, stream, e);
  const long long per_split = static_cast<long long>(B) * Cout * P;
  e.splits = splits;
  e.out_sstride = per_split;
  e.raw = 1;
  int rc = launch_pointwise_tc(x0, C0, nullptr, 0, B, P, blob, 1.f, nullptr, Cout, 0, nullptr, nullptr,
                               0, scratch, nullptr, stream, e);
  if (rc) return rc;
  launch_splitk_reduce(scratch, 1, splits, B, Cout, P, shift, relu, 0, P, 0, out, as_stream(stream));
  return check_launch("splitk_reduce");
}

// Train-mode variant: the weight blob was packed on the device this step
// (sonet_pointwise_tc_pack_device) and its 1/pre-scale is read from device memory.
extern "C" int sonet_pointwise_tc_forward_dev(const float* x0, int C0, int B, int P, const void* blob,
                                              const float* inv_scale_dev, const float* act_scale_dev,
                                              const float* shift, int Cout, int relu, int splits,
                                              float* out, float* scratch, sonet_stream_t stream) {
  SONET_REQUIRE_ACT(relu, "pointwise_tc_forward_dev");
  return pointwise_tc_dev(x0, C0, B, P, blob, inv_scale_dev, act_scale_dev, shift, Cout, relu, splits,
                          out, scratch, stream, 3);
}

// its one-product twin (SONET_TRAIN_TC=fp16): same arguments and blob, the hi images only
extern "C" int sonet_pointwise_tc_forward_dev_f16(const float* x0, int C0, int B, int P,
                                                  const void* blob, const float* inv_scale_dev,
                                                  const float* act_scale_dev, const float* shift,
                                                  int Cout, int relu, int splits, float* out,
                                                  float* scratch, sonet_stream_t stream) {
  SONET_REQUIRE_ACT(relu, "pointwise_tc_forward_dev_f16");
  return pointwise_tc_dev(x0, C0, B, P, blob, inv_scale_dev, act_scale_dev, shift, Cout, relu, splits,
                          out, scratch, stream, 1);
}

extern "C" int sonet_debug_pointwise_tc_timeline(const float* x0, int C0, int B, int P,
                                                 const void* blob, float inv_scale, int Cout,
                                                 float* out, long long* timeline128,
                                                 sonet_stream_t stream) {
  return launch_pointwise_tc(x0, C0, nullptr, 0, B, P, blob, inv_scale, nullptr, Cout, 1, nullptr,
                             nullptr, 0, out, timeline128, stream);
}
