// nodegemm_tc.cu — the point-wise shared-MLP layer (1x1 conv + folded BN + activation) at node-level
// row counts, as a wgmma GEMM whose two operands both arrive by bulk copy.
//
// The generic layer (csrc/pointwise_tc.cu) converts its activations to fp16 hi/lo images on the MMA
// warpgroups, chunk by chunk, for every out-channel tile again. Over the 49 k rows of the segmenter
// that amortises; over the B*M = 4096 rows of the encoder's final PointNet (515 -> 768 -> 1024) an
// item is a handful of chunks long and the conversion, its fences and its named barriers are most
// of it. Here the images are built once, in global memory:
//
//   * split_pack_kernel writes cat(x0, x1) [B,C,P] as fp16 hi and lo A images, K-major without
//     swizzle (tc::img_off, 8-row x 16-byte core matrices), laid out
//     [128-row tile][32-channel K stage][hi | lo], so one A stage is one contiguous bulk copy.
//     Rows >= B*P and channels >= C are zero. The split is tc::split_words, saturation included:
//     the images hold the bits the generic kernel builds in shared memory;
//   * nodegemm_kernel: an item is a 128-row tile x one n-tile of the weight blob (tc::wblob, up to
//     256 out channels). A producer warp streams A stages from the images and B stages from the
//     blob through one 4-stage mbarrier ring; two consumer warpgroups (64 rows each, 128
//     accumulators per thread at N = 256) wait `full`, issue wgmmas, commit and release `empty`.
//     Per 16-channel K step, in ascending K: hi*hi, lo*hi, hi*lo into one fp32 chain per output,
//     over the same K extent (C rounded up to 16) and with the same epilogue as the generic
//     kernel, so every output has the generic layer's bits;
//   * the epilogue stores either the fp32 tensor [B,Cout,P] or, for a hidden layer, the hi/lo
//     images of its activated output: the next layer's A operand, never held as fp32.
// NPROD = 1 is the opt-in fp16 mode (one product per MAC, the entries' f16 argument): hi images only.
#include <algorithm>

#include "tc_common.cuh"

namespace sonet {
namespace ngt {
constexpr int TILE = 128, KST = tc::wblob::WK, NT = tc::wblob::NT;
constexpr int A_IMG = TILE * KST * 2;           // one fp16 image of an A stage, 8 KB
constexpr int B_IMG = NT * KST * 2;             // one fp16 image of a full-width B stage, 16 KB
constexpr int STAGE_BYTES = 2 * A_IMG + 2 * B_IMG;
constexpr int NSTAGE = 4;
// warpgroups 0-1 consume, warpgroup 2 produces (its warp 8); registers per thread after the
// hand-over: 2 * 128 * 240 + 128 * 24 = 64512, the launch's 168 x 384
constexpr int NUM_THREADS = 384;
constexpr int CONSUMER_REGS = 240, PRODUCER_REGS = 24;
constexpr int OFF_BAR = NSTAGE * STAGE_BYTES;
constexpr int SMEM_BYTES = OFF_BAR + 2 * NSTAGE * 8;
constexpr int PACK_THREADS = 512;               // 128 rows x 4 channel octets of one K stage

__host__ __device__ inline int kstages(int C) { return (C + KST - 1) / KST; }
__host__ __device__ inline long long row_tiles(long long rows) { return (rows + TILE - 1) / TILE; }
// byte offset of the hi image of stage s of row tile `tile`; the lo image follows it
__host__ __device__ inline size_t stage_off(long long tile, int nst, int s, int nimg) {
  return (static_cast<size_t>(tile) * nst + s) * nimg * A_IMG;
}

template <int NPROD>
__global__ void __launch_bounds__(PACK_THREADS)
    split_pack_kernel(const float* __restrict__ x0, int C0, const float* __restrict__ x1, int C1, int B,
                      int P, unsigned char* __restrict__ img) {
  const int s = blockIdx.x, r = threadIdx.x & (TILE - 1), oct = threadIdx.x >> 7;
  const long long R = static_cast<long long>(blockIdx.y) * TILE + r;
  const bool valid = R < static_cast<long long>(B) * P;
  const int b = valid ? static_cast<int>(R / P) : 0;
  const int p = valid ? static_cast<int>(R - static_cast<long long>(b) * P) : 0;
  const float* r0 = x0 + static_cast<size_t>(b) * C0 * P + p;
  const float* r1 = C1 ? x1 + static_cast<size_t>(b) * C1 * P + p : x0;
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = s * KST + oct * 8 + i;
    const float* src = c < C0 ? r0 + static_cast<size_t>(c) * P : r1 + static_cast<size_t>(c - C0) * P;
    v[i] = (valid && c < C0 + C1) ? __ldg(src) : 0.f;
  }
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) tc::split_words<NPROD>(v[2 * j], v[2 * j + 1], hi[j], lo[j]);
  unsigned char* dst = img + stage_off(blockIdx.y, gridDim.x, s, NPROD == 3 ? 2 : 1) +
                       tc::img_off(r, oct * 8, KST);
  *reinterpret_cast<uint4*>(dst) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  if (NPROD == 3) *reinterpret_cast<uint4*>(dst + A_IMG) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

struct Dims {
  int Cin, B, P, Cout, relu;
  int nst;        // K stages of the input images
  int nst_out;    // K stages of the output images (image mode)
  int ksteps;     // 16-channel K steps: Cin rounded up to 16, the generic layer's K extent
  int kch;        // 64-channel chunks of the weight blob
  int ntiles;     // n-tiles of the blob
  int row_tiles;
  float inv;      // 1 / weight pre-scale
};

// one wgmma of N = 64, 128 or 256 columns
template <int N>
__device__ __forceinline__ void mma_n(float (&acc)[N / 2], uint64_t a, uint64_t b) {
  if constexpr (N == 256) tc::wgmma_f16_n256(acc, a, b, 1);
  else if constexpr (N == 128) tc::wgmma_f16_n128(acc, a, b, 1);
  else tc::wgmma_f16_n64(acc, a, b, 1);
}

// One item of a consumer warpgroup: 64 rows x the NW = 64, 128, 192 or 256 columns of n-tile nt,
// as one wgmma of N0 columns plus, at NW = 192, one of 64. q: ring position (stages consumed).
template <int NW, int NPROD, bool ELU>
__device__ __forceinline__ void run_item(const Dims& d, int tile, int nt, int wg, int warp, int lane,
                                         unsigned char* smem, uint64_t* full, uint64_t* empty,
                                         uint32_t& q, const float* __restrict__ shift,
                                         unsigned char* __restrict__ img_out, float* __restrict__ out) {
  constexpr int NIMG = NPROD == 3 ? 2 : 1;
  constexpr int N0 = NW == 192 ? 128 : NW, N1 = NW - N0;
  constexpr uint32_t B1_OFF = N0 / 8 * KST * 16;   // the second piece's rows of a B image
  const long long rows = static_cast<long long>(d.B) * d.P;
  const float floor_v = d.relu ? 0.f : -__int_as_float(0x7f800000);   // ReLU as one max
  float acc0[N0 / 2], acc1[N1 ? N1 / 2 : 32];
#pragma unroll
  for (int i = 0; i < N0 / 2; ++i) acc0[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) acc1[i] = 0.f;
  uint32_t prev_slot = 0;
#pragma unroll 1
  for (int s = 0; s < d.nst; ++s, ++q) {
    const uint32_t slot = q % NSTAGE;
    tc::mbar_wait_bounded(&full[slot], (q / NSTAGE) & 1, 211);
    const uint32_t a_hi = smem_u32(smem) + slot * STAGE_BYTES + wg * (A_IMG / 2);
    const uint32_t b_hi = smem_u32(smem) + slot * STAGE_BYTES + 2 * A_IMG;
    const uint32_t b_lo = b_hi + NW * KST * 2;
    const int nks = min(2, d.ksteps - 2 * s);
    tc::wg_fence();
#pragma unroll 1
    for (int ks = 0; ks < nks; ++ks) {
      // A: [64 x 32] rows of this warpgroup; B: [NW x 32]; both LBO 128, SBO 512
      const uint64_t ah = tc::smem_desc(a_hi + ks * 256, 128, KST * 16);
      const uint64_t al = tc::smem_desc(a_hi + A_IMG + ks * 256, 128, KST * 16);
      const uint64_t bh = tc::smem_desc(b_hi + ks * 256, 128, KST * 16);
      const uint64_t bl = tc::smem_desc(b_lo + ks * 256, 128, KST * 16);
      mma_n<N0>(acc0, ah, bh);
      if (NPROD == 3) {
        mma_n<N0>(acc0, al, bh);
        mma_n<N0>(acc0, ah, bl);
      }
      if constexpr (N1 != 0) {
        mma_n<64>(acc1, ah, bh + (B1_OFF >> 4));
        if (NPROD == 3) {
          mma_n<64>(acc1, al, bh + (B1_OFF >> 4));
          mma_n<64>(acc1, ah, bl + (B1_OFF >> 4));
        }
      }
    }
    tc::wg_commit();
    tc::wg_wait<1>();   // the previous stage is complete for this warp
    if (s > 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev_slot]);
    }
    prev_slot = slot;
  }
  tc::wg_wait<0>();
  __syncwarp();
  if (lane == 0) mbar_arrive(&empty[prev_slot]);

  // ---- epilogue: thread holds rows r0 = 16*(warp%4) + lane/4 and r0 + 8 of its warpgroup,
  // columns 8j + 2*(lane%4) + {0,1} (accumulators 4j+{0,1} and 4j+{2,3}) ----
  const int col0 = nt * NT + 2 * (lane & 3);
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int r = wg * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * rr;
    const long long R = static_cast<long long>(tile) * TILE + r;
    const bool valid = R < rows;
    const int b = valid ? static_cast<int>(R / d.P) : 0;
    const int p = valid ? static_cast<int>(R - static_cast<long long>(b) * d.P) : 0;
    float* o = out + static_cast<size_t>(b) * d.Cout * d.P + p;
    // image mode: the column pair is one fp16x2 word of the hi and of the lo image of the next
    // layer's A operand; a warp store fills one 128-byte core matrix
    unsigned char* oi = img_out + (r >> 3) * (KST * 16) + (r & 7) * 16;
#pragma unroll
    for (int j = 0; j < NW / 8; ++j) {
      float y[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int co = col0 + 8 * j + e;
        const float a = j < N0 / 8 ? acc0[(4 * j + 2 * rr + e) % (N0 / 2)]
                                   : acc1[(4 * (j - N0 / 8) + 2 * rr + e) % 32];
        y[e] = fmaf(a, d.inv, (shift != nullptr && co < d.Cout) ? __ldg(shift + co) : 0.f);
        y[e] = ELU ? elu1(y[e]) : fmaxf(y[e], floor_v);
        if (img_out == nullptr && valid && co < d.Cout) o[static_cast<size_t>(co) * d.P] = y[e];
        if (!valid || co >= d.Cout) y[e] = 0.f;   // image padding
      }
      const int co = col0 + 8 * j;
      if (img_out != nullptr && (co >> 5) < d.nst_out) {
        uint32_t hi, lo;
        tc::split_words<NPROD>(y[0], y[1], hi, lo);
        unsigned char* w = oi + stage_off(tile, d.nst_out, co >> 5, NIMG) + ((co & 31) >> 3) * 128 +
                           (co & 7) * 2;
        *reinterpret_cast<uint32_t*>(w) = hi;
        if (NPROD == 3) *reinterpret_cast<uint32_t*>(w + A_IMG) = lo;
      }
    }
  }
}

template <int NPROD, bool ELU>
__global__ void __launch_bounds__(NUM_THREADS, 1)
    nodegemm_kernel(const unsigned char* __restrict__ img, const unsigned char* __restrict__ blob,
                    const float* __restrict__ shift, unsigned char* __restrict__ img_out,
                    float* __restrict__ out, Dims d) {
  constexpr int NIMG = NPROD == 3 ? 2 : 1;
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + OFF_BAR);   // [NSTAGE] producer -> MMA
  uint64_t* empty = full + NSTAGE;                                // [NSTAGE] MMA -> producer

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int items = d.row_tiles * d.ntiles;
  const int my_items =
      (static_cast<int>(blockIdx.x) < items) ? (items - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);   // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ================= producer: one A stage and one B stage per ring slot =================
    tc::regs_dec<PRODUCER_REGS>();
    if (warp == 8 && lane == 0) {
      uint32_t q = 0;
      for (int it = 0; it < my_items; ++it) {
        const int item = blockIdx.x + it * gridDim.x;
        const int nt = item % d.ntiles, tile = item / d.ntiles;   // n-tile fastest: A stays in L2
        const uint32_t b_bytes = static_cast<uint32_t>(tc::wblob::tile_width(d.Cout, nt)) * KST * 2 * NIMG;
        for (int s = 0; s < d.nst; ++s, ++q) {
          const uint32_t slot = q % NSTAGE, use = q / NSTAGE;
          if (use > 0) tc::mbar_wait_relaxed(&empty[slot], (use - 1) & 1, 210);
          mbar_arrive_expect_tx(&full[slot], NIMG * A_IMG + b_bytes);
          unsigned char* dst = smem + slot * STAGE_BYTES;
          bulk_g2s(dst, img + stage_off(tile, d.nst, s, NIMG), NIMG * A_IMG, &full[slot]);
          // hi image, then (NPROD == 3) the lo image right behind it, as the blob stores them
          bulk_g2s(dst + 2 * A_IMG, blob + tc::wblob::stage_off(d.Cout, d.kch, nt, s >> 1, s & 1),
                   b_bytes, &full[slot]);
        }
      }
    }
    return;
  }

  // ================= consumers: 64 rows x the n-tile each =================
  tc::regs_inc<CONSUMER_REGS>();
  const int wg = warp >> 2;
  uint32_t q = 0;
  for (int it = 0; it < my_items; ++it) {
    const int item = blockIdx.x + it * gridDim.x;
    const int nt = item % d.ntiles, tile = item / d.ntiles;
    switch (tc::wblob::tile_width(d.Cout, nt)) {
      case 256: run_item<256, NPROD, ELU>(d, tile, nt, wg, warp, lane, smem, full, empty, q, shift, img_out, out); break;
      case 192: run_item<192, NPROD, ELU>(d, tile, nt, wg, warp, lane, smem, full, empty, q, shift, img_out, out); break;
      case 128: run_item<128, NPROD, ELU>(d, tile, nt, wg, warp, lane, smem, full, empty, q, shift, img_out, out); break;
      default: run_item<64, NPROD, ELU>(d, tile, nt, wg, warp, lane, smem, full, empty, q, shift, img_out, out); break;
    }
  }
}

}  // namespace ngt
}  // namespace sonet

extern "C" long long sonet_nodegemm_image_bytes(long long rows, int C, int f16) {
  using namespace sonet::ngt;
  if (rows < 0 || C < 1) return -1;
  return static_cast<long long>(stage_off(row_tiles(rows), kstages(C), 0, f16 ? 1 : 2));
}

extern "C" int sonet_nodegemm_split_pack(const float* x0, int C0, const float* x1, int C1, int B, int P,
                                         int f16, void* img, sonet_stream_t stream) {
  using namespace sonet;
  using namespace sonet::ngt;
  SONET_REQUIRE(B >= 0 && P >= 0 && C0 >= 1 && C1 >= 0, "nodegemm_split_pack: bad dimension");
  if (B == 0 || P == 0) return SONET_OK;
  SONET_REQUIRE(x0 && img, "nodegemm_split_pack: null pointer");
  SONET_REQUIRE(C1 == 0 || x1 != nullptr, "nodegemm_split_pack: x1 null with C1=%d", C1);
  SONET_REQUIRE(aligned16(img), "nodegemm_split_pack: the images must be 16-byte aligned");
  const long long tiles = row_tiles(static_cast<long long>(B) * P);
  SONET_REQUIRE(tiles <= 65535, "nodegemm_split_pack: too many rows");
  const dim3 grid(kstages(C0 + C1), static_cast<unsigned>(tiles));
  auto kern = f16 ? split_pack_kernel<1> : split_pack_kernel<3>;
  kern<<<grid, PACK_THREADS, 0, as_stream(stream)>>>(x0, C0, x1, C1, B, P,
                                                     static_cast<unsigned char*>(img));
  return check_launch("nodegemm_split_pack");
}

extern "C" int sonet_nodegemm_tc_forward(const void* img, int Cin, int B, int P, const void* blob,
                                         float inv_scale, const float* shift, int Cout, int act,
                                         int f16, void* img_out, float* out, sonet_stream_t stream) {
  using namespace sonet;
  using namespace sonet::ngt;
  SONET_REQUIRE_ACT(act, "nodegemm_tc_forward");
  SONET_REQUIRE(B >= 0 && P >= 0 && Cin >= 1 && Cout >= 1, "nodegemm_tc_forward: bad dimension");
  if (B == 0 || P == 0) return SONET_OK;
  SONET_REQUIRE(img && blob, "nodegemm_tc_forward: null pointer");
  SONET_REQUIRE((img_out != nullptr) != (out != nullptr),
                "nodegemm_tc_forward: exactly one of img_out and out");
  SONET_REQUIRE(aligned16(img) && aligned16(blob) && aligned16(img_out),
                "nodegemm_tc_forward: images and weight blob must be 16-byte aligned");
  Dims d;
  d.Cin = Cin; d.B = B; d.P = P; d.Cout = Cout; d.relu = act == SONET_ACT_RELU;
  d.nst = kstages(Cin);
  d.nst_out = kstages(Cout);
  d.ksteps = (Cin + 15) / 16;
  d.kch = tc::wblob::kchunks(Cin);
  d.ntiles = (tc::wblob::npad(Cout) + NT - 1) / NT;
  d.inv = inv_scale;
  const long long tiles = row_tiles(static_cast<long long>(B) * P);
  SONET_REQUIRE(tiles * d.ntiles < (1LL << 31), "nodegemm_tc_forward: too many tiles");
  d.row_tiles = static_cast<int>(tiles);
  SONET_REQUIRE(SMEM_BYTES <= max_smem_optin(), "nodegemm_tc_forward: needs %d B of shared memory",
                SMEM_BYTES);
  auto kern = act == SONET_ACT_ELU ? (f16 ? nodegemm_kernel<1, true> : nodegemm_kernel<3, true>)
                                   : (f16 ? nodegemm_kernel<1, false> : nodegemm_kernel<3, false>);
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  const int grid = static_cast<int>(std::min<long long>(tiles * d.ntiles, sm_count()));
  kern<<<grid, NUM_THREADS, SMEM_BYTES, as_stream(stream)>>>(
      static_cast<const unsigned char*>(img), static_cast<const unsigned char*>(blob), shift,
      static_cast<unsigned char*>(img_out), out, d);
  return check_launch("nodegemm_tc_forward");
}
