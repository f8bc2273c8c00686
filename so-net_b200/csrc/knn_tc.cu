// knn_tc.cu — the encoder's KNN module (models/layers.py:299-367: gather the K neighbour nodes,
// decentre, 1x1 conv 387 -> 512 -> 512 with BN + ReLU, max over the K neighbours) as ONE wgmma
// kernel for sm_90a, after a per-node GEMM for the feature part of layer 1.
//
// Layer 1 is linear in its input [dec; f(nbr)], so W1 [dec; f(nbr)] = W1d dec + (W1f f)(nbr): the
// 384 feature channels are the same vector for every row that gathers node nbr. The caller computes
// Y = W1f x once per NODE (the generic wgmma layer without shift or ReLU, 9x fewer rows than per
// (node, neighbour) row at som_k = 9), stored node-major [B,M,512] by the layer's point-major store
// mode; a channel-major [B,512,M] Y is accepted too (scalar loads, same results). This kernel then
// runs, per row (node m, neighbour j):
//
//   * layer-1 epilogue on CUDA cores: h1 = act(W1d . dec + Y[b,:,nbr] + shift1) in fp32 (ReLU or ELU), with
//     dec = coord[b,:,nbr] - center[b,:,m] (the same __fsub_rn as knn_assemble). Each thread builds
//     its part of the register A operand of m64k16 (2 rows x 8 channels, fp16 hi/lo) right before
//     the wgmmas of that K block; h1 never exists in memory. From a node-major Y a thread loads its
//     8 values of a K block as 4 float2 (a warp instruction reads 8 rows x 32 B, one sector each);
//     the loads of block kk+3 are issued while block kk's wgmmas run, into the buffer the build of
//     kk+1 just read (double-buffered), so each load has two blocks of wgmmas to land;
//   * layer 2 (512 -> 512) on wgmma with the fp16 hi/lo 3-product split, fp32 accumulators, in two
//     N halves of 256 (passes; 128 accumulators per thread); each pass builds its own A operand;
//   * max over the K neighbours on the RAW accumulators: y = act(fmaf(raw, inv2 > 0, shift2)) is
//     monotone (non-decreasing) in raw for both activations the kernel is built for: fmaf by a
//     positive constant and a round-to-nearest are, ReLU is, and so is ELU — x for x > 0, and
//     expm1f, non-decreasing in x, maps x <= 0 into (-1, 0], below every positive output. So
//     max_rows(y) == act(fmaf(max_rows(raw), inv2, shift2)) bit for bit (the argument of the POOL
//     epilogue of pointmlp_tc.cu). A non-monotone activation (swish) would break this. Every row reduces into per-node shared-memory
//     keys, which the warpgroup converts and stores as knn_feature_1 [B,512,M]. h2 is never written.
//     (A segmented shuffle reduction in front of the atomics spilled the accumulators; a
//     __match_any_sync + __reduce_max_sync one made the epilogue ~10x slower, as redux.sync with
//     lane-dependent masks serialises.)
//   * non-finite inputs: layer 1's ReLU maps a NaN to 0. Under ELU a NaN h1 makes its whole layer-2
//     row NaN; the wgmma returns that NaN with the sign bit clear (for NaN inputs of either sign),
//     so its key lies above +inf's and the node is NaN in every channel, as rowmax gives. +-inf
//     saturates in the split like any |h1| >= 131008 (-inf: h1 = 0 or -1). Ids are clamped to
//     [0, M-1]; padding rows read node 0 of cloud 0 and never reach a key
//     (tests/test_gpu_knn_envelope.py).
//
// Rows: a warpgroup owns a BLOCK of floor(64/K) whole consecutive nodes of the flattened (cloud,
// node) sequence (7 nodes = 63 rows at K = 9), so no node is split across warpgroups or CTAs and no
// global atomics are needed. A tile is two blocks (one per consumer warpgroup); a work item is one
// (tile, pass) pair, 2 x ceil(blocks / 2) items over min(items, SMs) CTAs, which shortens the
// critical path of the last round against whole tiles (cfg-2: 586 items, not 293 tiles of twice
// the work, over 132 SMs). Per item the producer thread streams the pass's half of the 1 MB
// layer-2 weight stream, 16 stages of [256 out x 32 k] hi|lo, 32 KB each, through a 4-slot ring
// (cp.async.bulk + mbarrier). Warp roles and the register hand-over (setmaxnreg 240 / 24) follow
// pointmlp_tc.cu.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "tc_common.cuh"

namespace sonet {

namespace kt {
constexpr int C1 = 512, C2 = 512;        // hidden and output widths (KNNModule (512, 512))
constexpr int NH = 256, NPASS = C2 / NH; // out channels per pass
constexpr int KT = 32;                   // K extent of one weight stage
constexpr int KSTAGES = C1 / KT;         // 16 stages per pass
constexpr int STAGES_PER_TILE = NPASS * KSTAGES;
constexpr int STAGE_BYTES = NH * KT * 2 * 2;          // hi + lo, 32 KB
constexpr int BLOB_BYTES = STAGES_PER_TILE * STAGE_BYTES;   // 1 MB
constexpr int NSLOT = 4;
constexpr int MAX_K = 16, MIN_K = 2;
constexpr int MAX_NPB = 64 / MIN_K;      // nodes per block
constexpr int KEY_LD = NH + 8;           // padded key row: leaders of adjacent nodes hit other banks
constexpr int NUM_THREADS = 384;
constexpr int CONSUMER_REGS = 240, PRODUCER_REGS = 24;
constexpr int OFF_RING = 0;
constexpr int OFF_W1 = OFF_RING + NSLOT * STAGE_BYTES;          // float4 {w1d[0..2], shift1} x C1
constexpr int OFF_SH2 = OFF_W1 + C1 * 16;                       // shift2 [C2]
constexpr int OFF_KEYS = OFF_SH2 + C2 * 4;                      // [2 wg][MAX_NPB][KEY_LD] int
constexpr int OFF_BAR = OFF_KEYS + 2 * MAX_NPB * KEY_LD * 4;
constexpr int SMEM_BYTES = OFF_BAR + 2 * NSLOT * 8;
}  // namespace kt

struct KnnArgs {
  const float* coord;     // [B,3,M]
  const float* center;    // [B,3,M]
  const int64_t* idx;     // [B,M,Kstride]
  const float* Y;         // element (b, c, n) at Y[b*C1*M + c*y_cs + n*y_ns]
  const float* w1;        // [C1][4] {W1d[c,0..2], shift1[c]}
  const float* shift2;    // [C2]
  float inv2;
  int B, M, K, Kstride;
  int npb, nblocks;
  long long y_cs, y_ns;
  float* out;             // [B,C2,M]
};

// YVEC: Y is node-major (y_cs == 1), so channels (c, c+1) of a row are one float2.
// NPROD: fp16 products per MAC in layer 2, 3 (the hi/lo split) or 1 (hi only, the opt-in fp16 mode:
// the A fragments carry no lo words and the producer copies the hi half of each stage).
// ACT: the activation of both layers, SONET_ACT_RELU or SONET_ACT_ELU.
template <bool YVEC, int NPROD, int ACT>
__global__ void __launch_bounds__(kt::NUM_THREADS, 1)
    knn_mlp_tc_kernel(const unsigned char* __restrict__ blob, KnnArgs a, long long* __restrict__ dbg) {
  using namespace kt;
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* empty = full + NSLOT;
  const float4* w1s = reinterpret_cast<const float4*>(smem + OFF_W1);
  const float* sh2 = reinterpret_cast<const float*>(smem + OFF_SH2);

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  if (dbg != nullptr && blockIdx.x == 0 && threadIdx.x == 0) dbg[64 + 62] = clock64();
  // work item = (tile, pass): item 2t + p is pass p of tile t, so the two passes of a tile run on
  // neighbouring CTAs of the same round and share their Y rows in L2
  const int num_items = 2 * ((a.nblocks + 1) / 2);
  const int my_items = (static_cast<int>(blockIdx.x) < num_items)
                           ? (num_items - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  for (int i = threadIdx.x; i < C1 * 4; i += NUM_THREADS)
    reinterpret_cast<float*>(smem + OFF_W1)[i] = __ldg(a.w1 + i);
  for (int i = threadIdx.x; i < C2; i += NUM_THREADS)
    reinterpret_cast<float*>(smem + OFF_SH2)[i] = __ldg(a.shift2 + i);
  for (int i = threadIdx.x; i < 2 * MAX_NPB * KEY_LD; i += NUM_THREADS)
    reinterpret_cast<int*>(smem + OFF_KEYS)[i] = POOL_KEY_INIT;
  if (threadIdx.x == 0) {
    for (int s = 0; s < NSLOT; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);   // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // =========================== TMA producer ===========================
    tc::regs_dec<PRODUCER_REGS>();
    if (warp == 8 && lane == 0) {
      uint32_t q = 0;
#pragma unroll 1
      for (int it = 0; it < my_items; ++it) {
        const int pass = (blockIdx.x + it * gridDim.x) & 1;
#pragma unroll 1
        for (int s = 0; s < KSTAGES; ++s, ++q) {
          const uint32_t slot = q % NSLOT, use = q / NSLOT;
          if (use > 0) tc::mbar_wait_relaxed(&empty[slot], (use - 1) & 1, 300 + s);
          constexpr uint32_t bytes = NPROD == 3 ? STAGE_BYTES : STAGE_BYTES / 2;   // [hi | lo]
          mbar_arrive_expect_tx(&full[slot], bytes);
          bulk_g2s(smem + OFF_RING + slot * STAGE_BYTES,
                   blob + static_cast<size_t>(KSTAGES * pass + s) * STAGE_BYTES, bytes,
                   &full[slot]);
        }
      }
    }
  } else {
    // =========================== consumer warpgroups ===========================
    tc::regs_inc<CONSUMER_REGS>();
    constexpr unsigned FULL = 0xffffffffu;
    const int wg = warp >> 2;
    const int tw = threadIdx.x & 127;
    const uint32_t ring_a = smem_u32(smem + OFF_RING);
    int* keys = reinterpret_cast<int*>(smem + OFF_KEYS) + wg * MAX_NPB * KEY_LD;
    // accumulator fragment: rows r0 = 16*(warp%4) + lane/4 and r0 + 8 of the warpgroup's 64,
    // columns 8j + 2*(lane%4) + {0,1} (registers 4j+{0,1} for r0, 4j+{2,3} for r0 + 8)
    const int r0 = 16 * (warp & 3) + (lane >> 2);
    const int cq = 2 * (lane & 3);
    const int rows_pb = a.npb * a.K;
    const long long nodes = static_cast<long long>(a.B) * a.M;
    uint32_t q = 0;

    auto stage_wait = [&]() -> uint32_t {
      const uint32_t slot = q % NSLOT;
      tc::mbar_wait_bounded(&full[slot], (q / NSLOT) & 1, 3);
      return ring_a + slot * STAGE_BYTES;
    };
    auto stage_release = [&](uint32_t qq) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[qq % NSLOT]);
    };

    // clock64 stamps of CTA 0, per warpgroup and item (it < 15): [64 wg + 4 it + phase], phase 0
    // item start, 1 first wgmma issued, 2 last wgmma retired, 3 epilogue done
    long long* stamp = (dbg != nullptr && blockIdx.x == 0 && tw == 0) ? dbg + 64 * wg : nullptr;

#pragma unroll 1
    for (int it = 0; it < my_items; ++it) {
      const int item = blockIdx.x + it * gridDim.x;
      const int pass = item & 1;
      const int block = 2 * (item >> 1) + wg;
      if (stamp != nullptr && it < 15) stamp[4 * it] = clock64();
      const long long gnode0 = static_cast<long long>(block) * a.npb;
      // this thread's two rows: block-local node (-1 = padding), Y base of the neighbour node,
      // decentred coords
      int ln[2];
      const float* yrow[2];
      float dec[2][3];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int lr = r0 + 8 * rr;
        const long long g = gnode0 + lr / a.K;
        ln[rr] = -1;
        yrow[rr] = a.Y;
        dec[rr][0] = dec[rr][1] = dec[rr][2] = 0.f;
        if (block < a.nblocks && lr < rows_pb && g < nodes) {
          const int b = static_cast<int>(g / a.M), m = static_cast<int>(g - static_cast<long long>(b) * a.M);
          const int j = lr - (lr / a.K) * a.K;
          const long long w = a.idx[(static_cast<size_t>(b) * a.M + m) * a.Kstride + j];
          const int nbr = static_cast<int>(w < 0 ? 0 : (w > a.M - 1 ? a.M - 1 : w));
          ln[rr] = lr / a.K;
          yrow[rr] = a.Y + static_cast<size_t>(b) * C1 * a.M + static_cast<size_t>(nbr) * a.y_ns;
#pragma unroll
          for (int c = 0; c < 3; ++c)
            dec[rr][c] = __fsub_rn(__ldg(a.coord + (static_cast<size_t>(b) * 3 + c) * a.M + nbr),
                                   __ldg(a.center + (static_cast<size_t>(b) * 3 + c) * a.M + m));
        }
      }
      // Y values of K block kk: word i of the A fragment = row i&1, channels 16kk + 8(i>>1) + cq + {0,1}
      auto load_y = [&](int kk, float (&yv)[8]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int c = 16 * kk + 8 * (i >> 1) + cq;
          if (YVEC) {
            const float2 v = __ldg(reinterpret_cast<const float2*>(yrow[i & 1] + c));
            yv[2 * i] = v.x;
            yv[2 * i + 1] = v.y;
          } else {
#pragma unroll
            for (int e = 0; e < 2; ++e)
              yv[2 * i + e] = __ldg(yrow[i & 1] + static_cast<size_t>(c + e) * a.y_cs);
          }
        }
      };
      auto build = [&](int kk, const float (&yv)[8], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float h[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float4 w = w1s[16 * kk + 8 * (i >> 1) + cq + e];
            const float* d = dec[i & 1];
            float v = yv[2 * i + e] + w.w;
            v = fmaf(w.x, d[0], v);
            v = fmaf(w.y, d[1], v);
            v = fmaf(w.z, d[2], v);
            h[e] = act_fn<ACT>(v);
          }
          tc::split_words<NPROD>(h[0], h[1], hi[i], lo[i]);
        }
      };

      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      uint32_t fh[2][4], fl[2][4];
      // Y of block kk lives in yv[kk & 1] from two blocks before its build until the build
      float yv[2][8];
      load_y(0, yv[0]);
      load_y(1, yv[1]);
      build(0, yv[0], fh[0], fl[0]);
      load_y(2, yv[0]);
#pragma unroll 1
      for (int st = 0; st < KSTAGES; ++st) {
        const uint32_t sb = stage_wait();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
          const int kk = 2 * st + ks;
          const uint64_t bh = tc::smem_desc(sb + ks * 256, 128, 512),
                         bl = tc::smem_desc(sb + STAGE_BYTES / 2 + ks * 256, 128, 512);
          tc::wg_fence();
          tc::wgmma_f16_rs_n256(acc, fh[ks], bh, 1);
          if (NPROD == 3) {
            tc::wgmma_f16_rs_n256(acc, fl[ks], bh, 1);
            tc::wgmma_f16_rs_n256(acc, fh[ks], bl, 1);
          }
          tc::wg_commit();
          if (kk == 0 && stamp != nullptr && it < 15) stamp[4 * it + 1] = clock64();
          // K block kk-1 has retired: its fragment buffer is free, and so is its stage if it
          // was the stage's second block
          tc::wg_wait<1>();
          if (ks == 0 && st > 0) stage_release(q - 1);
          if (kk + 1 < 2 * KSTAGES) {
            build(kk + 1, yv[ks ^ 1], fh[ks ^ 1], fl[ks ^ 1]);
            if (kk + 3 < 2 * KSTAGES) load_y(kk + 3, yv[ks ^ 1]);
          }
        }
        ++q;
      }
      tc::wg_wait<0>();
      stage_release(q - 1);
      if (stamp != nullptr && it < 15) stamp[4 * it + 2] = clock64();

      // ---- max over each node's rows: every thread reduces its raw accumulators into the
      // node's shared-memory keys (order-preserving ints); rows of one node share an address ----
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (ln[rr] < 0) continue;
        int* kr = keys + ln[rr] * KEY_LD + cq;
#pragma unroll
        for (int jn = 0; jn < 32; ++jn)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int bits = __float_as_int(acc[4 * jn + 2 * rr + e]);
            atomicMax(kr + 8 * jn + e, bits ^ ((bits >> 31) & 0x7fffffff));
          }
      }
      tc::named_sync(1 + wg, 128);
      // keys -> knn_feature_1[b, NH*pass + c, m] for the block's nodes; reset for the next item.
      // The block's nodes are consecutive from (b0, m0): one 64-bit division per item, not per
      // output (padding blocks start at b0 >= B)
      const int b0 = static_cast<int>(gnode0 / a.M);
      const int m0 = static_cast<int>(gnode0 - static_cast<long long>(b0) * a.M);
#pragma unroll 4
      for (int i = tw; i < a.npb * NH; i += 128) {
        const int c = i / a.npb, l = i - c * a.npb;
        int b = b0, m = m0 + l;
        while (m >= a.M) {   // a block can span clouds (and several when M < npb)
          m -= a.M;
          ++b;
        }
        int* kp = keys + l * KEY_LD + c;
        if (b < a.B) {
          const int key = *kp;
          const float raw = __int_as_float(key ^ ((key >> 31) & 0x7fffffff));
          const int co = NH * pass + c;
          a.out[(static_cast<size_t>(b) * C2 + co) * a.M + m] = act_fn<ACT>(fmaf(raw, a.inv2, sh2[co]));
        }
        *kp = POOL_KEY_INIT;
      }
      tc::named_sync(1 + wg, 128);
      if (stamp != nullptr && it < 15) stamp[4 * it + 3] = clock64();
    }
  }
  __syncthreads();
  if (dbg != nullptr && blockIdx.x == 0 && threadIdx.x == 0) dbg[64 + 63] = clock64();
}

}  // namespace sonet

extern "C" long long sonet_knn_mlp_tc_blob_bytes(void) { return sonet::kt::BLOB_BYTES; }

extern "C" int sonet_knn_mlp_tc_pack(const float* W2, void* blob_host, float* inv_scale) {
  using namespace sonet;
  using namespace sonet::kt;
  SONET_REQUIRE(W2 && blob_host && inv_scale, "knn_mlp_tc_pack: null pointer");
  unsigned char* blob = static_cast<unsigned char*>(blob_host);
  const float s = pow2_scale(W2, static_cast<size_t>(C2) * C1);
  size_t off = 0;
  for (int p = 0; p < NPASS; ++p)
    for (int ks = 0; ks < KSTAGES; ++ks) {
      pack_tile(W2, s, C1, NH * p, NH, KT * ks, KT, blob + off, blob + off + STAGE_BYTES / 2);
      off += STAGE_BYTES;
    }
  *inv_scale = 1.f / s;
  return SONET_OK;
}

static int launch_knn_mlp_tc(const float* coord, const float* center, const int64_t* idx, int B, int M,
                             int K, int Kstride, const float* Y, long long y_cs, long long y_ns,
                             const float* w1, const void* blob, float inv2, const float* shift2,
                             float* out, long long* dbg, sonet_stream_t stream, bool f16 = false,
                             int act = SONET_ACT_RELU) {
  using namespace sonet;
  using namespace sonet::kt;
  SONET_REQUIRE(act == SONET_ACT_RELU || act == SONET_ACT_ELU,
                "knn_mlp_tc: activation code %d is not SONET_ACT_RELU (1) or _ELU (2)", act);
  SONET_REQUIRE(B >= 0 && M >= 1 && Kstride >= K, "knn_mlp_tc: bad dimension");
  SONET_REQUIRE(K >= MIN_K && K <= MAX_K, "knn_mlp_tc: K=%d out of range [%d,%d]", K, MIN_K, MAX_K);
  SONET_REQUIRE(M <= 65535, "knn_mlp_tc: M=%d too large", M);
  // Y [B] x [512 channels, M nodes] in either order: channel-major (y_cs = M, y_ns = 1) or
  // node-major (y_cs = 1, y_ns = 512)
  SONET_REQUIRE((y_cs == M && y_ns == 1) || (y_cs == 1 && y_ns == C1),
                "knn_mlp_tc: Y strides (%lld, %lld) are neither [B,512,M] nor [B,M,512]", y_cs, y_ns);
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(coord && center && idx && Y && w1 && blob && shift2 && out, "knn_mlp_tc: null pointer");
  SONET_REQUIRE(aligned16(blob) && aligned16(w1), "knn_mlp_tc: blob and w1 must be 16-byte aligned");
  SONET_REQUIRE(y_cs != 1 || reinterpret_cast<uintptr_t>(Y) % 8 == 0,
                "knn_mlp_tc: node-major Y must be 8-byte aligned");
  SONET_REQUIRE(inv2 > 0.f, "knn_mlp_tc: inv_scale must be positive");
  KnnArgs a{coord, center, idx, Y, w1, shift2, inv2, B, M, K, Kstride, 64 / K, 0, y_cs, y_ns, out};
  const long long nodes = static_cast<long long>(B) * M;
  const long long nblocks = (nodes + a.npb - 1) / a.npb;
  SONET_REQUIRE(nblocks < (1LL << 30), "knn_mlp_tc: too many nodes");
  a.nblocks = static_cast<int>(nblocks);
  SONET_REQUIRE(SMEM_BYTES <= max_smem_optin(), "knn_mlp_tc: needs %d B of shared memory", SMEM_BYTES);
  const long long items = 2 * ((nblocks + 1) / 2);   // (tile, pass) pairs
  const int grid = static_cast<int>(std::min<long long>(items, sm_count()));
  constexpr int R = SONET_ACT_RELU, E = SONET_ACT_ELU;
  auto kernel =
      act == E ? (f16 ? (y_cs == 1 ? knn_mlp_tc_kernel<true, 1, E> : knn_mlp_tc_kernel<false, 1, E>)
                      : (y_cs == 1 ? knn_mlp_tc_kernel<true, 3, E> : knn_mlp_tc_kernel<false, 3, E>))
               : f16 ? (y_cs == 1 ? knn_mlp_tc_kernel<true, 1, R> : knn_mlp_tc_kernel<false, 1, R>)
                     : (y_cs == 1 ? knn_mlp_tc_kernel<true, 3, R> : knn_mlp_tc_kernel<false, 3, R>);
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  kernel<<<grid, NUM_THREADS, SMEM_BYTES, as_stream(stream)>>>(static_cast<const unsigned char*>(blob),
                                                               a, dbg);
  return check_launch("knn_mlp_tc");
}

extern "C" int sonet_knn_mlp_tc_forward(const float* coord, const float* center, const int64_t* idx,
                                        int B, int M, int K, int Kstride, const float* Y,
                                        long long y_cstride, long long y_nstride, const float* w1,
                                        const void* blob, float inv_scale, const float* shift2,
                                        float* out, sonet_stream_t stream) {
  return launch_knn_mlp_tc(coord, center, idx, B, M, K, Kstride, Y, y_cstride, y_nstride, w1, blob,
                           inv_scale, shift2, out, nullptr, stream);
}

// the opt-in fp16 mode: one product hi(x)*hi(w) per MAC in layer 2, same blob and arguments
extern "C" int sonet_knn_mlp_tc_forward_f16(const float* coord, const float* center, const int64_t* idx,
                                            int B, int M, int K, int Kstride, const float* Y,
                                            long long y_cstride, long long y_nstride, const float* w1,
                                            const void* blob, float inv_scale, const float* shift2,
                                            float* out, sonet_stream_t stream) {
  return launch_knn_mlp_tc(coord, center, idx, B, M, K, Kstride, Y, y_cstride, y_nstride, w1, blob,
                           inv_scale, shift2, out, nullptr, stream, true);
}

// explicit activation of both layers (SONET_ACT_RELU or SONET_ACT_ELU) and precision (f16 = 1: layer
// 2 as the one-product mode)
extern "C" int sonet_knn_mlp_tc_forward_act(const float* coord, const float* center, const int64_t* idx,
                                            int B, int M, int K, int Kstride, const float* Y,
                                            long long y_cstride, long long y_nstride, const float* w1,
                                            const void* blob, float inv_scale, const float* shift2,
                                            int act, int f16, float* out, sonet_stream_t stream) {
  return launch_knn_mlp_tc(coord, center, idx, B, M, K, Kstride, Y, y_cstride, y_nstride, w1, blob,
                           inv_scale, shift2, out, nullptr, stream, f16 != 0, act);
}

extern "C" int sonet_debug_knn_mlp_tc_timeline(const float* coord, const float* center,
                                               const int64_t* idx, int B, int M, int K, int Kstride,
                                               const float* Y, long long y_cstride,
                                               long long y_nstride, const float* w1,
                                               const void* blob, float inv_scale,
                                               const float* shift2, float* out,
                                               long long* timeline128, sonet_stream_t stream) {
  return launch_knn_mlp_tc(coord, center, idx, B, M, K, Kstride, Y, y_cstride, y_nstride, w1, blob,
                           inv_scale, shift2, out, timeline128, stream);
}
