// pointmlp_tc.cu — the first PointResNet (6|3 -> 64 -> 128 -> 256 -> [64+256] -> 384) of the SO-Net
// encoder as ONE persistent Hopper warpgroup-MMA (wgmma) kernel for sm_90a.
//
// Replaces Encoder.first_pointnet = PointResNet.forward (models/layers.py:419-432, wired at
// models/networks.py:82-83,176): four EquivariantLayers (Conv1d k=1 + eval BatchNorm + ReLU,
// layers.py:282-296) and the skip-concat torch.cat((layer0_out, x_tmp)) — 88 % of the forward's
// FLOPs. The reference round-trips every activation through HBM (~7.4 GB at B=64,N=5000); here a
// 128-point tile walks through all four layers inside one SM:
//
//   * points are the MMA M dimension, channels are N/K. Two consumer warpgroups own 64 points of
//     the tile each (wgmma M = 64) and run independently except for the shared weight stream;
//   * layer 0 (K=3|6, degenerate for tensor cores) runs on CUDA cores, one thread per point and
//     32 channels, and writes act0 as an fp16 hi/lo K-major no-swizzle image into the warpgroup's
//     16 KB of shared memory: layer 1 and layer 3's skip slab read it as a shared-memory A operand;
//   * layers 1-3 are wgmma f16 with fp32 accumulators in registers. A wgmma accumulator fragment
//     (m64nN) has the layout of the register A fragment of m64k16, so the epilogues of layers 1
//     and 2 (folded-BN shift, ReLU or ELU, fp16 hi/lo split) leave act1 / act2 in registers as the A
//     operand of the next layer (64 / 128 registers per thread). No shared-memory image, fence or
//     barrier separates the layers, the tensor cores read only weights from shared memory in
//     layers 2-3, and activations never touch HBM;
//   * fp32 parity (1e-4) on 16-bit tensor cores comes from the 3-product split
//     x*w ~= hi(x)*hi(w) + lo(x)*hi(w) + hi(x)*lo(w) with FP16 halves (hi+lo carry 22 mantissa
//     bits; the same split in bf16 carries 16 and measured 1.1e-4, outside the bar). Weights are
//     pre-scaled per layer by a power of two (undone exactly in the epilogue FMA) so their lo
//     halves stay normal fp16 numbers; activations saturate at the fp16 range (65504) in the conversion;
//   * weights (B operand, K-major no-swizzle core-matrix images packed once by the host) stream
//     L2 -> shared memory through a 5-slot ring (cp.async.bulk + mbarrier), 20 stages per tile:
//     layer 1 (N=128), four layer-2 K slabs (N=256), 3 chunks x 5 K slabs of layer 3 (N=128).
//     The blob is these 20 stages of 32 KB in that order, so each stage is one bulk copy.
//     N=128 chunks instead of 96 cut the drains and pool epilogues per tile from 4 to 3 and keep
//     the tensor pipe busier while a single warpgroup issues (measured on an H100 80GB HBM3 from
//     registers: 115 cycles per m64n128k16 against the ideal 64, 99 per m64n96k16 against 48).
//     Every consumer warp releases a slot as soon as the wgmmas that read it have retired;
//   * shared memory: 2 x 16 KB act0 images + 5 x 32 KB weight slots + W0 and the four shift
//     vectors = 197 KB (a sixth slot would not leave room for the shifts);
//   * warp roles: warpgroups 0-1 the consumers, warpgroup 2 the TMA producer (one thread). The
//     producer gives registers to the consumers (setmaxnreg 24 / 240), where act2, the layer-3
//     accumulators and the pool epilogue are live together;
//   * phasing: the consumers share the ring but no barrier, so either may run ahead of the other
//     by as many stages as the ring holds. An ordered hand-over of the tensor pipe (ping-pong: the
//     warpgroups take turns issuing each layer's / layer-3 chunk's wgmmas, so one's epilogue runs
//     under the other's MMAs) was measured against this free drift at cfg-2 on an H100 80GB HBM3.
//     With the earlier column-at-a-time pool epilogue, at 700 W, both took 1.81-1.83 ms. With the
//     one below, at 400 W, ping-pong took ~3 % fewer SM cycles but ran at a lower clock, for < 1 %
//     more clouds/s. That does not pay for the turn protocol, so free drift stays;
//   * the pool epilogue reduces the 8 lanes that share a thread's columns by reduce-scatter (28
//     shuffles for 32 columns, where a butterfly per column takes 96), and every lane then issues
//     the atomics of its 4 finished columns. At cfg-2 on an H100 80GB HBM3 (400 W) a chunk's
//     epilogue takes ~1.9 k cycles, as the 24-column butterfly of the N=96 chunks did; the
//     butterfly over 32 columns took ~3.2 k.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "tc_common.cuh"

namespace sonet {

namespace pm {
constexpr int C0 = 64, C1 = 128, C2 = 256, C3 = 384, K3 = C0 + C2;  // layer widths
constexpr int TILE = 128;                                            // points per tile
constexpr int SLOT_BYTES = 32768, NSLOT = 5;
constexpr int W1_BYTES = 2 * C1 * C0 * 2;                            // hi + lo images, 32 KB
constexpr int L2_STAGES = 4, L2_KT = 32;                             // [256 rows x 32 k] per stage
constexpr int L3_KSTAGES = 5, L3_KT = 64;                            // K slabs of layer 3
constexpr int L2_STAGE_BYTES = C2 * L2_KT * 2 * 2;                   // 32768
// layer 3: 3 chunks of 128 rows x 5 K slabs, each stage [128 rows x 64 k] hi | lo
constexpr int L3_CHUNKS = 3, L3_N = 128;
constexpr int L3_HALF = L3_N * L3_KT * 2;                            // 16384
constexpr int STAGES_PER_TILE = 1 + L2_STAGES + L3_CHUNKS * L3_KSTAGES;  // 20
constexpr int BLOB_BYTES = STAGES_PER_TILE * SLOT_BYTES;             // 655360
constexpr int NFP = C0 * 6 + C0 + C1 + C2 + C3 + 4;   // W0 | shift0..3 | 1/wscale1..3 (floats)
// warpgroups 0-1 consume (64 points each), warpgroup 2 produces; registers per thread after the
// hand-over: 2 * 128 * 240 + 128 * 24 = 64512, the launch's 168 x 384
constexpr int NUM_THREADS = 384;
constexpr int CONSUMER_REGS = 240, PRODUCER_REGS = 24;
// per-warpgroup act0 image [64 x 64] hi | lo (the A operand of layer 1 and of layer 3's skip slab)
constexpr int ACT0_HALF = 64 * C0 * 2;                 // 8 KB
constexpr int OFF_RING = 2 * 2 * ACT0_HALF;            // 32 KB
// W0 | shift0..3 (floats): the epilogues read their shifts with immediate shared-memory offsets;
// global loads needed a 64-bit address register each, which spilled next to act2
constexpr int NFP_SMEM = C0 * 6 + C0 + C1 + C2 + C3;
constexpr int OFF_FP = OFF_RING + NSLOT * SLOT_BYTES;
constexpr int OFF_BAR = OFF_FP + NFP_SMEM * 4;
constexpr int NBAR = 2 * NSLOT;
constexpr int OFF_TLW = OFF_BAR + NBAR * 8;            // [2] blocked cycles (debug timeline)
constexpr int SMEM_BYTES = OFF_TLW + 2 * 8;            // 201568 (the opt-in limit is 232448)
// debug timeline of CTA 0, per consumer warpgroup w: [64 w + TL_PHASES t + phase] for its tiles
// t < TL_TILES, [64 w + TL_WAIT] the cycles warp 4w spent blocked on `full` over all its tiles
constexpr int TL_PHASES = 4 + 2 * L3_CHUNKS, TL_TILES = 60 / TL_PHASES, TL_WAIT = 60;

// every stage fills exactly one slot
static_assert(W1_BYTES == SLOT_BYTES && L2_STAGE_BYTES == SLOT_BYTES && 2 * L3_HALF == SLOT_BYTES,
              "one weight stage per slot");
}  // namespace pm

// POOL variant (the classifier / auto-encoder path): the input rows are the stacked copies SORTED
// BY NODE (csrc/som_sort.cu) and the layer-3 epilogue, instead of storing the 384 channels of
// every copy (1.47 GB at B=64,N=5000) for a separate index_max launch to re-read, reduces them
// per node right away: for every run of rows in a warp that share a node (rows are node-sorted,
// so usually one) a shuffle reduction over the RAW accumulators leaves each column's maximum in
// lanes 0-3, which apply scale/shift, convert to an order-preserving integer key and issue
// `red.global.max` into keys[b,c,node]. y = fmaf(raw, inv3 > 0, shift) is monotone, so
// max_rows(y) == fmaf(max_rows(raw), ...) bit for bit. models/index_max_ext semantics (max must be
// > -1000, else the feature of copy 0) are restored when the keys are read
// (knn_assemble_pool_kernel / pool_finalize_kernel). first_pn_out is never written.
// The result does not depend on the order of the rows: the run loop takes the node ids of a warp's
// 16 rows in any arrangement (sorting only makes one pass per warp the common case, and the order
// inside a node is whatever som_sort left). A NaN row never becomes a node's maximum, as in
// index_max: fmaxf drops it next to any other row, and a run of NaN rows only is keyed as -inf.
// Required: node_sorted[b,j] < M (a negative id skips the row), 0 <= pos0[b] < P.
// RAGGED (sonet_pointresnet_tc_pool_ragged_forward): one batch row of P sorted copies of several
// clouds; node_sorted holds flat ids b*M + m (< B*M), grouped by them, a row is copy 0 of cloud b
// when it is row pos0[b], and its keys and p0 go to cloud b's [384,M] and [384] slices.
struct PoolArgs {
  const int32_t* node_sorted;  // [B,P] node id of each sorted row
  const int32_t* pos0;         // [B] sorted row of stacked copy 0
  int32_t* keys;               // [B,384,M] running max keys (POOL_KEY_INIT when untouched)
  float* p0;                   // [B,384] features of stacked copy 0
  int M;
};

// DBG: the debug entry points' build, which also stamps the phase timeline of CTA 0.
// NPROD: fp16 products per MAC, 3 (the hi/lo split) or 1 (hi only, the opt-in fp16 mode: act0
// has no lo image, act1 / act2 no lo fragments, and the producer copies the hi half of each stage).
// ACT: the activation of layers 0-2, SONET_ACT_RELU or SONET_ACT_ELU. Nothing downstream assumes
// it is non-negative: the hi/lo split of an ELU output in [-1, inf) saturates exactly as a ReLU
// output's does, and the pool, its -1000 sentinel and its keys act on the bare layer 3.
template <bool POOL, bool DBG, int NPROD, int ACT, bool RAGGED = false>
__global__ void __launch_bounds__(pm::NUM_THREADS, 1)
    pointresnet_tc_kernel(const float* __restrict__ x_in, int Cin, int B, int P,
                          const unsigned char* __restrict__ blob, const float* __restrict__ fparams,
                          float* __restrict__ out, long long* __restrict__ dbg, PoolArgs pool) {
  using namespace pm;
  extern __shared__ __align__(1024) unsigned char smem[];
  float* fps = reinterpret_cast<float*>(smem + OFF_FP);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + OFF_BAR);   // [NSLOT] TMA -> MMA
  uint64_t* empty = full + NSLOT;                                  // [NSLOT] MMA -> TMA

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  if (dbg != nullptr && blockIdx.x == 0 && threadIdx.x == 0) dbg[64 + 62] = clock64();
  const int tiles_per_cloud = (P + TILE - 1) / TILE;
  const int num_tiles = B * tiles_per_cloud;
  const int my_tiles = (static_cast<int>(blockIdx.x) < num_tiles)
                           ? (num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  for (int i = threadIdx.x; i < NFP_SMEM; i += NUM_THREADS) fps[i] = fparams[i];
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
      for (int t = 0; t < my_tiles; ++t) {
#pragma unroll 1
        for (int s = 0; s < STAGES_PER_TILE; ++s, ++q) {
          const uint32_t slot = q % NSLOT, use = q / NSLOT;
          if (use > 0) tc::mbar_wait_relaxed(&empty[slot], (use - 1) & 1, 100 + s);
          unsigned char* dst = smem + OFF_RING + slot * SLOT_BYTES;
          // every stage is [hi | lo], 16 KB each
          constexpr uint32_t bytes = NPROD == 3 ? SLOT_BYTES : SLOT_BYTES / 2;
          mbar_arrive_expect_tx(&full[slot], bytes);
          bulk_g2s(dst, blob + static_cast<uint32_t>(s) * SLOT_BYTES, bytes, &full[slot]);
        }
      }
    }
  } else {
    // =========================== consumer warpgroups ===========================
    tc::regs_inc<CONSUMER_REGS>();
    constexpr unsigned FULL = 0xffffffffu;
    const int wg = warp >> 2;
    const int tw = threadIdx.x & 127;
    unsigned char* act0 = smem + wg * 2 * ACT0_HALF;
    const uint32_t act0_a = smem_u32(act0);
    const uint32_t ring_a = smem_u32(smem + OFF_RING);
    const float* sh1 = fps + C0 * 6 + C0;
    const float* sh2 = sh1 + C1;
    const float* sh3 = sh2 + C2;
    const float* invs = fparams + NFP_SMEM;
    const float inv1 = __ldg(invs), inv2 = __ldg(invs + 1), inv3 = __ldg(invs + 2);
    // accumulator fragment: rows r0 = 16*(warp%4) + lane/4 and r0 + 8 of the warpgroup's 64,
    // columns 8j + 2*(lane%4) + {0,1} (registers 4j+{0,1} for r0, 4j+{2,3} for r0 + 8)
    const int r0 = 16 * (warp & 3) + (lane >> 2);
    const int cq = 2 * (lane & 3);
    uint32_t q = 0;   // weight stages consumed
    // clock64 stamps (debug entry points only): phase 0 tile start, 1 act0 written, 2 layer 1
    // retired, 3 layer-2 epilogue done, 4 + 2c layer-3 chunk c's last wgmma retired, 5 + 2c its
    // epilogue done
    // (pool variant only: next to the plain variant's stores the pointer would spill)
    long long* stamp = (POOL && DBG && blockIdx.x == 0 && tw == 0) ? dbg + 64 * wg : nullptr;
    int t = 0;
    // blocked cycles add up in shared memory: a register next to act2 spills, a global
    // read-modify-write puts an L2 round trip behind every stage
    long long* full_wait = reinterpret_cast<long long*>(smem + OFF_TLW) + wg;
    if (stamp != nullptr) *full_wait = 0;
    auto mark = [&](int phase) {
      if (stamp != nullptr && t < TL_TILES) stamp[TL_PHASES * t + phase] = clock64();
    };

    auto stage_wait = [&]() -> uint32_t {
      const uint32_t slot = q % NSLOT;
      const long long w0 = stamp != nullptr ? clock64() : 0;
      tc::mbar_wait_bounded(&full[slot], (q / NSLOT) & 1, 1);
      if (stamp != nullptr) *full_wait += clock64() - w0;
      return ring_a + slot * SLOT_BYTES;
    };
    auto stage_release = [&](uint32_t qq) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[qq % NSLOT]);
    };
    // Epilogue into the next layer's register A operand: the accumulator fragment of columns
    // [16kk, 16kk+16) is the m64k16 A fragment of K block kk, word i = registers 8kk+2i, 8kk+2i+1
    // (row r0 + 8*(i&1), columns 16kk + 8*(i>>1) + cq + {0,1}), split into fp16 hi/lo words.
    auto to_frags = [&](const float* acc, int kblocks, float inv, const float* sh, uint32_t (*hi)[4],
                        uint32_t (*lo)[4]) {
      const float* shq = sh + cq;
#pragma unroll
      for (int kk = 0; kk < kblocks; ++kk)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int k = 16 * kk + 8 * (i >> 1);
          tc::split_words<NPROD>(act_fn<ACT>(fmaf(acc[8 * kk + 2 * i], inv, shq[k])),
                                 act_fn<ACT>(fmaf(acc[8 * kk + 2 * i + 1], inv, shq[k + 1])),
                                 hi[kk][i], lo[kk][i]);
        }
    };

#pragma unroll 1
    for (; t < my_tiles; ++t) {
      const int tile = blockIdx.x + t * gridDim.x;
      const int b = tile / tiles_per_cloud;
      const int jbase = (tile - b * tiles_per_cloud) * TILE + wg * 64;   // first point of this warpgroup
      mark(0);

      // ---- layer 0 on CUDA cores: point m, channels [32 half, 32 half + 32) ----
      {
        const int m = tw & 63, half = tw >> 6;
        const int j = jbase + m;
        float xv[6];
#pragma unroll
        for (int c = 0; c < 6; ++c)
          xv[c] = (j < P && c < Cin) ? __ldg(x_in + (static_cast<size_t>(b) * Cin + c) * P + j) : 0.f;
        unsigned char* a_hi = act0 + (m >> 3) * 1024 + (m & 7) * 16;
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            float y[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int ch = half * 32 + o * 8 + 2 * jj + e;
              float a = fps[C0 * 6 + ch];
#pragma unroll
              for (int c = 0; c < 6; ++c) a = fmaf(fps[ch * 6 + c], xv[c], a);
              y[e] = act_fn<ACT>(a);
            }
            tc::split_words<NPROD>(y[0], y[1], hi[jj], lo[jj]);
          }
          const int oct = half * 4 + o;
          *reinterpret_cast<uint4*>(a_hi + oct * 128) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
          if (NPROD == 3)
            *reinterpret_cast<uint4*>(a_hi + ACT0_HALF + oct * 128) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
        // act0 writes of this warpgroup -> its wgmmas
        tc::fence_proxy_async();
        tc::named_sync(1 + wg, 128);
        mark(1);
      }

      // this thread's rows in the layer-3 epilogue (loaded here, where few registers are live)
      int nd[2] = {-1, -1};
      bool is_p0[2] = {false, false};
      const bool valid0 = jbase + r0 < P, valid1 = jbase + r0 + 8 < P;
      if (POOL) {
        const int p0row = __ldg(pool.pos0 + b);
        if (valid0) nd[0] = __ldg(pool.node_sorted + static_cast<size_t>(b) * P + jbase + r0);
        if (valid1) nd[1] = __ldg(pool.node_sorted + static_cast<size_t>(b) * P + jbase + r0 + 8);
        if (RAGGED) {
          is_p0[0] = valid0 && nd[0] >= 0 && jbase + r0 == __ldg(pool.pos0 + nd[0] / pool.M);
          is_p0[1] = valid1 && nd[1] >= 0 && jbase + r0 + 8 == __ldg(pool.pos0 + nd[1] / pool.M);
        } else {
          is_p0[0] = valid0 && jbase + r0 == p0row;
          is_p0[1] = valid1 && jbase + r0 + 8 == p0row;
        }
      }

      // ---- layer 1: D1[64 x 128] = act0[64 x 64] * W1^T, A from shared memory ----
      uint32_t a1_hi[C1 / 16][4], a1_lo[C1 / 16][4];
      {
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        const uint32_t sb = stage_wait();
        tc::wg_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint64_t ah = tc::smem_desc(act0_a + ks * 256, 128, 1024),
                         al = tc::smem_desc(act0_a + ACT0_HALF + ks * 256, 128, 1024),
                         bh = tc::smem_desc(sb + ks * 256, 128, 1024),
                         bl = tc::smem_desc(sb + W1_BYTES / 2 + ks * 256, 128, 1024);
          tc::wgmma_f16_n128(acc, ah, bh, 1);
          if (NPROD == 3) {
            tc::wgmma_f16_n128(acc, al, bh, 1);
            tc::wgmma_f16_n128(acc, ah, bl, 1);
          }
        }
        tc::wg_commit();
        tc::wg_wait<0>();
        mark(2);
        stage_release(q++);
        to_frags(acc, C1 / 16, inv1, sh1, a1_hi, a1_lo);
      }

      // ---- layer 2: D2[64 x 256] = act1[64 x 128] * W2^T, four K slabs of 32, A from registers ----
      uint32_t a2_hi[C2 / 16][4], a2_lo[C2 / 16][4];
      {
        float acc[128];
#pragma unroll
        for (int i = 0; i < 128; ++i) acc[i] = 0.f;
#pragma unroll
        for (int kc = 0; kc < L2_STAGES; ++kc) {
          const uint32_t sb = stage_wait();
          tc::wg_fence();
#pragma unroll
          for (int ks = 0; ks < 2; ++ks) {
            const int kk = kc * 2 + ks;
            const uint64_t bh = tc::smem_desc(sb + ks * 256, 128, 512),
                           bl = tc::smem_desc(sb + L2_STAGE_BYTES / 2 + ks * 256, 128, 512);
            tc::wgmma_f16_rs_n256(acc, a1_hi[kk], bh, 1);
            if (NPROD == 3) {
              tc::wgmma_f16_rs_n256(acc, a1_lo[kk], bh, 1);
              tc::wgmma_f16_rs_n256(acc, a1_hi[kk], bl, 1);
            }
          }
          tc::wg_commit();
          tc::wg_wait<1>();
          if (kc > 0) stage_release(q - 1);
          ++q;
        }
        tc::wg_wait<0>();
        stage_release(q - 1);
        to_frags(acc, C2 / 16, inv2, sh2, a2_hi, a2_lo);
        mark(3);
      }

      // ---- layer 3: D3[64 x 384] = cat(act0, act2)[64 x 320] * W3^T, 3 chunks of N=128; bare ----
#pragma unroll 1
      for (int nc = 0; nc < L3_CHUNKS; ++nc) {
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        // K slab 0 = act0 (shared memory), slabs 1-4 = act2 K blocks 4(kc-1) .. 4(kc-1)+3 (registers)
#pragma unroll
        for (int kc = 0; kc < L3_KSTAGES; ++kc) {
          const uint32_t sb = stage_wait();
          tc::wg_fence();
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            const uint64_t bh = tc::smem_desc(sb + ks * 256, 128, 1024),
                           bl = tc::smem_desc(sb + L3_HALF + ks * 256, 128, 1024);
            if (kc == 0) {
              const uint64_t ah = tc::smem_desc(act0_a + ks * 256, 128, 1024),
                             al = tc::smem_desc(act0_a + ACT0_HALF + ks * 256, 128, 1024);
              tc::wgmma_f16_n128(acc, ah, bh, 1);
              if (NPROD == 3) {
                tc::wgmma_f16_n128(acc, al, bh, 1);
                tc::wgmma_f16_n128(acc, ah, bl, 1);
              }
            } else {
              const int kk = 4 * (kc - 1) + ks;
              tc::wgmma_f16_rs_n128(acc, a2_hi[kk], bh, 1);
              if (NPROD == 3) {
                tc::wgmma_f16_rs_n128(acc, a2_lo[kk], bh, 1);
                tc::wgmma_f16_rs_n128(acc, a2_hi[kk], bl, 1);
              }
            }
          }
          tc::wg_commit();
          tc::wg_wait<1>();
          if (kc > 0) stage_release(q - 1);
          ++q;
        }
        tc::wg_wait<0>();
        mark(4 + 2 * nc);
        stage_release(q - 1);

        const int cbase = L3_N * nc + cq;
        if (!POOL) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int j = jbase + r0 + 8 * rr;
            if (j >= P) continue;
            float* o = out + (static_cast<size_t>(b) * C3 + cbase) * P + j;
#pragma unroll
            for (int jn = 0; jn < 16; ++jn, o += 8 * static_cast<size_t>(P))
#pragma unroll
              for (int e = 0; e < 2; ++e)
                o[e * static_cast<size_t>(P)] =
                    fmaf(acc[4 * jn + 2 * rr + e], inv3, sh3[cbase + 8 * jn + e]);
          }
        } else {
          // per-node max over the warp's 16 rows, one pass per run of equal node ids
          unsigned rem0 = __ballot_sync(FULL, nd[0] >= 0), rem1 = __ballot_sync(FULL, nd[1] >= 0);
#pragma unroll 1
          while ((rem0 | rem1) != 0) {
            const int node = rem0 ? __shfl_sync(FULL, nd[0], __ffs(rem0) - 1)
                                  : __shfl_sync(FULL, nd[1], __ffs(rem1) - 1);
            const bool in0 = nd[0] == node, in1 = nd[1] == node;
            rem0 &= ~__ballot_sync(FULL, in0);
            rem1 &= ~__ballot_sync(FULL, in1);
            // reduce-scatter over the 8 lanes that hold the same 32 columns (lane xor 16, 8, 4):
            // each step keeps half of the columns and takes the partner's maxima of that half, so
            // the 32 columns cost 16 + 8 + 4 shuffles (a full butterfly per column costs 96) and
            // every lane ends with 4 finished columns, slots base .. base + 3 of the thread's 32
            // (slot s = column 8 (s / 2) + s % 2 + cq of the chunk)
            const bool b2 = lane & 16, b1 = lane & 8, b0 = lane & 4;
            float r1[16];
#pragma unroll
            for (int c = 0; c < 16; ++c) {
              const int s = c, u = c + 16;
              const float vs = fmaxf(in0 ? acc[4 * (s >> 1) + (s & 1)] : -INFINITY,
                                     in1 ? acc[4 * (s >> 1) + 2 + (s & 1)] : -INFINITY);
              const float vu = fmaxf(in0 ? acc[4 * (u >> 1) + (u & 1)] : -INFINITY,
                                     in1 ? acc[4 * (u >> 1) + 2 + (u & 1)] : -INFINITY);
              r1[c] = fmaxf(b2 ? vu : vs, __shfl_xor_sync(FULL, b2 ? vs : vu, 16));
            }
            float r2[8];
#pragma unroll
            for (int c = 0; c < 8; ++c)
              r2[c] = fmaxf(b1 ? r1[c + 8] : r1[c], __shfl_xor_sync(FULL, b1 ? r1[c] : r1[c + 8], 8));
            float r3[4];
#pragma unroll
            for (int c = 0; c < 4; ++c)
              r3[c] = fmaxf(b0 ? r2[c + 4] : r2[c], __shfl_xor_sync(FULL, b0 ? r2[c] : r2[c + 4], 4));
            const int col = cbase + 8 * ((16 * b2 + 8 * b1 + 4 * b0) >> 1);   // slot base's column
            const int kcloud = RAGGED ? node / pool.M : b, knode = RAGGED ? node - kcloud * pool.M : node;
            int32_t* kb = pool.keys + (static_cast<size_t>(kcloud) * C3 + col) * pool.M + knode;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int dc = 8 * (i >> 1) + (i & 1);
              // fmaxf(NaN, -inf) = -inf: a run whose 16 rows are all NaN in this column must not
              // leave a NaN key, which would order above +inf and displace the node's finite maximum
              const int bits = __float_as_int(fmaxf(fmaf(r3[i], inv3, sh3[col + dc]), -INFINITY));
              const int key = bits ^ ((bits >> 31) & 0x7fffffff);   // order-preserving float -> int
              atomicMax(kb + dc * static_cast<size_t>(pool.M), key);
            }
          }
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            if (!is_p0[rr]) continue;   // rare: one row per cloud
            const int pcloud = RAGGED ? nd[rr] / pool.M : b;
#pragma unroll
            for (int jn = 0; jn < 16; ++jn)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                pool.p0[static_cast<size_t>(pcloud) * C3 + cbase + 8 * jn + e] =
                    fmaf(acc[4 * jn + 2 * rr + e], inv3, sh3[cbase + 8 * jn + e]);
          }
        }
        mark(5 + 2 * nc);
      }
      // the next tile's layer 0 overwrites act0, which this tile's layer-3 wgmmas read: all are
      // complete (wait_group 0 above); the other warps of the warpgroup must be past them too
      tc::named_sync(1 + wg, 128);
    }
    if (stamp != nullptr) stamp[TL_WAIT] = *full_wait;
  }
  __syncthreads();
  if (dbg != nullptr && blockIdx.x == 0 && threadIdx.x == 0) dbg[64 + 63] = clock64();
}

}  // namespace sonet

extern "C" int sonet_pointresnet_tc_blob_bytes(void) { return sonet::pm::BLOB_BYTES; }
extern "C" int sonet_pointresnet_tc_fparam_count(void) { return sonet::pm::NFP; }

extern "C" int sonet_pointresnet_tc_pack(const float* W0, int Cin, const float* W1, const float* W2,
                                         const float* W3, const float* shift0, const float* shift1,
                                         const float* shift2, const float* shift3, void* blob_host,
                                         float* fparams_host) {
  using namespace sonet;
  using namespace sonet::pm;
  SONET_REQUIRE(Cin >= 1 && Cin <= 6, "pointresnet_tc_pack: Cin=%d out of range [1,6]", Cin);
  SONET_REQUIRE(W0 && W1 && W2 && W3 && shift0 && shift1 && shift2 && shift3 && blob_host &&
                    fparams_host,
                "pointresnet_tc_pack: null pointer");
  unsigned char* blob = static_cast<unsigned char*>(blob_host);
  std::memset(blob, 0, BLOB_BYTES);
  const float s1 = pow2_scale(W1, static_cast<size_t>(C1) * C0),
              s2 = pow2_scale(W2, static_cast<size_t>(C2) * C1),
              s3 = pow2_scale(W3, static_cast<size_t>(C3) * K3);
  // layer 1, resident: [128 rows x 64 k]
  pack_tile(W1, s1, C0, 0, C1, 0, C0, blob, blob + W1_BYTES / 2);
  size_t off = W1_BYTES;
  // layer 2: four K slabs [256 rows x 32 k]
  for (int kc = 0; kc < L2_STAGES; ++kc) {
    pack_tile(W2, s2, C1, 0, C2, L2_KT * kc, L2_KT, blob + off, blob + off + L2_STAGE_BYTES / 2);
    off += L2_STAGE_BYTES;
  }
  // layer 3: three 128-row chunks x five K slabs [128 rows x 64 k]
  for (int nc = 0; nc < L3_CHUNKS; ++nc)
    for (int kc = 0; kc < L3_KSTAGES; ++kc) {
      pack_tile(W3, s3, K3, L3_N * nc, L3_N, L3_KT * kc, L3_KT, blob + off, blob + off + L3_HALF);
      off += 2 * L3_HALF;
    }
  if (off != static_cast<size_t>(BLOB_BYTES)) SONET_FAIL(SONET_ERR_BAD_ARG, "pack: size mismatch");
  float* f = fparams_host;
  for (int c = 0; c < C0; ++c)
    for (int i = 0; i < 6; ++i) f[c * 6 + i] = (i < Cin) ? W0[c * Cin + i] : 0.f;
  std::memcpy(f + C0 * 6, shift0, C0 * 4);
  std::memcpy(f + C0 * 6 + C0, shift1, C1 * 4);
  std::memcpy(f + C0 * 6 + C0 + C1, shift2, C2 * 4);
  std::memcpy(f + C0 * 6 + C0 + C1 + C2, shift3, C3 * 4);
  float* inv = f + C0 * 6 + C0 + C1 + C2 + C3;
  inv[0] = 1.f / s1;
  inv[1] = 1.f / s2;
  inv[2] = 1.f / s3;
  inv[3] = 0.f;
  return SONET_OK;
}

static int launch_pointresnet_tc(const float* x, int Cin, int B, int P, const void* blob,
                                 const float* fparams, float* out, long long* dbg,
                                 const sonet::PoolArgs* pool, sonet_stream_t stream, bool f16 = false,
                                 int act = SONET_ACT_RELU, bool ragged = false) {
  using namespace sonet;
  using namespace sonet::pm;
  SONET_REQUIRE(act == SONET_ACT_RELU || act == SONET_ACT_ELU,
                "pointresnet_tc: activation code %d is not SONET_ACT_RELU (1) or _ELU (2)", act);
  SONET_REQUIRE(B >= 0 && P >= 0, "pointresnet_tc: negative dimension");
  SONET_REQUIRE(Cin >= 1 && Cin <= 6, "pointresnet_tc: Cin=%d out of range [1,6]", Cin);
  if (B == 0 || P == 0) return SONET_OK;
  SONET_REQUIRE(x && blob && fparams && (out || pool), "pointresnet_tc: null pointer");
  SONET_REQUIRE(!pool || (pool->node_sorted && pool->pos0 && pool->keys && pool->p0 && pool->M >= 1),
                "pointresnet_tc: incomplete pool arguments");
  SONET_REQUIRE(aligned16(blob), "pointresnet_tc: weight blob must be 16-byte aligned");
  const long long tiles = static_cast<long long>(B) * ((P + TILE - 1) / TILE);
  SONET_REQUIRE(tiles < (1LL << 31), "pointresnet_tc: too many tiles");
  SONET_REQUIRE(SMEM_BYTES <= max_smem_optin(), "pointresnet_tc: needs %d B of shared memory",
                SMEM_BYTES);
  const int grid = static_cast<int>(std::min<long long>(tiles, sm_count()));
  SONET_REQUIRE(!(f16 && dbg), "pointresnet_tc: the debug timeline has no fp16 build");
  SONET_REQUIRE(!(act != SONET_ACT_RELU && dbg), "pointresnet_tc: the debug timeline has no ELU build");
  constexpr int R = SONET_ACT_RELU, E = SONET_ACT_ELU;
  auto kern =
      ragged ? (act == E ? (f16 ? pointresnet_tc_kernel<true, false, 1, E, true> : pointresnet_tc_kernel<true, false, 3, E, true>)
                         : (f16 ? pointresnet_tc_kernel<true, false, 1, R, true> : pointresnet_tc_kernel<true, false, 3, R, true>))
      : act == E ? (f16 ? (pool ? pointresnet_tc_kernel<true, false, 1, E> : pointresnet_tc_kernel<false, false, 1, E>)
                      : (pool ? pointresnet_tc_kernel<true, false, 3, E> : pointresnet_tc_kernel<false, false, 3, E>))
      : f16 ? (pool ? pointresnet_tc_kernel<true, false, 1, R> : pointresnet_tc_kernel<false, false, 1, R>)
      : pool ? (dbg ? pointresnet_tc_kernel<true, true, 3, R> : pointresnet_tc_kernel<true, false, 3, R>)
             : (dbg ? pointresnet_tc_kernel<false, true, 3, R> : pointresnet_tc_kernel<false, false, 3, R>);
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  PoolArgs pa = pool ? *pool : PoolArgs{nullptr, nullptr, nullptr, nullptr, 0};
  kern<<<grid, NUM_THREADS, SMEM_BYTES, as_stream(stream)>>>(
      x, Cin, B, P, static_cast<const unsigned char*>(blob), fparams, out, dbg, pa);
  return check_launch("pointresnet_tc");
}

extern "C" int sonet_pointresnet_tc_forward(const float* x, int Cin, int B, int P, const void* blob,
                                            const float* fparams, float* out,
                                            sonet_stream_t stream) {
  return launch_pointresnet_tc(x, Cin, B, P, blob, fparams, out, nullptr, nullptr, stream);
}

extern "C" int sonet_pointresnet_tc_pool_forward(const float* x_sorted, int Cin, int B, int P,
                                                 const void* blob, const float* fparams,
                                                 const int32_t* node_sorted, const int32_t* pos0,
                                                 int M, int32_t* pool_keys, float* p0,
                                                 sonet_stream_t stream) {
  sonet::PoolArgs pa{node_sorted, pos0, pool_keys, p0, M};
  return launch_pointresnet_tc(x_sorted, Cin, B, P, blob, fparams, nullptr, nullptr, &pa, stream);
}

// the opt-in fp16 mode of the two entries above: one product hi(x)*hi(w) per MAC, same blob
extern "C" int sonet_pointresnet_tc_forward_f16(const float* x, int Cin, int B, int P, const void* blob,
                                                const float* fparams, float* out,
                                                sonet_stream_t stream) {
  return launch_pointresnet_tc(x, Cin, B, P, blob, fparams, out, nullptr, nullptr, stream, true);
}

extern "C" int sonet_pointresnet_tc_pool_forward_f16(const float* x_sorted, int Cin, int B, int P,
                                                     const void* blob, const float* fparams,
                                                     const int32_t* node_sorted, const int32_t* pos0,
                                                     int M, int32_t* pool_keys, float* p0,
                                                     sonet_stream_t stream) {
  sonet::PoolArgs pa{node_sorted, pos0, pool_keys, p0, M};
  return launch_pointresnet_tc(x_sorted, Cin, B, P, blob, fparams, nullptr, nullptr, &pa, stream, true);
}

// explicit activation (SONET_ACT_RELU or SONET_ACT_ELU) and precision (f16 = 1: the one-product mode)
extern "C" int sonet_pointresnet_tc_forward_act(const float* x, int Cin, int B, int P, const void* blob,
                                                const float* fparams, int act, int f16, float* out,
                                                sonet_stream_t stream) {
  return launch_pointresnet_tc(x, Cin, B, P, blob, fparams, out, nullptr, nullptr, stream, f16 != 0, act);
}

extern "C" int sonet_pointresnet_tc_pool_forward_act(const float* x_sorted, int Cin, int B, int P,
                                                     const void* blob, const float* fparams,
                                                     const int32_t* node_sorted, const int32_t* pos0,
                                                     int M, int act, int f16, int32_t* pool_keys,
                                                     float* p0, sonet_stream_t stream) {
  sonet::PoolArgs pa{node_sorted, pos0, pool_keys, p0, M};
  return launch_pointresnet_tc(x_sorted, Cin, B, P, blob, fparams, nullptr, nullptr, &pa, stream, f16 != 0,
                               act);
}

// the pool over the sorted copies of a ragged batch laid out as one row (PoolArgs, RAGGED)
extern "C" int sonet_pointresnet_tc_pool_ragged_forward(const float* x_sorted, int Cin, int P,
                                                        const void* blob, const float* fparams,
                                                        const int32_t* node_sorted, const int32_t* pos0,
                                                        int B, int M, int act, int f16,
                                                        int32_t* pool_keys, float* p0,
                                                        sonet_stream_t stream) {
  SONET_REQUIRE(B >= 1 && M >= 1 && M <= 256 && static_cast<long long>(B) * M < (1LL << 31),
                "pointresnet_tc_pool_ragged: bad dimension (B=%d, M=%d)", B, M);
  sonet::PoolArgs pa{node_sorted, pos0, pool_keys, p0, M};
  return launch_pointresnet_tc(x_sorted, Cin, 1, P, blob, fparams, nullptr, nullptr, &pa, stream, f16 != 0,
                               act, true);
}

extern "C" int sonet_debug_pointresnet_tc_pool_timeline(const float* x_sorted, int Cin, int B, int P,
                                                        const void* blob, const float* fparams,
                                                        const int32_t* node_sorted,
                                                        const int32_t* pos0, int M,
                                                        int32_t* pool_keys, float* p0,
                                                        long long* timeline64,
                                                        sonet_stream_t stream) {
  sonet::PoolArgs pa{node_sorted, pos0, pool_keys, p0, M};
  return launch_pointresnet_tc(x_sorted, Cin, B, P, blob, fparams, nullptr, timeline64, &pa, stream);
}

extern "C" int sonet_debug_pointresnet_tc_timeline(const float* x, int Cin, int B, int P,
                                                   const void* blob, const float* fparams,
                                                   float* out, long long* timeline64,
                                                   sonet_stream_t stream) {
  return launch_pointresnet_tc(x, Cin, B, P, blob, fparams, out, timeline64, nullptr, stream);
}
