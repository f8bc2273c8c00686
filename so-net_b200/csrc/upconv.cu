// upconv.cu — the auto-encoder's up-convolution decoder (SURVEY.md §8f-1) for sm_90a.
//
// Replaces UpConv.forward (models/layers.py:214-240: nn.Upsample(scale_factor=2) + Conv2d 3x3 pad 1
// + BatchNorm2d + ReLU) as used by DecoderConv (models/networks.py:394-431).
//
// Nearest x2 up-sampling followed by a 3x3 convolution never needs the up-sampled image: output
// pixel (2i+py, 2j+px) only sees the 2x2 low-resolution neighbourhood rows {i-1+py, i+py} x
// columns {j-1+px, j+px}, and the three kernel rows (columns) collapse onto those two — rows
// {0}|{1,2} for py = 0 and {0,1}|{2} for py = 1. The layer is therefore FOUR GEMMs (one per output
// parity) with K = 4*Cin instead of one with K = 9*Cin over 4x the pixels: 2.25x fewer flops, and
// the zero padding of the up-sampled image coincides with zero padding of the low-resolution one.
// The host folds BN and the tap sums into four [Cout, 4*Cin] matrices once per weight change
// (sonet_b200/layers.py); here:
//   upconv_im2col_kernel    gathers the 2x2 neighbourhoods of all four parities,
//                           xcol[g][b][t*Cin+ci][i*W+j], coalesced along j;
//   sonet_pointwise_tc_grouped_forward (csrc/pointwise_tc.cu) runs the four GEMMs as ONE grouped
//                           wgmma launch (fp16 hi/lo split, fp32 accumulate) whose epilogue —
//                           or, for the small maps that need a K split to fill the SMs, the
//                           split-K reduce kernel — adds the folded shift, applies ReLU and
//                           interleaves the parities into the [B, Cout, 2H, 2W] output.
#include <algorithm>

#include "common.cuh"

namespace sonet {

// IT = uint32_t whenever the element count fits (the four divisions per element bound this kernel
// when they were 64-bit ones)
template <typename IT>
__global__ void __launch_bounds__(256)
    upconv_im2col_kernel(const float* __restrict__ in, int B, int Cin, int H, int W,
                         float* __restrict__ xcol) {
  const int HW = H * W;
  const IT uHW = static_cast<IT>(HW), uK = static_cast<IT>(4 * Cin);
  const IT per_g = static_cast<IT>(B) * uK * uHW;
  const IT total = per_g * 4;
  for (IT e = static_cast<IT>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<IT>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(e / per_g);
    IT r = e - g * per_g;
    const IT q = r / uHW;
    const int p = static_cast<int>(r - q * uHW);
    const int b = static_cast<int>(q / uK);
    const int k = static_cast<int>(q - static_cast<IT>(b) * uK);
    const int t = k / Cin, ci = k - t * Cin;
    const int i = p / W, j = p - i * W;
    const int y = i + (t >> 1) - 1 + (g >> 1), x = j + (t & 1) - 1 + (g & 1);
    float v = 0.f;
    if (y >= 0 && y < H && x >= 0 && x < W)
      v = __ldg(in + (static_cast<size_t>(b) * Cin + ci) * HW + y * W + x);
    xcol[e] = v;
  }
}

// W % 4 == 0: a thread produces 4 consecutive pixels of one xcol row (one 16-byte store; the write
// stream is what bounds this kernel — every input element is re-read 16 times, but from L1/L2).
// blockDim = (TX, TY): TX threads cover the H*W/4 quads of a row, TY rows per block; a row is
// (g, b, k) with k = t*Cin + ci.
__global__ void __launch_bounds__(256)
    upconv_im2col_vec4_kernel(const float* __restrict__ in, int B, int Cin, int H, int W,
                              float* __restrict__ xcol) {
  const int HW = H * W, K = 4 * Cin;
  const int rows = 4 * B * K;
  const int row = blockIdx.x * blockDim.y + threadIdx.y;
  if (row >= rows) return;
  const int k = row % K;
  const int gb = row / K;
  const int b = gb % B, g = gb / B;
  const int t = k / Cin, ci = k - t * Cin;
  const int dy = (t >> 1) - 1 + (g >> 1), dx = (t & 1) - 1 + (g & 1);
  const float* src = in + (static_cast<size_t>(b) * Cin + ci) * HW;
  float4* dst = reinterpret_cast<float4*>(xcol + static_cast<size_t>(row) * HW);
  for (int q = threadIdx.x; q < (HW >> 2); q += blockDim.x) {
    const int p = q << 2;
    const int i = p / W, j = p - i * W;
    const int y = i + dy;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (y >= 0 && y < H) {
      const float* r = src + y * W;
      const int x = j + dx;
      if (x >= 0) v.x = __ldg(r + x);          // x .. x+3 < W+1: only the ends can fall outside
      v.y = __ldg(r + x + 1);
      v.z = __ldg(r + x + 2);
      if (x + 3 < W) v.w = __ldg(r + x + 3);
    }
    __stcs(dst + q, v);
  }
}

// The three horizontally shifted copies [3][B][Cin][H*W] (dx = -1, 0, +1, zero at the row ends)
// that the conv mode of the grouped wgmma kernel reads instead of a 16x im2col: a vertical shift
// is a plain offset of the point coordinate (the kernel reads zeros for its out-of-range part),
// only the horizontal one wraps across image rows and has to be materialised.
__global__ void __launch_bounds__(256)
    upconv_hshift_kernel(const float* __restrict__ in, long long rows, int H, int W,
                         float* __restrict__ out) {
  const int HW = H * W;
  const long long total = rows * HW;                         // rows = B * Cin
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(e % W);
    const float v = __ldg(in + e);
    out[total + e] = v;                                      // block 1: dx = 0
    out[e] = (j > 0) ? __ldg(in + e - 1) : 0.f;              // block 0: reads column j-1
    out[2 * total + e] = (j + 1 < W) ? __ldg(in + e + 1) : 0.f;   // block 2: column j+1
  }
}

// ---- training (sonet_b200/train_ops.py: UpConvTC) -------------------------------------------------
// Tap a (c) of output parity py (px) collects kernel rows (columns) fold_lo..fold_hi: {0} | {1,2}
// for parity 0, {0,1} | {2} for parity 1.
__device__ __forceinline__ int fold_lo(int parity, int a) { return a == 0 ? 0 : 1 + parity; }
__device__ __forceinline__ int fold_hi(int parity, int a) { return a == 0 ? parity : 2; }
// ... and kernel row k belongs to tap fold_tap(parity, k)
__device__ __forceinline__ int fold_tap(int parity, int k) { return k > parity ? 1 : 0; }

// sum of the taps of W [Cout,Cin,3,3] that (g, t) collects, rows then columns ascending
__device__ __forceinline__ float fold_sum(const float* __restrict__ w, int Cin, int g, int t, int co,
                                          int ci) {
  const int py = g >> 1, px = g & 1, a = t >> 1, c = t & 1;
  const float* k = w + (static_cast<size_t>(co) * Cin + ci) * 9;
  float s = 0.f;
  for (int ky = fold_lo(py, a); ky <= fold_hi(py, a); ++ky)
    for (int kx = fold_lo(px, c); kx <= fold_hi(px, c); ++kx) s += k[ky * 3 + kx];
  return s;
}

// Wg [4][Cout][4*Cin]: element (g, co, t*Cin + ci)
__global__ void __launch_bounds__(256)
    upconv_fold_kernel(const float* __restrict__ w, int Cout, int Cin, float* __restrict__ wg) {
  const long long K = 4LL * Cin, total = 4LL * Cout * K;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(e % K);
    const long long gco = e / K;
    const int co = static_cast<int>(gco % Cout), g = static_cast<int>(gco / Cout);
    wg[e] = fold_sum(w, Cin, g, k / Cin, co, k % Cin);
  }
}

// the dgrad matrix [Cin][16*Cout]: element (ci, (g*4 + t)*Cout + co) = Wg[g][co][t*Cin + ci]
__global__ void __launch_bounds__(256)
    upconv_fold_dgrad_kernel(const float* __restrict__ w, int Cout, int Cin, float* __restrict__ wd) {
  const long long K = 16LL * Cout, total = K * Cin;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(e % K), ci = static_cast<int>(e / K);
    const int gt = k / Cout, co = k - gt * Cout;
    wd[e] = fold_sum(w, Cin, gt >> 2, gt & 3, co, ci);
  }
}

// adjoint: dW [Cout,Cin,3,3] from dWT [4][4*Cin][Cout] (per parity, the wgrad GEMM's layout); every
// tap is the sum of exactly one entry per parity, added in ascending parity order
__global__ void __launch_bounds__(256)
    upconv_fold_adjoint_kernel(const float* __restrict__ dwt, int Cout, int Cin, float* __restrict__ dw) {
  const long long total = 9LL * Cout * Cin;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int kk = static_cast<int>(e % 9), ky = kk / 3, kx = kk - ky * 3;
    const long long coci = e / 9;
    const int ci = static_cast<int>(coci % Cin), co = static_cast<int>(coci / Cin);
    float s = 0.f;
    for (int g = 0; g < 4; ++g) {
      const int t = fold_tap(g >> 1, ky) * 2 + fold_tap(g & 1, kx);
      s += dwt[(static_cast<size_t>(g) * 4 * Cin + static_cast<size_t>(t) * Cin + ci) * Cout + co];
    }
    dw[e] = s;
  }
}

// D [B][16*Cout][H*W] from dz [B,Cout,2H,2W]: row (g*4 + t)*Cout + co, point i*W + j holds
// dz[b, co, 2(i-oy)+py, 2(j-ox)+px] with oy = a-1+py, ox = c-1+px (0 outside the map) — the
// operand whose product with the dgrad matrix is dx.
template <typename IT>
__global__ void __launch_bounds__(256)
    upconv_dgrad_im2col_kernel(const float* __restrict__ dz, int B, int Cout, int H, int W,
                               float* __restrict__ d) {
  const IT uHW = static_cast<IT>(H) * W, uK = 16 * static_cast<IT>(Cout);
  const IT total = static_cast<IT>(B) * uK * uHW;
  for (IT e = static_cast<IT>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<IT>(gridDim.x) * blockDim.x) {
    const IT q = e / uHW;
    const int p = static_cast<int>(e - q * uHW);
    const int b = static_cast<int>(q / uK);
    const int k = static_cast<int>(q - static_cast<IT>(b) * uK);
    const int gt = k / Cout, co = k - gt * Cout;
    const int g = gt >> 2, t = gt & 3;
    const int py = g >> 1, px = g & 1;
    const int i = p / W - ((t >> 1) - 1 + py), j = p % W - ((t & 1) - 1 + px);
    float v = 0.f;
    if (i >= 0 && i < H && j >= 0 && j < W)
      v = __ldg(dz + ((static_cast<size_t>(b) * Cout + co) * 2 * H + 2 * i + py) * 2 * W + 2 * j + px);
    d[e] = v;
  }
}

static int grid_for(long long total) {
  return static_cast<int>(std::min<long long>((total + 255) / 256, 16LL * sm_count()));
}

}  // namespace sonet

extern "C" int sonet_upconv_fold_weights_f32(const float* in, int Cout, int Cin, int adjoint, float* out,
                                             float* out_dgrad, sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(Cout >= 1 && Cin >= 1, "upconv_fold_weights: bad dimension Cout=%d Cin=%d", Cout, Cin);
  SONET_REQUIRE(adjoint == 0 || adjoint == 1, "upconv_fold_weights: adjoint must be 0 or 1 (got %d)",
                adjoint);
  SONET_REQUIRE(in != nullptr, "upconv_fold_weights: null input pointer");
  if (adjoint) {
    SONET_REQUIRE(out != nullptr && out_dgrad == nullptr,
                  "upconv_fold_weights: the adjoint writes dW to out only (out_dgrad must be null)");
  } else {
    SONET_REQUIRE(out != nullptr || out_dgrad != nullptr,
                  "upconv_fold_weights: null output pointers (Wg and the dgrad matrix)");
  }
  const long long n = 36LL * Cout * Cin;      // 9 * Cout * Cin for the adjoint
  SONET_REQUIRE(n < (1LL << 40), "upconv_fold_weights: too many weights");
  cudaStream_t st = as_stream(stream);
  if (adjoint) {
    upconv_fold_adjoint_kernel<<<grid_for(n / 4), 256, 0, st>>>(in, Cout, Cin, out);
    return check_launch("upconv_fold_weights(adjoint)");
  }
  if (out != nullptr) upconv_fold_kernel<<<grid_for(4 * n / 9), 256, 0, st>>>(in, Cout, Cin, out);
  if (out_dgrad != nullptr)
    upconv_fold_dgrad_kernel<<<grid_for(4 * n / 9), 256, 0, st>>>(in, Cout, Cin, out_dgrad);
  return check_launch("upconv_fold_weights");
}

extern "C" int sonet_upconv_dgrad_im2col_f32(const float* dz, int B, int Cout, int H, int W, float* d,
                                             sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && Cout >= 1 && H >= 1 && W >= 1, "upconv_dgrad_im2col: bad dimension");
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(dz && d, "upconv_dgrad_im2col: null pointer");
  const long long total = 16LL * B * Cout * H * W;
  if (total < (1LL << 32))
    upconv_dgrad_im2col_kernel<uint32_t><<<grid_for(total), 256, 0, as_stream(stream)>>>(dz, B, Cout, H, W, d);
  else
    upconv_dgrad_im2col_kernel<unsigned long long><<<grid_for(total), 256, 0, as_stream(stream)>>>(
        dz, B, Cout, H, W, d);
  return check_launch("upconv_dgrad_im2col");
}

extern "C" int sonet_upconv_hshift_f32(const float* in, int B, int Cin, int H, int W, float* out,
                                       sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && Cin >= 1 && H >= 1 && W >= 1, "upconv_hshift: bad dimension");
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(in && out, "upconv_hshift: null pointer");
  const long long rows = static_cast<long long>(B) * Cin;
  const long long total = rows * H * W;
  const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, 16LL * sm_count()));
  upconv_hshift_kernel<<<grid, 256, 0, as_stream(stream)>>>(in, rows, H, W, out);
  return check_launch("upconv_hshift");
}

extern "C" int sonet_upconv_im2col_f32(const float* in, int B, int Cin, int H, int W, float* xcol,
                                       sonet_stream_t stream) {
  using namespace sonet;
  SONET_REQUIRE(B >= 0 && Cin >= 1 && H >= 1 && W >= 1, "upconv_im2col: bad dimension");
  if (B == 0) return SONET_OK;
  SONET_REQUIRE(in && xcol, "upconv_im2col: null pointer");
  const long long total = 16LL * B * Cin * H * W;
  const long long rows = 16LL * B * Cin;
  if (W % 4 == 0 && aligned16(xcol) && rows < (1LL << 31)) {
    int tx = std::min(256, H * W / 4), ty = 1;
    tx = std::max(tx, 1);
    while (tx * ty * 2 <= 256) ty *= 2;
    const long long blocks = (rows + ty - 1) / ty;
    SONET_REQUIRE(blocks < (1LL << 31), "upconv_im2col: too many rows");
    upconv_im2col_vec4_kernel<<<static_cast<unsigned>(blocks), dim3(tx, ty), 0, as_stream(stream)>>>(
        in, B, Cin, H, W, xcol);
    return check_launch("upconv_im2col");
  }
  const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, 16LL * sm_count()));
  if (total < (1LL << 32))
    upconv_im2col_kernel<uint32_t><<<grid, 256, 0, as_stream(stream)>>>(in, B, Cin, H, W, xcol);
  else
    upconv_im2col_kernel<unsigned long long><<<grid, 256, 0, as_stream(stream)>>>(in, B, Cin, H, W, xcol);
  return check_launch("upconv_im2col");
}
