// The VGG19 perceptual loss of training (training.perceptual_loss) and its gradient d(loss)/d(out), in overlapping
// windows on the tensor cores.  DESIGN.md 4.12.
//
//   L = mean over (n, c < 512, i < H/16, j < W/16) of (255 * (F(out) - F(ref)))^2,
//   F = VGG19 features[:-1] (conv5_4 + ReLU) of the ImageNet-normalised image.
//
//   vgg_pack_kernel        strided fp32 NCHW -> (v - mean) / std -> the 16-channel bf16 hi/lo planes of each window
//   conv_umma_kernel       the 16 convolutions (kEpiAct) and their data gradients (kEpiDgrad, ReLU' from the saved
//                          planes) -- the kernel of the WaterNet layers, from the spec tables below
//   vgg_pool_kernel        2 x 2 max-pool on planes: the first maximum of hi + lo in row-major order, hi/lo copied
//   vgg_pool_bwd_kernel    routes each pooled gradient to the element the forward chose
//   vgg_seed_kernel        each window's owned features: loss partials (float64) and the seed of the backward
//   vgg_fold_kernel        the 3 normalised-channel gradients of a pass, / std, added into d(out) in window order
//
// Windows: a window owns features [q0, q1) per axis and reads input [16 q0 - 128, 16 q1 + 128) clamped to the image,
// so that it holds the 252-pixel support of every owned feature and its pooling grid is the image's.  The windows of
// one pass have one size (a "class": a run of windows of equal extent per axis), so every level of a pass is an exact
// tensor of floor(extent / 2^level) pixels per axis: beyond it the convolutions read zeros, as torch pads.
//
// Arithmetic: the handle's training mode (wn_set_train_mode), DESIGN.md 4.14.  bf16x3 issues three bf16 products per
// product.  WN_MODE_BF16 issues one, a_hi x w_hi (UmmaCfg kFmtHi, the same packed weight images), and the pack, the
// convolutions and the seed store bf16(v) with lo = 0; the pools, the fold and the decoders read hi + lo either way.
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "umma_conv.cuh"

namespace wn {

constexpr int kVggConvs = 16;
constexpr int kVggSteps = 20;                    // 16 convolutions and 4 pools, in features order
constexpr int kVggHalo = 128;                    // input pixels read beyond the owned features, per side
constexpr long long kVggPassPixels = 2ll << 20;  // window pixels per pass by default (max_pass_pixels = 0)
constexpr long long kVggMaxPixels = 8ll << 20;   // cap on a window and on max_pass_pixels
constexpr int kSeedBlocks = 16;                  // loss partials per window

// Forward launches (UmmaCfg): cinpad = K, gw = output channels per column group, ng groups; cout = gw * ng.
struct VggConvSpec {
  int cinpad, gw, concat, tps, mw, ng, cin, cout, level;
};
static constexpr VggConvSpec kVggFwd[kVggConvs] = {
    // cinpad gw concat tps mw ng cin cout level
    {16, 64, 1, 9, 2, 1, 3, 64, 0},          // conv1_1
    {64, 64, 1, 9, 2, 1, 64, 64, 0},         // conv1_2
    {64, 128, 0, 3, 1, 1, 64, 128, 1},       // conv2_1
    {128, 128, 0, 3, 1, 1, 128, 128, 1},     // conv2_2
    {128, 128, 0, 3, 1, 2, 128, 256, 2},     // conv3_1
    {256, 128, 0, 3, 1, 2, 256, 256, 2},     // conv3_2
    {256, 128, 0, 3, 1, 2, 256, 256, 2},     // conv3_3
    {256, 128, 0, 3, 1, 2, 256, 256, 2},     // conv3_4
    {256, 128, 0, 3, 1, 4, 256, 512, 3},     // conv4_1
    {512, 128, 0, 3, 1, 4, 512, 512, 3},     // conv4_2
    {512, 128, 0, 3, 1, 4, 512, 512, 3},     // conv4_3
    {512, 128, 0, 3, 1, 4, 512, 512, 3},     // conv4_4
    {512, 128, 0, 3, 1, 4, 512, 512, 4},     // conv5_1
    {512, 128, 0, 3, 1, 4, 512, 512, 4},     // conv5_2
    {512, 128, 0, 3, 1, 4, 512, 512, 4},     // conv5_3
    {512, 128, 0, 3, 1, 4, 512, 512, 4}};    // conv5_4
// Data-gradient launches of the same convolutions: K = the forward cout, npad * ng = the forward cin (16: 3 real).
struct VggDgradSpec {
  int kpad, npad, ng, concat, tps;
};
static constexpr VggDgradSpec kVggBwd[kVggConvs] = {
    {64, 16, 1, 1, 9},   {64, 64, 1, 1, 9},   {128, 64, 1, 1, 9},  {128, 128, 1, 0, 3},
    {256, 128, 1, 0, 3}, {256, 128, 2, 0, 3}, {256, 128, 2, 0, 3}, {256, 128, 2, 0, 3},
    {512, 128, 2, 0, 3}, {512, 128, 4, 0, 3}, {512, 128, 4, 0, 3}, {512, 128, 4, 0, 3},
    {512, 128, 4, 0, 3}, {512, 128, 4, 0, 3}, {512, 128, 4, 0, 3}, {512, 128, 4, 0, 3}};
static_assert(kVggBwd[0].npad * kVggBwd[0].ng == 16 && kVggBwd[15].kpad == kVggFwd[15].cout, "dgrad table");

// The 20 launches of the forward: conv index, or -1 for a pool into `level`; `c` = output channels.
struct VggStep {
  int conv, level, c;
};
static constexpr VggStep kSteps[kVggSteps] = {
    {0, 0, 64},   {1, 0, 64},   {-1, 1, 64},  {2, 1, 128},  {3, 1, 128},  {-1, 2, 128}, {4, 2, 256},
    {5, 2, 256},  {6, 2, 256},  {7, 2, 256},  {-1, 3, 256}, {8, 3, 512},  {9, 3, 512},  {10, 3, 512},
    {11, 3, 512}, {-1, 4, 512}, {12, 4, 512}, {13, 4, 512}, {14, 4, 512}, {15, 4, 512}};

struct VggWeights {
  uint8_t* fwd[kVggConvs];
  float* bias[kVggConvs];
  uint8_t* bwd[kVggConvs];
  float* zero_bias;  // 512 zeros: the dgrad epilogue has no bias
  float* dense;      // packing scratch, 512 x 512 x 9
};

// ------------------------------------------------------------------------------------------
// Window geometry (host and device)
// ------------------------------------------------------------------------------------------
// One axis: S pixels, F = S / 16 features, q features per window, count windows.  Window k owns [k q, min(F, (k+1) q))
// and reads [max(0, 16 k q - 128), min(S, 16 (k+1) q + 128)).
struct VggAxis {
  int S, F, q, count;
};
__host__ __device__ __forceinline__ int ax_start(const VggAxis& a, int k) {
  const long long v = 16ll * k * a.q - kVggHalo;
  return v < 0 ? 0 : (int)v;
}
__host__ __device__ __forceinline__ int ax_end(const VggAxis& a, int k) {
  const long long v = 16ll * (k + 1) * a.q + kVggHalo;
  return v > a.S ? a.S : (int)v;
}
static VggAxis vgg_axis(int S, int tile) {
  VggAxis a;
  a.S = S;
  a.F = S / 16;
  a.q = tile > 0 ? (tile + 15) / 16 : a.F;
  if (a.q > a.F) a.q = a.F;
  a.count = (a.F + a.q - 1) / a.q;
  return a;
}

// A pass: `count` windows of one class, the windows w0 .. w0 + count - 1 of the class's enumeration (image, window
// row ky in [ky0, ky0 + nky), window column kx in [kx0, kx0 + nkx)), all h x w pixels.  base = global index of the
// class's first window (the order of the loss partials).
struct VggPass {
  VggAxis ay, ax;
  int ky0, nky, kx0, nkx;
  int h, w;
  long long w0, base;
  int count;
};
struct VggWin {
  int img, ys, xs, fy0, fy1, fx0, fx1;
};
__device__ __forceinline__ VggWin vgg_window(const VggPass& p, int i) {
  const long long j = p.w0 + i;
  const int per = p.nky * p.nkx;
  const int r = (int)(j % per);
  const int ky = p.ky0 + r / p.nkx, kx = p.kx0 + r % p.nkx;
  VggWin v;
  v.img = (int)(j / per);
  v.ys = ax_start(p.ay, ky);
  v.xs = ax_start(p.ax, kx);
  v.fy0 = ky * p.ay.q;
  v.fy1 = min(p.ay.F, (ky + 1) * p.ay.q);
  v.fx0 = kx * p.ax.q;
  v.fx1 = min(p.ax.F, (kx + 1) * p.ax.q);
  return v;
}

// Runs of consecutive windows of equal extent along one axis: (first window, count, extent).
struct VggRun {
  int k0, nk, size;
};
static std::vector<VggRun> vgg_runs(const VggAxis& a) {
  std::vector<VggRun> runs;
  for (int k = 0; k < a.count; k++) {
    const int s = ax_end(a, k) - ax_start(a, k);
    if (!runs.empty() && runs.back().size == s) runs.back().nk++;
    else runs.push_back({k, 1, s});
  }
  return runs;
}

// The passes of a call, in order; every pass carries its class's base.  Returns 0 or a WN_E_* code (error set).
static int vgg_plan(int n, int H, int W, int tile_h, int tile_w, long long max_pass_pixels, std::vector<VggPass>* out,
                    long long* total_windows) {
  if (n <= 0 || n > 65535 || H < 16 || W < 16 || tile_h < 0 || tile_w < 0 || (tile_h == 0) != (tile_w == 0) ||
      max_pass_pixels < 0) {
    set_error("perceptual loss: bad arguments n=%d h=%d w=%d tile=%dx%d max_pass_pixels=%lld (n in 1..65535, images "
              "at least 16 x 16, tiles both 0 or both positive)", n, H, W, tile_h, tile_w, max_pass_pixels);
    return WN_E_INVALID;
  }
  if ((size_t)H * W > (size_t)0x7fffffff / 3 || max_pass_pixels > kVggMaxPixels) {
    set_error("perceptual loss: image of %dx%d or max_pass_pixels=%lld over the limits", H, W, max_pass_pixels);
    return WN_E_UNSUPPORTED;
  }
  const long long limit = max_pass_pixels ? max_pass_pixels : kVggPassPixels;
  const VggAxis ay = vgg_axis(H, tile_h), ax = vgg_axis(W, tile_w);
  const std::vector<VggRun> ry = vgg_runs(ay), rx = vgg_runs(ax);
  long long base = 0;
  for (const VggRun& a : ry)
    for (const VggRun& b : rx) {
      const long long px = (long long)a.size * b.size;
      if (px > kVggMaxPixels) {
        set_error("perceptual loss: a %dx%d window exceeds %lld pixels; pass a tile", a.size, b.size, kVggMaxPixels);
        return WN_E_UNSUPPORTED;
      }
      const long long total = (long long)n * a.nk * b.nk;
      long long per = limit / px;
      per = per < 1 ? 1 : per > 65535 ? 65535 : per;
      for (long long w0 = 0; w0 < total; w0 += per) {
        VggPass p;
        p.ay = ay;
        p.ax = ax;
        p.ky0 = a.k0; p.nky = a.nk;
        p.kx0 = b.k0; p.nkx = b.nk;
        p.h = a.size; p.w = b.size;
        p.w0 = w0;
        p.base = base;
        p.count = (int)(total - w0 < per ? total - w0 : per);
        if (out) out->push_back(p);
      }
      base += total;
    }
  *total_windows = base;
  return WN_OK;
}

// Buffers of one pass; every region 1 KiB aligned.  px(l) = (h >> l) * (w >> l).
struct VggBuffers {
  uint4* act0;           // 16 channels, level 0
  uint4* ping;           // scratch of the ref forward and of the gradient chain
  uint4* pong;
  uint4* fref;           // conv5_4 of ref
  uint4* saved[kVggSteps];  // every launch's output of the out forward
};
static size_t a1k(size_t v) { return (v + 1023) / 1024 * 1024; }
static size_t step_bytes(int k, int h, int w) {
  const int l = kSteps[k].level;
  return (size_t)(h >> l) * (w >> l) * kSteps[k].c * 4;
}
static size_t scratch_bytes(int h, int w) {
  size_t m = (size_t)h * w * 64;
  for (int k = 0; k < kVggSteps; k++) m = step_bytes(k, h, w) > m ? step_bytes(k, h, w) : m;
  return m;
}
static size_t pass_bytes(int cnt, int h, int w, VggBuffers* b, uint8_t* ws) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint4* p = ws ? (uint4*)(ws + off) : nullptr;
    off += a1k((size_t)cnt * bytes);
    return p;
  };
  VggBuffers t;
  t.act0 = take((size_t)h * w * 64);
  t.ping = take(scratch_bytes(h, w));
  t.pong = take(scratch_bytes(h, w));
  t.fref = take(step_bytes(kVggSteps - 1, h, w));
  for (int k = 0; k < kVggSteps; k++) t.saved[k] = take(step_bytes(k, h, w));
  if (b) *b = t;
  return off;
}
// [partials: kSeedBlocks doubles per window][one pass], + 1 KiB for the alignment of the base
static size_t workspace_from_plan(const std::vector<VggPass>& passes, long long total) {
  size_t m = 0;
  for (const VggPass& p : passes) {
    const size_t b = pass_bytes(p.count, p.h, p.w, nullptr, nullptr);
    m = b > m ? b : m;
  }
  return a1k((size_t)total * kSeedBlocks * sizeof(double)) + m + 1024;
}

size_t vgg_loss_workspace_bytes(int n, int H, int W, int tile_h, int tile_w, long long max_pass_pixels) {
  std::vector<VggPass> passes;
  long long total = 0;
  if (vgg_plan(n, H, W, tile_h, tile_w, max_pass_pixels, &passes, &total)) return 0;
  return workspace_from_plan(passes, total);
}

// ------------------------------------------------------------------------------------------
// Kernels
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float bf_at(const uint4& u, int j) {
  const uint32_t w = j < 2 ? u.x : j < 4 ? u.y : j < 6 ? u.z : u.w;
  return __uint_as_float((j & 1) ? (w & 0xffff0000u) : (w << 16));
}
__device__ __forceinline__ uint32_t bf_bits(const uint4& u, int j) {
  const uint32_t w = j < 2 ? u.x : j < 4 ? u.y : j < 6 ? u.z : u.w;
  return (j & 1) ? (w >> 16) : (w & 0xffffu);
}
__device__ __forceinline__ void bf_put(uint32_t* w, int j, uint32_t bits) { w[j >> 1] |= bits << ((j & 1) * 16); }

// scatter one OIHW 3 x 3 tensor into dense [row][K][9]: forward rows = cout, K = cin; transposed (the data gradient)
// rows = cin, K = cout, taps flipped
static __global__ void vgg_scatter_kernel(const float* __restrict__ src, float* __restrict__ dense, int co, int ci,
                                          int kpad, int transposed) {
  const int total = co * ci * 9;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int t = i % 9, c = (i / 9) % ci, o = i / (9 * ci);
    if (transposed) dense[((size_t)c * kpad + o) * 9 + (8 - t)] = src[i];
    else dense[((size_t)o * kpad + c) * 9 + t] = src[i];
  }
}

// pixel blockIdx.x * 256 + tid of window blockIdx.y of the pass: (v - mean) / std of the 3 channels (as torch
// evaluates it in fp32) -> hi/lo planes of 16 channels (13 zero).  HI: single-pass bf16, bf16(v) and lo = 0.
struct ImgArgs {
  const float* p;
  long long s[4];
};
template <bool HI = false>
static __global__ void __launch_bounds__(256) vgg_pack_kernel(ImgArgs a, VggPass p, uint4* __restrict__ act0) {
  const int hw = p.h * p.w;
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= hw) return;
  const VggWin v = vgg_window(p, blockIdx.y);
  const int wy = pix / p.w, wx = pix - wy * p.w;
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
  float f[4] = {0.f, 0.f, 0.f, 0.f};
  const float* src = a.p + v.img * a.s[0] + (v.ys + wy) * a.s[2] + (v.xs + wx) * a.s[3];
#pragma unroll
  for (int c = 0; c < 3; c++) f[c] = __fdiv_rn(__fsub_rn(src[c * a.s[1]], mean[c]), stdv[c]);
  uint32_t hi[2], lo[2];
  if constexpr (HI) {
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const __nv_bfloat162 hb = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
      hi[j] = *reinterpret_cast<const uint32_t*>(&hb);
      lo[j] = 0u;
    }
  } else {
    split_bf16x2(f[0], f[1], hi[0], lo[0]);
    split_bf16x2(f[2], f[3], hi[1], lo[1]);
  }
  uint4* o = act0 + (size_t)blockIdx.y * 4 * hw + pix;
  const uint4 z = make_uint4(0, 0, 0, 0);
  o[0] = make_uint4(hi[0], hi[1], 0, 0);
  o[hw] = z;
  o[2 * (size_t)hw] = make_uint4(lo[0], lo[1], 0, 0);
  o[3 * (size_t)hw] = z;
}

// index (0..3, row-major) of the first maximum of hi + lo among the four candidates, per channel
__device__ __forceinline__ void pool_choose(const uint4* hi, const uint4* lo, int* best) {
#pragma unroll
  for (int j = 0; j < 8; j++) {
    float m = bf_at(hi[0], j) + bf_at(lo[0], j);
    int b = 0;
#pragma unroll
    for (int k = 1; k < 4; k++) {
      const float v = bf_at(hi[k], j) + bf_at(lo[k], j);
      if (v > m) { m = v; b = k; }
    }
    best[j] = b;
  }
}

// 2 x 2 max-pool of planes [cnt][2P][H][W] -> [cnt][2P][H/2][W/2]; item = (plane, output pixel) of window blockIdx.y
static __global__ void __launch_bounds__(256) vgg_pool_kernel(const uint4* __restrict__ in, uint4* __restrict__ out,
                                                              int P, int H, int W) {
  const int Ho = H / 2, Wo = W / 2, hwo = Ho * Wo;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= P * hwo) return;
  const int pl = t / hwo, o = t - pl * hwo, oy = o / Wo, ox = o - oy * Wo;
  const size_t hw = (size_t)H * W;
  const uint4* bh = in + ((size_t)blockIdx.y * 2 * P + pl) * hw;
  const uint4* bl = bh + (size_t)P * hw;
  uint4 hi[4], lo[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const size_t q = (size_t)(2 * oy + (k >> 1)) * W + 2 * ox + (k & 1);
    hi[k] = bh[q];
    lo[k] = bl[q];
  }
  uint32_t oh[4] = {0, 0, 0, 0}, ol[4] = {0, 0, 0, 0};
#pragma unroll
  for (int j = 0; j < 8; j++) {  // the selection of pool_choose, carrying the chosen element's bits
    float m = bf_at(hi[0], j) + bf_at(lo[0], j);
    uint32_t bh = bf_bits(hi[0], j), bl = bf_bits(lo[0], j);
#pragma unroll
    for (int k = 1; k < 4; k++) {
      const float v = bf_at(hi[k], j) + bf_at(lo[k], j);
      if (v > m) {
        m = v;
        bh = bf_bits(hi[k], j);
        bl = bf_bits(lo[k], j);
      }
    }
    bf_put(oh, j, bh);
    bf_put(ol, j, bl);
  }
  uint4* d = out + ((size_t)blockIdx.y * 2 * P + pl) * hwo + o;
  d[0] = make_uint4(oh[0], oh[1], oh[2], oh[3]);
  d[(size_t)P * hwo] = make_uint4(ol[0], ol[1], ol[2], ol[3]);
}

// backward of the pool: item = (plane, input pixel); the pooled gradient goes to the element the forward chose
// (recomputed from the saved input planes), every other element and the floored edge get 0
static __global__ void __launch_bounds__(256) vgg_pool_bwd_kernel(const uint4* __restrict__ g, const uint4* __restrict__ saved,
                                                                  uint4* __restrict__ out, int P, int H, int W) {
  const int Ho = H / 2, Wo = W / 2, hw = H * W, hwo = Ho * Wo;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= P * hw) return;
  const int pl = t / hw, q = t - pl * hw, y = q / W, x = q - y * W;
  uint32_t oh[4] = {0, 0, 0, 0}, ol[4] = {0, 0, 0, 0};
  if (y < 2 * Ho && x < 2 * Wo) {
    const uint4* bh = saved + ((size_t)blockIdx.y * 2 * P + pl) * hw;
    const uint4* bl = bh + (size_t)P * hw;
    const int oy = y >> 1, ox = x >> 1, self = (y & 1) * 2 + (x & 1);
    uint4 hi[4], lo[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const size_t c = (size_t)(2 * oy + (k >> 1)) * W + 2 * ox + (k & 1);
      hi[k] = bh[c];
      lo[k] = bl[c];
    }
    int best[8];
    pool_choose(hi, lo, best);
    const uint4* gp = g + ((size_t)blockIdx.y * 2 * P + pl) * hwo + oy * Wo + ox;
    const uint4 gh = gp[0], gl = gp[(size_t)P * hwo];
#pragma unroll
    for (int j = 0; j < 8; j++)
      if (best[j] == self) {
        bf_put(oh, j, bf_bits(gh, j));
        bf_put(ol, j, bf_bits(gl, j));
      }
  }
  uint4* d = out + ((size_t)blockIdx.y * 2 * P + pl) * hw + q;
  d[0] = make_uint4(oh[0], oh[1], oh[2], oh[3]);
  d[(size_t)P * hw] = make_uint4(ol[0], ol[1], ol[2], ol[3]);
}

// Window blockIdx.y, block blockIdx.x of kSeedBlocks: over its owned features, partial = sum of (255 (Fo - Fr))^2 in
// float64, stored at partials[(base + w0 + window) * kSeedBlocks + block]; with g, the seed of the backward: scale *
// (Fo - Fr) where Fo > 0 (ReLU' of conv5_4) at owned features, 0 everywhere else in the window.  HI: the seed of the
// single-pass bf16 backward, bf16 and lo = 0 (the loss partials are the same sums of the decoded features).
template <bool HI = false>
static __global__ void __launch_bounds__(256) vgg_seed_kernel(const uint4* __restrict__ fo, const uint4* __restrict__ fr,
                                                              uint4* __restrict__ g, double* __restrict__ partials,
                                                              VggPass p, float scale) {
  __shared__ double red[256];
  const int h4 = p.h >> 4, w4 = p.w >> 4, hw = h4 * w4;
  const int items = 64 * hw;
  const VggWin v = vgg_window(p, blockIdx.y);
  const size_t wbase = (size_t)blockIdx.y * 128 * hw;
  double acc = 0.0;
  for (int t = blockIdx.x * 256 + threadIdx.x; t < items; t += kSeedBlocks * 256) {
    const int pl = t / hw, q = t - pl * hw, wy = q / w4, wx = q - wy * w4;
    const int fy = (v.ys >> 4) + wy, fx = (v.xs >> 4) + wx;
    const bool own = fy >= v.fy0 && fy < v.fy1 && fx >= v.fx0 && fx < v.fx1;
    const size_t o = wbase + (size_t)pl * hw + q, ol = o + (size_t)64 * hw;
    uint32_t sh[4] = {0, 0, 0, 0}, sl[4] = {0, 0, 0, 0};
    if (own) {
      const uint4 oh = fo[o], olo = fo[ol], rh = fr[o], rl = fr[ol];
      float s[8];
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const float a = bf_at(oh, j) + bf_at(olo, j);
        const float d = a - (bf_at(rh, j) + bf_at(rl, j));
        const double e = 255.0 * (double)d;
        acc += e * e;
        s[j] = a > 0.f ? scale * d : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        if constexpr (HI) {
          const __nv_bfloat162 hb = __floats2bfloat162_rn(s[j], s[j + 1]);
          sh[j >> 1] = *reinterpret_cast<const uint32_t*>(&hb);
        } else {
          split_bf16x2(s[j], s[j + 1], sh[j >> 1], sl[j >> 1]);
        }
      }
    }
    if (g) {
      g[o] = make_uint4(sh[0], sh[1], sh[2], sh[3]);
      g[ol] = make_uint4(sl[0], sl[1], sl[2], sl[3]);
    }
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) partials[(size_t)(p.base + p.w0 + blockIdx.y) * kSeedBlocks + blockIdx.x] = red[0];
}

// loss = (sum of the partials in index order per thread, then a fixed tree) / count
static __global__ void __launch_bounds__(256) vgg_loss_kernel(const double* __restrict__ partials, long long m,
                                                              double inv_count, float* __restrict__ loss) {
  __shared__ double red[256];
  double s = 0.0;
  for (long long k = threadIdx.x; k < m; k += 256) s += partials[k];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = (float)(red[0] * inv_count);
}

// the windows along one axis that contain coordinate v, clipped to the run [k0, k0 + nk)
__device__ __forceinline__ void cover(const VggAxis& a, int v, int k0, int nk, int* lo, int* hi) {
  const int step = 16 * a.q;
  int l = (v - kVggHalo) / step - 1, u = (v + kVggHalo) / step;
  l = max(l, k0);
  u = min(u, k0 + nk - 1);
  while (l <= u && ax_end(a, l) <= v) l++;
  while (u >= l && ax_start(a, u) > v) u--;
  *lo = l;
  *hi = u;
}

// d(out) of image img0 + blockIdx.y at pixel (y0 + r, x0 + c): += g / std of every window of the pass containing it,
// in ascending window order.  gin: the pass's gradient with respect to the 16 normalised channels (3 real).
static __global__ void __launch_bounds__(256) vgg_fold_kernel(const uint4* __restrict__ gin, float* __restrict__ dout,
                                                              VggPass p, int img0, int y0, int x0, int rh, int rw) {
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= rh * rw) return;
  const int y = y0 + t / rw, x = x0 + t % rw, img = img0 + blockIdx.y;
  int ylo, yhi, xlo, xhi;
  cover(p.ay, y, p.ky0, p.nky, &ylo, &yhi);
  cover(p.ax, x, p.kx0, p.nkx, &xlo, &xhi);
  const size_t ihw = (size_t)p.ay.S * p.ax.S;
  float* d = dout + (size_t)img * 3 * ihw + (size_t)y * p.ax.S + x;
  float acc[3] = {d[0], d[ihw], d[2 * ihw]};
  const float stdv[3] = {0.229f, 0.224f, 0.225f};
  const size_t hw = (size_t)p.h * p.w;
  for (int ky = ylo; ky <= yhi; ky++)
    for (int kx = xlo; kx <= xhi; kx++) {
      const long long j = ((long long)img * p.nky + (ky - p.ky0)) * p.nkx + (kx - p.kx0);
      if (j < p.w0 || j >= p.w0 + p.count) continue;
      const size_t pix = (size_t)(y - ax_start(p.ay, ky)) * p.w + (x - ax_start(p.ax, kx));
      const uint4* b = gin + (size_t)(j - p.w0) * 4 * hw + pix;
      const uint4 gh = b[0], gl = b[2 * hw];
#pragma unroll
      for (int c = 0; c < 3; c++) acc[c] += __fdiv_rn(bf_at(gh, c) + bf_at(gl, c), stdv[c]);
    }
  d[0] = acc[0];
  d[ihw] = acc[1];
  d[2 * ihw] = acc[2];
}

// test aids: planes [cnt][2C/8][H][W] -> fp32 [cnt][C][H][W]; owned conv5_4 features -> fp32 (N, 512, F_h, F_w)
static __global__ void __launch_bounds__(256) vgg_decode_kernel(const uint4* __restrict__ src, float* __restrict__ dst,
                                                                int P, int hw) {
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= P * hw) return;
  const int pl = t / hw, q = t - pl * hw;
  const uint4* s = src + ((size_t)blockIdx.y * 2 * P + pl) * hw + q;
  const uint4 h = s[0], l = s[(size_t)P * hw];
#pragma unroll
  for (int j = 0; j < 8; j++) dst[((size_t)blockIdx.y * 8 * P + pl * 8 + j) * hw + q] = bf_at(h, j) + bf_at(l, j);
}
static __global__ void __launch_bounds__(256) vgg_store_features_kernel(const uint4* __restrict__ fo,
                                                                        float* __restrict__ dst, VggPass p) {
  const int h4 = p.h >> 4, w4 = p.w >> 4, hw = h4 * w4;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= 64 * hw) return;
  const VggWin v = vgg_window(p, blockIdx.y);
  const int pl = t / hw, q = t - pl * hw, wy = q / w4, wx = q - wy * w4;
  const int fy = (v.ys >> 4) + wy, fx = (v.xs >> 4) + wx;
  if (fy < v.fy0 || fy >= v.fy1 || fx < v.fx0 || fx >= v.fx1) return;
  const size_t o = (size_t)blockIdx.y * 128 * hw + (size_t)pl * hw + q;
  const uint4 h = fo[o], l = fo[o + (size_t)64 * hw];
  const size_t fhw = (size_t)p.ay.F * p.ax.F;
#pragma unroll
  for (int j = 0; j < 8; j++)
    dst[((size_t)v.img * 512 + pl * 8 + j) * fhw + (size_t)fy * p.ax.F + fx] = bf_at(h, j) + bf_at(l, j);
}

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
int vgg_pack_weights(wn_handle* h, const float* const* params, cudaStream_t stream) {
  if (!h->vgg) h->vgg = (VggWeights*)calloc(1, sizeof(VggWeights));
  VggWeights* u = h->vgg;
  for (int i = 0; i < kVggConvs; i++) {  // (re)allocate whatever an earlier, failed call left unallocated
    const VggConvSpec& f = kVggFwd[i];
    const VggDgradSpec& d = kVggBwd[i];
    if (!u->fwd[i]) WN_CUDA(cudaMalloc(&u->fwd[i], (size_t)(f.cinpad / 16) * 9 * f.cout * 64));
    if (!u->bias[i]) WN_CUDA(cudaMalloc(&u->bias[i], f.cout * sizeof(float)));
    if (!u->bwd[i]) WN_CUDA(cudaMalloc(&u->bwd[i], (size_t)(d.kpad / 16) * 9 * d.npad * d.ng * 64));
  }
  if (!u->zero_bias) WN_CUDA(cudaMalloc(&u->zero_bias, 512 * sizeof(float)));
  if (!u->dense) WN_CUDA(cudaMalloc(&u->dense, (size_t)512 * 512 * 9 * sizeof(float)));
  WN_CUDA(cudaMemsetAsync(u->zero_bias, 0, 512 * sizeof(float), stream));
  for (int i = 0; i < kVggConvs; i++) {
    const VggConvSpec& f = kVggFwd[i];
    const VggDgradSpec& d = kVggBwd[i];
    // forward: dense [cout][cinpad][9], column group g = rows [g gw, (g + 1) gw)
    WN_CUDA(cudaMemsetAsync(u->dense, 0, (size_t)f.cout * f.cinpad * 9 * sizeof(float), stream));
    vgg_scatter_kernel<<<256, 256, 0, stream>>>(params[2 * i], u->dense, f.cout, f.cin, f.cinpad, 0);
    WN_LAUNCH_CHECK(h);
    WN_CUDA(cudaMemcpyAsync(u->bias[i], params[2 * i + 1], f.cout * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    const size_t fgroup = (size_t)(f.cinpad / 16) * 9 * f.gw * 64;
    for (int g = 0; g < f.ng; g++) {
      pack_stages_kernel<<<256, 256, 0, stream>>>(u->dense, (__nv_bfloat16*)(u->fwd[i] + g * fgroup), f.gw, f.cinpad, 9,
                                                  f.concat, 1, g * f.gw);
      WN_LAUNCH_CHECK(h);
    }
    // data gradient: dense [cin (padded)][cout][9], taps flipped
    const int rows = d.npad * d.ng;
    WN_CUDA(cudaMemsetAsync(u->dense, 0, (size_t)rows * d.kpad * 9 * sizeof(float), stream));
    vgg_scatter_kernel<<<256, 256, 0, stream>>>(params[2 * i], u->dense, f.cout, f.cin, d.kpad, 1);
    WN_LAUNCH_CHECK(h);
    const size_t bgroup = (size_t)(d.kpad / 16) * 9 * d.npad * 64;
    for (int g = 0; g < d.ng; g++) {
      pack_stages_kernel<<<256, 256, 0, stream>>>(u->dense, (__nv_bfloat16*)(u->bwd[i] + g * bgroup), d.npad, d.kpad, 9,
                                                  d.concat, 1, g * d.npad);
      WN_LAUNCH_CHECK(h);
    }
  }
  return WN_OK;
}

void vgg_free(wn_handle* h) {
  if (!h->vgg) return;
  for (int i = 0; i < kVggConvs; i++) {
    if (h->vgg->fwd[i]) cudaFree(h->vgg->fwd[i]);
    if (h->vgg->bias[i]) cudaFree(h->vgg->bias[i]);
    if (h->vgg->bwd[i]) cudaFree(h->vgg->bwd[i]);
  }
  if (h->vgg->zero_bias) cudaFree(h->vgg->zero_bias);
  if (h->vgg->dense) cudaFree(h->vgg->dense);
  free(h->vgg);
  h->vgg = nullptr;
}

template <int LI>
static int conv_fwd(wn_handle* h, const uint4* in, uint4* out, int cnt, int H, int W, cudaStream_t stream) {
  constexpr VggConvSpec s = kVggFwd[LI];
  ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.N = cnt; a.H = H; a.W = W;
  a.dst0.base = out;
  a.dst0.planes_half = s.cout / 8;
  a.split_c = s.cout;
  a.cout = s.cout;
  // single-pass bf16: the hi rows of the same weight images, at the table's tile geometry
  if (h->train_bf16)
    return launch_conv<3, s.cinpad, s.gw, kEpiAct, s.concat, 1, s.tps, kFmtHi, false, s.mw, s.ng>(
        h, kSlotPost, h->vgg->fwd[LI], h->vgg->bias[LI], (void*)in, a, stream);
  return launch_conv<3, s.cinpad, s.gw, kEpiAct, s.concat, 1, s.tps, 0, false, s.mw, s.ng>(
      h, kSlotPost, h->vgg->fwd[LI], h->vgg->bias[LI], (void*)in, a, stream);
}
template <int LI>
static int conv_dgrad(wn_handle* h, const uint4* in, uint4* out, const uint4* mask, int cnt, int H, int W,
                      cudaStream_t stream) {
  constexpr VggDgradSpec s = kVggBwd[LI];
  constexpr int cout = s.npad * s.ng;
  ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.N = cnt; a.H = H; a.W = W;
  a.dst0.base = out;
  a.dst0.planes_half = cout / 8;
  a.split_c = cout;
  a.cout = cout;
  a.mask_base = mask;  // nullptr: the normalised image, no ReLU in front
  a.mask_planes_half = cout / 8;
  if (h->train_bf16)
    return launch_conv<3, s.kpad, s.npad, kEpiDgrad, s.concat, 1, s.tps, kFmtHi, false, 1, s.ng>(
        h, kSlotPost, h->vgg->bwd[LI], h->vgg->zero_bias, (void*)in, a, stream);
  return launch_conv<3, s.kpad, s.npad, kEpiDgrad, s.concat, 1, s.tps, 0, false, 1, s.ng>(
      h, kSlotPost, h->vgg->bwd[LI], h->vgg->zero_bias, (void*)in, a, stream);
}
template <int LI = 0>
static int conv(wn_handle* h, int li, bool dgrad, const uint4* in, uint4* out, const uint4* mask, int cnt, int H,
                int W, cudaStream_t stream) {
  if (li == LI)
    return dgrad ? conv_dgrad<LI>(h, in, out, mask, cnt, H, W, stream) : conv_fwd<LI>(h, in, out, cnt, H, W, stream);
  if constexpr (LI + 1 < kVggConvs) return conv<LI + 1>(h, li, dgrad, in, out, mask, cnt, H, W, stream);
  set_error("vgg: no convolution %d", li);
  return WN_E_INVALID;
}

// The 20 launches from act0.  keep: every output into b.saved (the backward needs them); otherwise they alternate
// between ping and pong and conv5_4 lands in `last`.  stop >= 0: stop after that launch.
static int vgg_forward(wn_handle* h, const VggBuffers& b, bool keep, uint4* last, int cnt, int H, int W,
                       cudaStream_t stream, int stop = -1) {
  const uint4* in = b.act0;
  for (int k = 0; k < kVggSteps; k++) {
    const VggStep& s = kSteps[k];
    uint4* out = keep ? b.saved[k] : k == kVggSteps - 1 ? last : (k & 1) ? b.pong : b.ping;
    const int hl = H >> s.level, wl = W >> s.level;
    int rc;
    if (s.conv >= 0) {
      rc = conv(h, s.conv, false, in, out, nullptr, cnt, hl, wl, stream);
    } else {
      const int P = s.c / 8, hwo = hl * wl;
      vgg_pool_kernel<<<dim3((P * hwo + 255) / 256, cnt), 256, 0, stream>>>(in, out, P, H >> (s.level - 1),
                                                                            W >> (s.level - 1));
      WN_LAUNCH_CHECK(h);
      rc = WN_OK;
    }
    if (rc) return rc;
    if (k == stop) return WN_OK;
    in = out;
  }
  return WN_OK;
}

// From the seed in ping (conv5_4's gradient, level 4) down to the gradient of the 16 normalised channels; returns the
// buffer that holds it (ping or pong).  stop > 0: stop after the backward of launch `stop` (the gradient with
// respect to that launch's input).
static int vgg_backward(wn_handle* h, const VggBuffers& b, int cnt, int H, int W, cudaStream_t stream, uint4** result,
                        int stop = 0) {
  uint4* g = b.ping;
  uint4* o = b.pong;
  for (int k = kVggSteps - 1; k >= stop; k--) {
    const VggStep& s = kSteps[k];
    const int hl = H >> s.level, wl = W >> s.level;
    if (s.conv >= 0) {
      const int rc = conv(h, s.conv, true, g, o, k > 0 ? b.saved[k - 1] : nullptr, cnt, hl, wl, stream);
      if (rc) return rc;
    } else {
      const int P = s.c / 8, hi = H >> (s.level - 1), wi = W >> (s.level - 1);
      vgg_pool_bwd_kernel<<<dim3((P * hi * wi + 255) / 256, cnt), 256, 0, stream>>>(g, b.saved[k - 1], o, P, hi, wi);
      WN_LAUNCH_CHECK(h);
    }
    uint4* t = g;
    g = o;
    o = t;
  }
  *result = g;
  return WN_OK;
}

static int pack_window(wn_handle* h, const float* img, const int64_t st[4], const VggPass& p, uint4* act0,
                       cudaStream_t stream) {
  ImgArgs a;
  a.p = img;
  for (int k = 0; k < 4; k++) a.s[k] = st[k];
  const dim3 grid((p.h * p.w + 255) / 256, p.count);
  if (h->train_bf16) vgg_pack_kernel<true><<<grid, 256, 0, stream>>>(a, p, act0);
  else vgg_pack_kernel<<<grid, 256, 0, stream>>>(a, p, act0);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

// the loss partials of the pass's windows and, with g, the seed of the backward in the handle's training mode
static int seed_window(wn_handle* h, const uint4* fo, const uint4* fr, uint4* g, double* partials, const VggPass& p,
                       float scale, cudaStream_t stream) {
  const dim3 grid(kSeedBlocks, p.count);
  if (h->train_bf16) vgg_seed_kernel<true><<<grid, 256, 0, stream>>>(fo, fr, g, partials, p, scale);
  else vgg_seed_kernel<<<grid, 256, 0, stream>>>(fo, fr, g, partials, p, scale);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

// features != nullptr: the windowed conv5_4 of `out` into features (N, 512, F_h, F_w), nothing else
static int vgg_run(wn_handle* h, const float* out, const int64_t out_st[4], const float* ref, const int64_t ref_st[4],
                   int n, int H, int W, int tile_h, int tile_w, long long max_pass_pixels, float* loss, float* grad,
                   float* features, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  std::vector<VggPass> passes;
  long long total = 0;
  int rc = vgg_plan(n, H, W, tile_h, tile_w, max_pass_pixels, &passes, &total);
  if (rc) return rc;
  const size_t need = workspace_from_plan(passes, total);
  if (workspace_bytes < need) {
    set_error("perceptual loss workspace too small: %zu < %zu", workspace_bytes, need);
    return WN_E_WORKSPACE;
  }
  if (!h->vgg) {
    set_error("perceptual loss: wn_vgg_pack_weights has not been called");
    return WN_E_STATE;
  }
  if ((rc = get_encoder())) return rc;
  uint8_t* ws = (uint8_t*)(((uintptr_t)workspace + 1023) / 1024 * 1024);
  double* partials = (double*)ws;
  uint8_t* pass_ws = ws + a1k((size_t)total * kSeedBlocks * sizeof(double));
  const long long count = (long long)n * 512 * (H / 16) * (W / 16);
  const float scale = (float)(2.0 * 255.0 * 255.0 / (double)count);
  if (grad) WN_CUDA(cudaMemsetAsync(grad, 0, (size_t)n * 3 * H * W * sizeof(float), stream));
  for (const VggPass& p : passes) {
    VggBuffers b;
    pass_bytes(p.count, p.h, p.w, &b, pass_ws);
    if (features) {
      if ((rc = pack_window(h, out, out_st, p, b.act0, stream))) return rc;
      if ((rc = vgg_forward(h, b, false, b.fref, p.count, p.h, p.w, stream))) return rc;
      const int hw4 = (p.h >> 4) * (p.w >> 4);
      vgg_store_features_kernel<<<dim3((64 * hw4 + 255) / 256, p.count), 256, 0, stream>>>(b.fref, features, p);
      WN_LAUNCH_CHECK(h);
      continue;
    }
    if ((rc = pack_window(h, ref, ref_st, p, b.act0, stream))) return rc;
    if ((rc = vgg_forward(h, b, false, b.fref, p.count, p.h, p.w, stream))) return rc;
    if ((rc = pack_window(h, out, out_st, p, b.act0, stream))) return rc;
    uint4* fo = grad ? b.saved[kVggSteps - 1] : b.saved[0];
    if ((rc = vgg_forward(h, b, grad != nullptr, fo, p.count, p.h, p.w, stream))) return rc;
    if ((rc = seed_window(h, fo, b.fref, grad ? b.ping : nullptr, partials, p, scale, stream))) return rc;
    if (!grad) continue;
    uint4* gin = nullptr;
    if ((rc = vgg_backward(h, b, p.count, p.h, p.w, stream, &gin))) return rc;
    // the bounding box of the pass's windows: windows w0 .. w0 + count - 1 of the (image, row, column) enumeration.
    // Within one image: the window rows from the first window's to the last's, and within one window row the columns
    // from the first to the last; otherwise the class's whole rows or columns.
    const long long per = (long long)p.nky * p.nkx, j1 = p.w0 + p.count - 1;
    const int img0 = (int)(p.w0 / per), img1 = (int)(j1 / per);
    int ra = 0, rb = p.nky - 1, ca = 0, cb = p.nkx - 1;
    if (img0 == img1) {
      ra = (int)(p.w0 % per) / p.nkx;
      rb = (int)(j1 % per) / p.nkx;
      if (ra == rb) {
        ca = (int)(p.w0 % per) % p.nkx;
        cb = (int)(j1 % per) % p.nkx;
      }
    }
    const int y0 = ax_start(p.ay, p.ky0 + ra), y1 = ax_end(p.ay, p.ky0 + rb);
    const int x0 = ax_start(p.ax, p.kx0 + ca), x1 = ax_end(p.ax, p.kx0 + cb);
    const int rh = y1 - y0, rw = x1 - x0;
    vgg_fold_kernel<<<dim3((unsigned)(((long long)rh * rw + 255) / 256), img1 - img0 + 1), 256, 0, stream>>>(
        gin, grad, p, img0, y0, x0, rh, rw);
    WN_LAUNCH_CHECK(h);
  }
  if (features) return WN_OK;
  vgg_loss_kernel<<<1, 256, 0, stream>>>(partials, total * kSeedBlocks, 1.0 / (double)count, loss);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

int vgg_perceptual_loss(wn_handle* h, const float* out, const int64_t out_st[4], const float* ref,
                        const int64_t ref_st[4], int n, int H, int W, int tile_h, int tile_w, long long max_pass_pixels,
                        float* loss, float* grad, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return vgg_run(h, out, out_st, ref, ref_st, n, H, W, tile_h, tile_w, max_pass_pixels, loss, grad, nullptr, workspace,
                 workspace_bytes, stream);
}

// Test aid, whole images in one pass (tile 0 x 0) unless noted:
//   layer 0..19   the output of forward launch `layer` of x, as fp32 (n, C, H >> level, W >> level)
//   layer 20      the conv5_4 features of the windowed call with the tile, (n, 512, H/16, W/16)
//   layer 21      the seed of the backward of the loss of (x, ref): d(loss)/d(conv5_4 before its ReLU), level 4
//   layer 22 + k  the output of the backward launch of forward launch k: d(loss)/d(input of launch k); k = 0 gives
//                 the 16 normalised channels (3 real)
int vgg_debug_layer(wn_handle* h, const float* x, const int64_t st[4], const float* ref, const int64_t ref_st[4],
                    int n, int H, int W, int tile_h, int tile_w, int layer, float* dst, void* workspace,
                    size_t workspace_bytes, cudaStream_t stream) {
  if (layer == kVggSteps)
    return vgg_run(h, x, st, x, st, n, H, W, tile_h, tile_w, 0, nullptr, nullptr, dst, workspace, workspace_bytes,
                   stream);
  const bool bwd = layer > kVggSteps;
  if (layer < 0 || layer > 2 * kVggSteps + 1 || tile_h || tile_w || (bwd && (!ref || !ref_st))) {
    set_error("wn_debug_vgg_layer: layer %d with tile %dx%d (layers 0..19 and 21..41 take whole images, tile 0 x 0; "
              "21..41 need ref)", layer, tile_h, tile_w);
    return WN_E_INVALID;
  }
  std::vector<VggPass> passes;
  long long total = 0;
  int rc = vgg_plan(n, H, W, 0, 0, 0, &passes, &total);
  if (rc) return rc;
  if (passes.size() != 1) {
    set_error("wn_debug_vgg_layer: the %d images do not fit one pass", n);
    return WN_E_UNSUPPORTED;
  }
  if (workspace_bytes < workspace_from_plan(passes, total) || !h->vgg) {
    set_error("wn_debug_vgg_layer: weights not packed or workspace too small");
    return WN_E_WORKSPACE;
  }
  if ((rc = get_encoder())) return rc;
  const VggPass& p = passes[0];
  uint8_t* ws = (uint8_t*)(((uintptr_t)workspace + 1023) / 1024 * 1024);
  VggBuffers b;
  pass_bytes(p.count, p.h, p.w, &b, ws + a1k((size_t)total * kSeedBlocks * sizeof(double)));
  if (!bwd) {
    if ((rc = pack_window(h, x, st, p, b.act0, stream))) return rc;
    if ((rc = vgg_forward(h, b, true, nullptr, p.count, p.h, p.w, stream, layer))) return rc;
    const int l = kSteps[layer].level, P = kSteps[layer].c / 8, hw = (H >> l) * (W >> l);
    vgg_decode_kernel<<<dim3((P * hw + 255) / 256, n), 256, 0, stream>>>(b.saved[layer], dst, P, hw);
    WN_LAUNCH_CHECK(h);
    return WN_OK;
  }
  // the pass of vgg_run with a gradient, stopped after the wanted backward launch
  double* partials = (double*)ws;
  const long long count = (long long)n * 512 * (H / 16) * (W / 16);
  if ((rc = pack_window(h, ref, ref_st, p, b.act0, stream))) return rc;
  if ((rc = vgg_forward(h, b, false, b.fref, p.count, p.h, p.w, stream))) return rc;
  if ((rc = pack_window(h, x, st, p, b.act0, stream))) return rc;
  if ((rc = vgg_forward(h, b, true, nullptr, p.count, p.h, p.w, stream))) return rc;
  if ((rc = seed_window(h, b.saved[kVggSteps - 1], b.fref, b.ping, partials, p,
                        (float)(2.0 * 255.0 * 255.0 / (double)count), stream)))
    return rc;
  uint4* g = b.ping;
  int l = 4, c = 512;
  if (layer > kVggSteps + 1) {
    const int k = layer - (kVggSteps + 2);
    if ((rc = vgg_backward(h, b, p.count, p.h, p.w, stream, &g, k))) return rc;
    l = k ? kSteps[k - 1].level : 0;
    c = k ? kSteps[k - 1].c : 16;
  }
  const int P = c / 8, hw = (H >> l) * (W >> l);
  vgg_decode_kernel<<<dim3((P * hw + 255) / 256, n), 256, 0, stream>>>(g, dst, P, hw);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

}  // namespace wn
