// SSIM and PSNR statistics of image pairs of their own sizes (wn_quality; DESIGN.md 4.16).
//
// Two launches per call, no per-pixel scratch:
//   quality_reduce_kernel  per image: min and max of out and ref, and the sum of squared differences, as one float64
//                          partial per block; the last block of an image reduces its partials in index order, and the
//                          last image of a group derives the group's c1, c2 and shift from the group's data range
//   quality_ssim_kernel    one 32 x 32 output tile of one channel plane per CTA: out and ref with their 5-pixel halo
//                          (reflect indexing) in shared memory, the 11-tap Gaussian run separably over the five
//                          moments, the SSIM of every pixel inside the crop summed into one float64 partial; the last
//                          CTA of an image reduces its partials in index order
// The "last block" of each reduction is found with an integer counter per image and group (zeroed by the table
// upload); no floating-point atomics, so every sum is taken in an order fixed by the image's own size.
//
// SSIM's gradient with respect to out (wn_ssim_grad; DESIGN.md 4.17) runs the same two launches, then:
//   ssim_grad_kernel       one 32 x 32 tile of d(out) of one channel plane per CTA: out and ref with a 10-pixel halo,
//                          the five moments on the tile plus a 5-pixel ring as above, per counted pixel the derivatives
//                          of its SSIM by mu_out, E[out^2] and E[out ref] (A, B, C), their transposed 11-tap pass
//                          folded onto the reflected sources where nothing is cropped, and
//                          d(out) = w*A + 2 out (w*B) + ref (w*C) of centred values; the derivatives by c1 and c2
//                          and the ties of out at the image's min and max are summed per CTA and reduced in index
//                          order by the image's last CTA, then over the group's images by the group's last one
//   ssim_range_kernel      the data-range term: d(loss)/d(range), split evenly over the group's tied extremal elements
#include <limits.h>
#include <math.h>
#include <algorithm>

#include "common.cuh"

namespace wn {
namespace {

constexpr int kThreads = 256;
constexpr long long kReduceMinElems = 8192;  // elements of out (and of ref) per reduction block, at least
constexpr long long kReduceMaxBlocks = 1024; // reduction blocks per image, at most
constexpr int kRad = 5, kTaps = 2 * kRad + 1;
constexpr int kTileW = 32, kTileH = 32;       // output pixels of a CTA
constexpr int kInW = kTileW + 2 * kRad, kInH = kTileH + 2 * kRad;
constexpr int kInStride = kInW + 1;           // odd row stride: the horizontal pass reads rows conflict-free
constexpr int kHStride = kTileW + 1;          // ... and writes its sums conflict-free
constexpr int kMinSide = kRad + 1;            // reflect padding of 5 needs a side of 6

struct QImage {
  const float* out;
  const float* ref;
  int H, W, group;
  int y0, x0, oh, ow;       // the output rectangle SSIM averages (the crop)
  int tiles_x, tiles_y;
  long long r_first;        // first reduction block (and partial) of the image
  long long r_per;          // elements per reduction block
  int r_blocks;
  int s_blocks;
  long long s_first;        // first SSIM CTA (and partial) of the image
};

struct QGroup {
  int first, count;  // the group's images: members[first .. first + count)
};

struct QParams {     // per group, written by the reduction
  float c1, c2, shift;
};

struct Taps {
  float g[kTaps];
};

// the image of block b: the last entry whose first block is <= b
template <class Img, class F>
__device__ int find_image(const Img* imgs, int n, long long b, F first) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first(imgs[mid]) <= b) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// sum over threads in a fixed tree; the result is in red[0]
__device__ void block_sum(double* red, double v) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
}

__device__ void block_minmax(float* lo, float* hi, float a, float b) {
  lo[threadIdx.x] = a;
  hi[threadIdx.x] = b;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      lo[threadIdx.x] = fminf(lo[threadIdx.x], lo[threadIdx.x + s]);
      hi[threadIdx.x] = fmaxf(hi[threadIdx.x], hi[threadIdx.x + s]);
    }
    __syncthreads();
  }
}

// true in every thread of the block that arrives last at counter *cnt of `total` arrivals
__device__ bool arrive_last(int* cnt, int total) {
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(cnt, 1) == total - 1;
  __syncthreads();
  if (last) __threadfence();
  return last;
}

// partial p of an image: {sum of squared differences, min out, max out, min ref, max ref}
constexpr int kRedVals = 5;

__global__ void __launch_bounds__(kThreads) quality_reduce_kernel(const QImage* __restrict__ imgs, int n,
                                                                  const QGroup* __restrict__ groups,
                                                                  const int* __restrict__ members, int* cnt_img,
                                                                  int* cnt_grp, QParams* params, double* part,
                                                                  double* stats) {
  __shared__ double red[kThreads];
  __shared__ float lo[kThreads], hi[kThreads];
  const int i = find_image(imgs, n, blockIdx.x, [](const QImage& q) { return q.r_first; });
  const QImage im = imgs[i];
  const long long k = blockIdx.x - im.r_first;
  const long long total = 3ll * im.H * im.W;
  const long long beg = k * im.r_per, end = min(total, beg + im.r_per);
  float omin = INFINITY, omax = -INFINITY, rmin = INFINITY, rmax = -INFINITY;
  double sq = 0.0;
#pragma unroll 4
  for (long long e = beg + threadIdx.x; e < end; e += kThreads) {
    const float o = __ldg(im.out + e), r = __ldg(im.ref + e);
    omin = fminf(omin, o);
    omax = fmaxf(omax, o);
    rmin = fminf(rmin, r);
    rmax = fmaxf(rmax, r);
    const double d = (double)o - (double)r;
    sq = fma(d, d, sq);
  }
  double* mine = part + (im.r_first + k) * kRedVals;
  block_sum(red, sq);
  if (threadIdx.x == 0) mine[0] = red[0];
  block_minmax(lo, hi, omin, omax);
  if (threadIdx.x == 0) mine[1] = lo[0], mine[2] = hi[0];
  block_minmax(lo, hi, rmin, rmax);
  if (threadIdx.x == 0) mine[3] = lo[0], mine[4] = hi[0];
  if (!arrive_last(cnt_img + i, im.r_blocks)) return;

  // the image's partials in index order
  const double* all = part + im.r_first * kRedVals;
  sq = 0.0;
  omin = rmin = INFINITY;
  omax = rmax = -INFINITY;
  for (int j = threadIdx.x; j < im.r_blocks; j += kThreads) {
    sq += __ldcg(all + j * kRedVals);
    omin = fminf(omin, (float)__ldcg(all + j * kRedVals + 1));
    omax = fmaxf(omax, (float)__ldcg(all + j * kRedVals + 2));
    rmin = fminf(rmin, (float)__ldcg(all + j * kRedVals + 3));
    rmax = fmaxf(rmax, (float)__ldcg(all + j * kRedVals + 4));
  }
  double* st = stats + (size_t)i * WN_QUALITY_STATS;
  block_sum(red, sq);
  if (threadIdx.x == 0) st[2] = red[0];
  block_minmax(lo, hi, omin, omax);
  if (threadIdx.x == 0) st[3] = lo[0], st[4] = hi[0];
  block_minmax(lo, hi, rmin, rmax);
  if (threadIdx.x == 0) st[5] = lo[0], st[6] = hi[0];
  const QGroup g = groups[im.group];
  if (!arrive_last(cnt_grp + im.group, g.count)) return;

  // the group's data range: min and max are exact in any order
  omin = rmin = INFINITY;
  omax = rmax = -INFINITY;
  for (int j = threadIdx.x; j < g.count; j += kThreads) {
    const double* s = stats + (size_t)members[g.first + j] * WN_QUALITY_STATS;
    omin = fminf(omin, (float)__ldcg(s + 3));
    omax = fmaxf(omax, (float)__ldcg(s + 4));
    rmin = fminf(rmin, (float)__ldcg(s + 5));
    rmax = fmaxf(rmax, (float)__ldcg(s + 6));
  }
  block_minmax(lo, hi, omin, omax);
  omin = lo[0];
  omax = hi[0];
  __syncthreads();
  block_minmax(lo, hi, rmin, rmax);
  rmin = lo[0];
  rmax = hi[0];
  if (threadIdx.x == 0) {
    const double range = fmax((double)omax - omin, (double)rmax - rmin);
    QParams p;
    p.c1 = (float)((0.01 * range) * (0.01 * range));
    p.c2 = (float)((0.03 * range) * (0.03 * range));
    // SSIM's variances and covariance are shift-invariant: moments of values centred on the group's mid-range keep
    // E[x^2] - E[x]^2 from cancelling in fp32 (the means are shifted back for the luminance term)
    p.shift = (float)(0.5 * ((double)fminf(omin, rmin) + (double)fmaxf(omax, rmax)));
    params[im.group] = p;
  }
}

__device__ __forceinline__ int reflect_clamp(int v, int n) {
  v = v < 0 ? -v : (v >= n ? 2 * n - 2 - v : v);  // reflect padding: exact for v in [-5, n + 4]
  return min(max(v, 0), n - 1);                     // beyond: only outputs outside the image read it
}

__global__ void __launch_bounds__(kThreads) quality_ssim_kernel(const QImage* __restrict__ imgs, int n,
                                                                const QParams* __restrict__ params, int* cnt_img,
                                                                double* part, double* stats, Taps taps) {
  __shared__ float sp[kInH * kInStride], st[kInH * kInStride];
  __shared__ float sh[5][kInH * kHStride];
  __shared__ double red[kThreads];
  const int i = find_image(imgs, n, blockIdx.x, [](const QImage& q) { return q.s_first; });
  const QImage im = imgs[i];
  const QParams prm = params[im.group];
  const int local = (int)(blockIdx.x - im.s_first);
  const int per_plane = im.tiles_x * im.tiles_y;
  const int plane = local / per_plane, t = local - plane * per_plane;
  const int oy0 = im.y0 + (t / im.tiles_x) * kTileH, ox0 = im.x0 + (t % im.tiles_x) * kTileW;
  const size_t plane_off = (size_t)plane * im.H * im.W;
  const float* P = im.out + plane_off;
  const float* T = im.ref + plane_off;

  for (int idx = threadIdx.x; idx < kInH * kInW; idx += kThreads) {
    const int r = idx / kInW, c = idx - r * kInW;
    const int y = reflect_clamp(oy0 - kRad + r, im.H), x = reflect_clamp(ox0 - kRad + c, im.W);
    const size_t e = (size_t)y * im.W + x;
    sp[r * kInStride + c] = __ldg(P + e) - prm.shift;
    st[r * kInStride + c] = __ldg(T + e) - prm.shift;
  }
  __syncthreads();

  // horizontal pass: rows of the halo, 4 output columns per item (consecutive threads take consecutive rows)
  for (int it = threadIdx.x; it < kInH * (kTileW / 4); it += kThreads) {
    const int r = it % kInH, c0 = (it / kInH) * 4;
    float a[4 + kTaps - 1], b[4 + kTaps - 1];
#pragma unroll
    for (int j = 0; j < 4 + kTaps - 1; j++) {
      a[j] = sp[r * kInStride + c0 + j];
      b[j] = st[r * kInStride + c0 + j];
    }
#pragma unroll
    for (int o = 0; o < 4; o++) {
      float m0 = 0.f, m1 = 0.f, m2 = 0.f, m3 = 0.f, m4 = 0.f;
#pragma unroll
      for (int k = 0; k < kTaps; k++) {
        const float g = taps.g[k], p = a[o + k], q = b[o + k];
        m0 = fmaf(g, p, m0);
        m1 = fmaf(g, q, m1);
        m2 = fmaf(g, p * p, m2);
        m3 = fmaf(g, q * q, m3);
        m4 = fmaf(g, p * q, m4);
      }
      const int s = r * kHStride + c0 + o;
      sh[0][s] = m0;
      sh[1][s] = m1;
      sh[2][s] = m2;
      sh[3][s] = m3;
      sh[4][s] = m4;
    }
  }
  __syncthreads();

  // vertical pass: one column, 4 output rows per thread, and the SSIM of the pixels inside the crop
  const int c = threadIdx.x % kTileW, r0 = (threadIdx.x / kTileW) * 4;
  float m[5][4];
#pragma unroll
  for (int q = 0; q < 5; q++) {
    float v[4 + kTaps - 1];
#pragma unroll
    for (int j = 0; j < 4 + kTaps - 1; j++) v[j] = sh[q][(r0 + j) * kHStride + c];
#pragma unroll
    for (int o = 0; o < 4; o++) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < kTaps; k++) s = fmaf(taps.g[k], v[o + k], s);
      m[q][o] = s;
    }
  }
  double acc = 0.0;
  const bool col_in = ox0 + c < im.x0 + im.ow;
#pragma unroll
  for (int o = 0; o < 4; o++) {
    if (!col_in || oy0 + r0 + o >= im.y0 + im.oh) continue;
    const float mp = m[0][o], mt = m[1][o];
    const float var_p = m[2][o] - mp * mp, var_t = m[3][o] - mt * mt, cov = m[4][o] - mp * mt;
    const float up = mp + prm.shift, ut = mt + prm.shift;
    const float num = (2.f * up * ut + prm.c1) * (2.f * cov + prm.c2);
    const float den = (up * up + ut * ut + prm.c1) * (var_p + var_t + prm.c2);
    acc += (double)(num / den);
  }
  block_sum(red, acc);
  if (threadIdx.x == 0) part[im.s_first + local] = red[0];
  if (!arrive_last(cnt_img + i, im.s_blocks)) return;

  const double* all = part + im.s_first;
  acc = 0.0;
  for (int j = threadIdx.x; j < im.s_blocks; j += kThreads) acc += __ldcg(all + j);
  block_sum(red, acc);
  if (threadIdx.x == 0) {
    double* s = stats + (size_t)i * WN_QUALITY_STATS;
    s[0] = red[0];
    s[1] = 3.0 * im.oh * im.ow;
  }
}

// ---- the gradient (wn_ssim_grad)
constexpr int kGM = kTileW + 2 * kRad;   // 42: moments (and A, B, C) per row and column of a CTA: tile plus ring
constexpr int kGIn = kGM + 2 * kRad;     // 52: input rows and columns: tile plus a 10-pixel halo
constexpr int kGInStride = kGIn + 1;
constexpr int kGMStride = kGM + 1;
constexpr int kGTStride = kTileW + 1;
constexpr int kGItem = 6;                // outputs per item of the forward passes (42 = 7 x 6)
static_assert(kTileW == kTileH && kGM % kGItem == 0, "square tiles, whole items");
// dynamic shared memory: [out, ref halo | later A, B, C on the ring] [5 horizontal moments | later 3 transposed sums]
constexpr int kGRegion0 = 2 * kGIn * kGInStride;
constexpr int kGRegion1 = 5 * kGIn * kGMStride;
static_assert(3 * kGM * kGMStride <= kGRegion0 && 3 * kGM * kGTStride <= kGRegion1, "aliased regions fit");
constexpr size_t kGSmem = (size_t)(kGRegion0 + kGRegion1) * sizeof(float);

struct GImage {
  float* grad;
  double scale;          // of the image's SSIM in the differentiated sum
  long long g_first;     // first gradient CTA (and partial) of the image
  int tiles_x, tiles_y;  // 32 x 32 tiles of the whole plane
  int g_blocks;
};

struct GPart {           // per CTA, then per image (times scale / count): sums of ds/dc1, ds/dc2 and the ties of out
  double d1, d2;         // at the image's max and min
  long long nmax, nmin;
};

struct GRange {          // per group: its extremes of out and what the range term adds at one tied element
  float omin, omax;
  double add_max, add_min;
};

__device__ void block_sum_ll(long long* red, long long v) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
}

// The transposed 11-tap pass at output j of a side of n, from v[k] = the coefficient at j - 5 + k, k in 0..10:
// sum_k g[k] v[k] (the window is symmetric), plus with `fold` the padded positions that reflect onto j: -j for
// j in 1..5, 2n - 2 - j for j in n-6..n-2, each of which gathers the coefficients within 5 of it (all inside v).
// `gs` holds the taps in shared memory for the fold's indexing.
__device__ __forceinline__ float transposed_tap(const Taps& taps, const float* gs, const float* v, int stride, int j,
                                                int n, bool fold) {
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < kTaps; k++) s = fmaf(taps.g[k], v[k * stride], s);
  if (fold) {
    if (j >= 1 && j <= kRad)
      for (int i = 0; i <= kRad - j; i++) s = fmaf(gs[kRad - j - i], v[(i - j + kRad) * stride], s);
    if (j >= n - 1 - kRad && j <= n - 2) {
      const int q = 2 * n - 2 - j;
      for (int i = q - kRad; i < n; i++) s = fmaf(gs[q - i + kRad], v[(i - j + kRad) * stride], s);
    }
  }
  return s;
}

__global__ void __launch_bounds__(kThreads) ssim_grad_kernel(const QImage* __restrict__ imgs,
                                                             const GImage* __restrict__ gimgs, int n,
                                                             const QGroup* __restrict__ groups,
                                                             const int* __restrict__ members,
                                                             const QParams* __restrict__ params,
                                                             const double* __restrict__ stats, int* cnt_img,
                                                             int* cnt_grp, GPart* part, GPart* img_part,
                                                             GRange* ranges, Taps taps) {
  extern __shared__ float smem[];
  float* sp = smem;                        // centred out and ref with the 10-pixel halo
  float* st = smem + kGIn * kGInStride;
  float* coef = smem;                      // A, B, C on the ring (after the horizontal pass)
  float* sh = smem + kGRegion0;            // the horizontal moments, then the transposed horizontal sums
  __shared__ double red[kThreads];
  __shared__ long long redl[kThreads];
  __shared__ float gs[kTaps];
  if (threadIdx.x == 0)  // constant indices: the parameter struct stays out of local memory
#pragma unroll
    for (int k = 0; k < kTaps; k++) gs[k] = taps.g[k];
  const int i = find_image(gimgs, n, blockIdx.x, [](const GImage& q) { return q.g_first; });
  const QImage im = imgs[i];
  const GImage gi = gimgs[i];
  const QParams prm = params[im.group];
  const int local = (int)(blockIdx.x - gi.g_first);
  const int per_plane = gi.tiles_x * gi.tiles_y;
  const int plane = local / per_plane, t = local - plane * per_plane;
  const int gy0 = (t / gi.tiles_x) * kTileH, gx0 = (t % gi.tiles_x) * kTileW;
  const size_t plane_off = (size_t)plane * im.H * im.W;
  const float* P = im.out + plane_off;
  const float* T = im.ref + plane_off;
  const bool fold = im.y0 == 0;            // nothing cropped: padded positions reach counted windows

  for (int idx = threadIdx.x; idx < kGIn * kGIn; idx += kThreads) {
    const int r = idx / kGIn, c = idx - r * kGIn;
    const int y = reflect_clamp(gy0 - 2 * kRad + r, im.H), x = reflect_clamp(gx0 - 2 * kRad + c, im.W);
    const size_t e = (size_t)y * im.W + x;
    sp[r * kGInStride + c] = __ldg(P + e) - prm.shift;
    st[r * kGInStride + c] = __ldg(T + e) - prm.shift;
  }
  __syncthreads();

  // horizontal pass, as quality_ssim_kernel's: kGItem output columns per item
  for (int it = threadIdx.x; it < kGIn * (kGM / kGItem); it += kThreads) {
    const int r = it % kGIn, c0 = (it / kGIn) * kGItem;
    float a[kGItem + kTaps - 1], b[kGItem + kTaps - 1];
#pragma unroll
    for (int j = 0; j < kGItem + kTaps - 1; j++) {
      a[j] = sp[r * kGInStride + c0 + j];
      b[j] = st[r * kGInStride + c0 + j];
    }
#pragma unroll
    for (int o = 0; o < kGItem; o++) {
      float m0 = 0.f, m1 = 0.f, m2 = 0.f, m3 = 0.f, m4 = 0.f;
#pragma unroll
      for (int k = 0; k < kTaps; k++) {
        const float g = taps.g[k], p = a[o + k], q = b[o + k];
        m0 = fmaf(g, p, m0);
        m1 = fmaf(g, q, m1);
        m2 = fmaf(g, p * p, m2);
        m3 = fmaf(g, q * q, m3);
        m4 = fmaf(g, p * q, m4);
      }
      const int s = r * kGMStride + c0 + o;
      sh[0 * kGIn * kGMStride + s] = m0;
      sh[1 * kGIn * kGMStride + s] = m1;
      sh[2 * kGIn * kGMStride + s] = m2;
      sh[3 * kGIn * kGMStride + s] = m3;
      sh[4 * kGIn * kGMStride + s] = m4;
    }
  }
  __syncthreads();

  // vertical pass on the tile and its ring, and at every counted pixel the derivatives of its SSIM s:
  //   A = ds/dmu_out, B = ds/dE[out^2], C = ds/dE[out ref], each times the image's scale over its count;
  // on the tile itself also ds/dc1 and ds/dc2 (the data-range term), in float64
  const float sc = (float)(gi.scale / (3.0 * im.oh * im.ow));
  double d1 = 0.0, d2 = 0.0;
  for (int it = threadIdx.x; it < kGM * (kGM / kGItem); it += kThreads) {
    const int c = it % kGM, r0 = (it / kGM) * kGItem;
    float m[5][kGItem];
#pragma unroll
    for (int q = 0; q < 5; q++) {
      float v[kGItem + kTaps - 1];
#pragma unroll
      for (int j = 0; j < kGItem + kTaps - 1; j++) v[j] = sh[q * kGIn * kGMStride + (r0 + j) * kGMStride + c];
#pragma unroll
      for (int o = 0; o < kGItem; o++) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < kTaps; k++) s = fmaf(taps.g[k], v[o + k], s);
        m[q][o] = s;
      }
    }
    const int x = gx0 - kRad + c;
    const bool col_in = x >= im.x0 && x < im.x0 + im.ow;
    const bool col_core = c >= kRad && c < kRad + kTileW;
#pragma unroll
    for (int o = 0; o < kGItem; o++) {
      const int r = r0 + o, y = gy0 - kRad + r;
      float ca = 0.f, cb = 0.f, cc = 0.f;
      if (col_in && y >= im.y0 && y < im.y0 + im.oh) {
        const float mp = m[0][o], mt = m[1][o];
        const float var_p = m[2][o] - mp * mp, var_t = m[3][o] - mt * mt, cov = m[4][o] - mp * mt;
        const float up = mp + prm.shift, ut = mt + prm.shift;
        const float a1 = 2.f * up * ut + prm.c1, b1 = 2.f * cov + prm.c2;
        const float a2 = up * up + ut * ut + prm.c1, b2 = var_p + var_t + prm.c2;
        const float s = (a1 * b1) / (a2 * b2);
        // d/dmu_out: luminance (ut a2 - up a1 = (ut - up)(ut (ut + up) + c1), no cancellation) and the
        // -mu_out^2 and -mu_out mu_ref of the variance and covariance
        const float lum = 2.f * (ut - up) * (ut * (ut + up) + prm.c1) / (a1 * a2);
        ca = sc * s * (lum + 2.f * (mp / b2 - mt / b1));
        cb = -sc * s / b2;
        cc = 2.f * sc * s / b1;
        if (col_core && r >= kRad && r < kRad + kTileH) {
          const double du = (double)up - ut, dv = (double)var_p + var_t - 2.0 * cov;  // a2 - a1, b2 - b1
          d1 += (double)s * (du * du) / ((double)a1 * a2);
          d2 += (double)s * dv / ((double)b1 * b2);
        }
      }
      const int s = r * kGMStride + c;
      coef[0 * kGM * kGMStride + s] = ca;
      coef[1 * kGM * kGMStride + s] = cb;
      coef[2 * kGM * kGMStride + s] = cc;
    }
  }
  __syncthreads();

  // transposed horizontal pass: ring rows, tile columns, 4 columns per item
  float* th = sh;
  for (int it = threadIdx.x; it < kGM * (kTileW / 4); it += kThreads) {
    const int r = it % kGM, c0 = (it / kGM) * 4;
#pragma unroll
    for (int q = 0; q < 3; q++) {
      const float* v = coef + q * kGM * kGMStride + r * kGMStride + c0;
#pragma unroll
      for (int o = 0; o < 4; o++)
        th[q * kGM * kGTStride + r * kGTStride + c0 + o] = transposed_tap(taps, gs, v + o, 1, gx0 + c0 + o, im.W, fold);
    }
  }
  __syncthreads();

  // transposed vertical pass: one column, 4 rows per thread; d(out) of centred values, and the ties
  const int c = threadIdx.x % kTileW, r0 = (threadIdx.x / kTileW) * 4;
  const int x = gx0 + c;
  const double* sti = stats + (size_t)i * WN_QUALITY_STATS;
  const float imin = (float)sti[3], imax = (float)sti[4];
  long long nmax = 0, nmin = 0;
#pragma unroll
  for (int o = 0; o < 4; o++) {
    const int y = gy0 + r0 + o;
    if (x >= im.W || y >= im.H) continue;
    float tv[3];
#pragma unroll
    for (int q = 0; q < 3; q++)
      tv[q] = transposed_tap(taps, gs, th + q * kGM * kGTStride + (r0 + o) * kGTStride + c, kGTStride, y, im.H, fold);
    const size_t e = (size_t)y * im.W + x;
    const float po = __ldg(P + e), pc = po - prm.shift, tc = __ldg(T + e) - prm.shift;
    gi.grad[plane_off + e] = tv[0] + 2.f * pc * tv[1] + tc * tv[2];
    nmax += po == imax;
    nmin += po == imin;
  }

  GPart* mine = part + gi.g_first + local;
  block_sum(red, d1);
  if (threadIdx.x == 0) mine->d1 = red[0];
  __syncthreads();
  block_sum(red, d2);
  if (threadIdx.x == 0) mine->d2 = red[0];
  block_sum_ll(redl, nmax);
  if (threadIdx.x == 0) mine->nmax = redl[0];
  __syncthreads();
  block_sum_ll(redl, nmin);
  if (threadIdx.x == 0) mine->nmin = redl[0];
  if (!arrive_last(cnt_img + i, gi.g_blocks)) return;

  // the image's partials in index order, times scale / count
  const GPart* all = part + gi.g_first;
  d1 = d2 = 0.0;
  nmax = nmin = 0;
  for (int j = threadIdx.x; j < gi.g_blocks; j += kThreads) {
    d1 += __ldcg(&all[j].d1);
    d2 += __ldcg(&all[j].d2);
    nmax += __ldcg(&all[j].nmax);
    nmin += __ldcg(&all[j].nmin);
  }
  const double per_pixel = gi.scale / (3.0 * im.oh * im.ow);
  block_sum(red, d1);
  if (threadIdx.x == 0) img_part[i].d1 = red[0] * per_pixel;
  __syncthreads();
  block_sum(red, d2);
  if (threadIdx.x == 0) img_part[i].d2 = red[0] * per_pixel;
  block_sum_ll(redl, nmax);
  if (threadIdx.x == 0) img_part[i].nmax = redl[0];
  __syncthreads();
  block_sum_ll(redl, nmin);
  if (threadIdx.x == 0) img_part[i].nmin = redl[0];
  const QGroup g = groups[im.group];
  if (!arrive_last(cnt_grp + im.group, g.count)) return;

  // the group: its extremes as quality_reduce_kernel takes them, then its images' sums in member order
  __shared__ float lo[kThreads], hi[kThreads];
  float omin = INFINITY, omax = -INFINITY, rmin = INFINITY, rmax = -INFINITY;
  for (int j = threadIdx.x; j < g.count; j += kThreads) {
    const double* s = stats + (size_t)members[g.first + j] * WN_QUALITY_STATS;
    omin = fminf(omin, (float)s[3]);
    omax = fmaxf(omax, (float)s[4]);
    rmin = fminf(rmin, (float)s[5]);
    rmax = fmaxf(rmax, (float)s[6]);
  }
  block_minmax(lo, hi, omin, omax);
  omin = lo[0];
  omax = hi[0];
  __syncthreads();
  block_minmax(lo, hi, rmin, rmax);
  rmin = lo[0];
  rmax = hi[0];
  __syncthreads();
  d1 = d2 = 0.0;
  nmax = nmin = 0;
  for (int j = threadIdx.x; j < g.count; j += kThreads) {
    const int m = members[g.first + j];
    const double* s = stats + (size_t)m * WN_QUALITY_STATS;
    d1 += __ldcg(&img_part[m].d1);
    d2 += __ldcg(&img_part[m].d2);
    if ((float)s[4] == omax) nmax += __ldcg(&img_part[m].nmax);
    if ((float)s[3] == omin) nmin += __ldcg(&img_part[m].nmin);
  }
  block_sum(red, d1);
  d1 = red[0];
  __syncthreads();
  block_sum(red, d2);
  d2 = red[0];
  block_sum_ll(redl, nmax);
  nmax = redl[0];
  __syncthreads();
  block_sum_ll(redl, nmin);
  nmin = redl[0];
  if (threadIdx.x == 0) {
    // range = maximum(max out - min out, max ref - min ref): torch.maximum gives out's side all of the gradient,
    // half of it on a tie, none when ref's range is larger; c1 = (0.01 range)^2, c2 = (0.03 range)^2
    const double ro = (double)omax - omin, rr = (double)rmax - rmin, range = fmax(ro, rr);
    const double share = ro > rr ? 1.0 : (ro == rr ? 0.5 : 0.0);
    const double d_range = share * (2e-4 * range * d1 + 18e-4 * range * d2);
    GRange gr;
    gr.omin = omin;
    gr.omax = omax;
    gr.add_max = share == 0.0 ? 0.0 : d_range / (double)nmax;  // max() and min() split evenly over ties
    gr.add_min = share == 0.0 ? 0.0 : d_range / (double)nmin;
    ranges[im.group] = gr;
  }
}

// d(loss)/d(range) at the group's extremal elements of out: + at the max, - at the min, over the reduction blocks
__global__ void __launch_bounds__(kThreads) ssim_range_kernel(const QImage* __restrict__ imgs,
                                                              const GImage* __restrict__ gimgs, int n,
                                                              const GRange* __restrict__ ranges) {
  const int i = find_image(imgs, n, blockIdx.x, [](const QImage& q) { return q.r_first; });
  const QImage im = imgs[i];
  const GRange gr = ranges[im.group];
  if (gr.add_max == 0.0 && gr.add_min == 0.0) return;
  float* grad = gimgs[i].grad;
  const long long k = blockIdx.x - im.r_first;
  const long long total = 3ll * im.H * im.W;
  const long long beg = k * im.r_per, end = min(total, beg + im.r_per);
#pragma unroll 4
  for (long long e = beg + threadIdx.x; e < end; e += kThreads) {
    const float o = __ldg(im.out + e);
    if (o != gr.omax && o != gr.omin) continue;
    double v = grad[e];
    if (o == gr.omax) v += gr.add_max;
    if (o == gr.omin) v -= gr.add_min;
    grad[e] = (float)v;
  }
}

// The plan of a call: per image its crop, tiles and blocks, and the sizes of the workspace parts.
struct QPlan {
  std::vector<QImage> imgs;
  long long r_total = 0, s_total = 0;
};

QImage plan_image(int H, int W) {
  QImage q = {};
  q.H = H;
  q.W = W;
  const bool crop = H > 2 * kRad && W > 2 * kRad;  // metrics.ssim crops only when both sides exceed 10
  q.y0 = q.x0 = crop ? kRad : 0;
  q.oh = crop ? H - 2 * kRad : H;
  q.ow = crop ? W - 2 * kRad : W;
  q.tiles_y = (q.oh + kTileH - 1) / kTileH;
  q.tiles_x = (q.ow + kTileW - 1) / kTileW;
  const long long total = 3ll * H * W;
  const long long per = (total + kReduceMaxBlocks - 1) / kReduceMaxBlocks;
  q.r_per = (per < kReduceMinElems ? kReduceMinElems : (per + kThreads - 1) / kThreads * kThreads);
  q.r_blocks = (int)((total + q.r_per - 1) / q.r_per);
  q.s_blocks = 3 * q.tiles_x * q.tiles_y;
  return q;
}

// false when an image is below 6 x 6 or over the size limit, or the grid would not fit an int
bool plan(const int* hs, const int* ws, int n, QPlan* p) {
  p->imgs.resize(n);
  for (int i = 0; i < n; i++) {
    if (hs[i] < kMinSide || ws[i] < kMinSide || (size_t)hs[i] * ws[i] > (size_t)0x7fffffff / 3) return false;
    QImage q = plan_image(hs[i], ws[i]);
    q.r_first = p->r_total;
    q.s_first = p->s_total;
    p->r_total += q.r_blocks;
    p->s_total += q.s_blocks;
    p->imgs[i] = q;
  }
  return p->r_total <= INT_MAX && p->s_total <= INT_MAX;
}

HostTable quality_table(int n) {
  return HostTable({(size_t)n * sizeof(QImage), (size_t)n * sizeof(QGroup), (size_t)n * sizeof(int),
                    (size_t)3 * n * sizeof(int)});
}

// workspace: [table | params | reduction partials | SSIM partials] from the first 256-byte boundary
size_t workspace_bytes(const QPlan& p, int n) {
  return 256 + quality_table(n).bytes() + align256((size_t)n * sizeof(QParams)) +
         align256((size_t)p.r_total * kRedVals * sizeof(double)) + align256((size_t)p.s_total * sizeof(double));
}

Taps gaussian_taps() {
  double g[kTaps], sum = 0.0;
  for (int k = 0; k < kTaps; k++) {
    const double x = k - kRad;
    g[k] = exp(-(x * x) / (2.0 * 1.5 * 1.5));
    sum += g[k];
  }
  Taps t;
  for (int k = 0; k < kTaps; k++) t.g[k] = (float)(g[k] / sum);
  return t;
}

// the gradient CTAs of each image: 32 x 32 tiles of its whole planes; their count, 0 when it would not fit an int
long long grad_plan(const QPlan& p, std::vector<GImage>* g) {
  g->resize(p.imgs.size());
  long long total = 0;
  for (size_t i = 0; i < p.imgs.size(); i++) {
    GImage q = {};
    q.tiles_y = (p.imgs[i].H + kTileH - 1) / kTileH;
    q.tiles_x = (p.imgs[i].W + kTileW - 1) / kTileW;
    q.g_blocks = 3 * q.tiles_x * q.tiles_y;
    q.g_first = total;
    total += q.g_blocks;
    (*g)[i] = q;
  }
  return total <= INT_MAX ? total : 0;
}

HostTable grad_table(int n) { return HostTable({(size_t)n * sizeof(GImage), (size_t)2 * n * sizeof(int)}); }

// workspace: wn_quality's, then [gradient table | per-image sums | per-group range terms | per-CTA partials]
size_t grad_workspace_bytes(const QPlan& p, long long g_total, int n) {
  return workspace_bytes(p, n) + grad_table(n).bytes() + align256((size_t)n * sizeof(GPart)) +
         align256((size_t)n * sizeof(GRange)) + align256((size_t)g_total * sizeof(GPart));
}

// the device table of a call and wn_quality's two launches
struct QDevice {
  const QImage* imgs;
  const QGroup* groups;
  const int* members;
  const QParams* params;
  size_t bytes;  // of the workspace they take from `base`
};

template <class Img>
int quality_launches(wn_handle* h, const Img* images, int n, const QPlan& p, double* stats, uint8_t* base,
                     cudaStream_t stream, QDevice* dev) {
  // the groups' member lists: images in index order within each group
  std::vector<int> count(n, 0), first(n, 0);
  for (int i = 0; i < n; i++) count[images[i].group]++;
  for (int g = 1; g < n; g++) first[g] = first[g - 1] + count[g - 1];
  HostTable table = quality_table(n);
  QImage* ti = table.part<QImage>(0);
  QGroup* tg = table.part<QGroup>(1);
  int* tm = table.part<int>(2);
  for (int g = 0; g < n; g++) tg[g] = QGroup{first[g], 0};
  for (int i = 0; i < n; i++) {
    QImage q = p.imgs[i];
    q.out = images[i].out;
    q.ref = images[i].ref;
    q.group = images[i].group;
    ti[i] = q;
    QGroup& g = tg[q.group];
    tm[g.first + g.count++] = i;
  }
  // part 3, the counters, stays zero

  if (table.upload(base, stream)) return WN_E_CUDA;
  const QImage* d_imgs = table.dev<QImage>(base, 0);
  const QGroup* d_groups = table.dev<QGroup>(base, 1);
  const int* d_members = table.dev<int>(base, 2);
  int* d_cnt = table.dev<int>(base, 3);
  QParams* d_params = (QParams*)(base + table.bytes());
  double* d_rpart = (double*)((uint8_t*)d_params + align256((size_t)n * sizeof(QParams)));
  double* d_spart = (double*)((uint8_t*)d_rpart + align256((size_t)p.r_total * kRedVals * sizeof(double)));

  quality_reduce_kernel<<<(unsigned)p.r_total, kThreads, 0, stream>>>(d_imgs, n, d_groups, d_members, d_cnt,
                                                                      d_cnt + n, d_params, d_rpart, stats);
  WN_LAUNCH_CHECK(h);
  quality_ssim_kernel<<<(unsigned)p.s_total, kThreads, 0, stream>>>(d_imgs, n, d_params, d_cnt + 2 * n, d_spart,
                                                                    stats, gaussian_taps());
  WN_LAUNCH_CHECK(h);
  *dev = QDevice{d_imgs, d_groups, d_members, d_params, workspace_bytes(p, n) - 256};
  return WN_OK;
}

}  // namespace

int quality_plan_check(const int* hs, const int* ws, int n, const char* what) {
  for (int i = 0; i < n; i++)
    if (hs[i] < kMinSide || ws[i] < kMinSide) {
      set_error("%s: image %d is %d x %d: SSIM's reflect padding of 5 needs both sides at least 6", what, i, hs[i],
                ws[i]);
      return WN_E_INVALID;
    }
  QPlan p;
  if (!plan(hs, ws, n, &p)) {
    set_error("%s: images too large", what);
    return WN_E_UNSUPPORTED;
  }
  return WN_OK;
}

size_t quality_workspace_bytes(const int* hs, const int* ws, int n) {
  QPlan p;
  return plan(hs, ws, n, &p) ? workspace_bytes(p, n) : 0;
}

int quality(wn_handle* h, const wn_quality_image* images, int n, double* stats, void* workspace, size_t,
            cudaStream_t stream) {
  std::vector<int> hs, ws;
  ragged_sizes(images, n, &hs, &ws);
  QPlan p;
  plan(hs.data(), ws.data(), n, &p);  // sizes and workspace checked by the caller
  QDevice d;
  return quality_launches(h, images, n, p, stats, (uint8_t*)align256((size_t)workspace), stream, &d);
}

int ssim_grad_plan_check(const int* hs, const int* ws, int n, const char* what) {
  int rc = quality_plan_check(hs, ws, n, what);
  if (rc) return rc;
  QPlan p;
  plan(hs, ws, n, &p);
  std::vector<GImage> g;
  if (!grad_plan(p, &g)) {
    set_error("%s: images too large", what);
    return WN_E_UNSUPPORTED;
  }
  return WN_OK;
}

size_t ssim_grad_workspace_bytes(const int* hs, const int* ws, int n) {
  QPlan p;
  std::vector<GImage> g;
  if (!plan(hs, ws, n, &p)) return 0;
  const long long g_total = grad_plan(p, &g);
  return g_total ? grad_workspace_bytes(p, g_total, n) : 0;
}

int ssim_grad(wn_handle* h, const wn_ssim_grad_image* images, int n, double* stats, void* workspace, size_t,
              cudaStream_t stream) {
  std::vector<int> hs, ws;
  ragged_sizes(images, n, &hs, &ws);
  QPlan p;
  plan(hs.data(), ws.data(), n, &p);  // sizes and workspace checked by the caller
  std::vector<GImage> gimgs;
  const long long g_total = grad_plan(p, &gimgs);
  HostTable table = grad_table(n);
  GImage* ti = table.part<GImage>(0);
  for (int i = 0; i < n; i++) {
    ti[i] = gimgs[i];
    ti[i].grad = images[i].grad;
    ti[i].scale = images[i].scale;
  }
  // part 1, the counters, stays zero

  uint8_t* base = (uint8_t*)align256((size_t)workspace);
  QDevice d;
  int rc = quality_launches(h, images, n, p, stats, base, stream, &d);
  if (rc) return rc;
  uint8_t* gbase = base + d.bytes;
  if (table.upload(gbase, stream)) return WN_E_CUDA;
  const GImage* d_gimgs = table.dev<GImage>(gbase, 0);
  int* d_cnt = table.dev<int>(gbase, 1);
  GPart* d_img_part = (GPart*)(gbase + table.bytes());
  GRange* d_ranges = (GRange*)((uint8_t*)d_img_part + align256((size_t)n * sizeof(GPart)));
  GPart* d_part = (GPart*)((uint8_t*)d_ranges + align256((size_t)n * sizeof(GRange)));

  WN_CUDA(cudaFuncSetAttribute(ssim_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGSmem));
  ssim_grad_kernel<<<(unsigned)g_total, kThreads, kGSmem, stream>>>(d.imgs, d_gimgs, n, d.groups, d.members, d.params,
                                                                    stats, d_cnt, d_cnt + n, d_part, d_img_part,
                                                                    d_ranges, gaussian_taps());
  WN_LAUNCH_CHECK(h);
  ssim_range_kernel<<<(unsigned)p.r_total, kThreads, 0, stream>>>(d.imgs, d_gimgs, n, d_ranges);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

}  // namespace wn
