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
#include <limits.h>
#include <math.h>

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
template <class F>
__device__ int find_image(const QImage* imgs, int n, long long b, F first) {
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

  uint8_t* base = (uint8_t*)align256((size_t)workspace);
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
  return WN_OK;
}

}  // namespace wn
