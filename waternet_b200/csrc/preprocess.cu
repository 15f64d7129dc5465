// WaterNet preprocess on the GPU: white balance, gamma, Lab+CLAHE hist-eq, u8->fp32.
//
// Replaces /root/reference/waternet/data.py:6-90 (+ hubconf.py:8-21 arr2ten,
// hubconf.py:24-34 ten2arr).  All three transforms are "global or tile histogram
// -> small LUTs -> one per-pixel pass", so the GPU form is
//
//   stats_kernel   one read of the u8 image: 3x256 RGB histograms per image and
//                  8x8 per-tile histograms of the Lab L channel (shared-memory
//                  atomics, one global merge per CTA)
//   luts_kernel    64 CLAHE LUTs (clip, redistribute, prefix sum) + the 3x256
//                  white-balance LUT (float64 quantiles as numpy computes them)
//   apply_kernel   one per-pixel pass: WB LUT, gamma LUT, RGB->Lab->CLAHE blend->
//                  Lab->RGB in OpenCV's 8-bit fixed point, u/255, writes the four
//                  fp32 NCHW tensors and/or u8 NHWC images and/or -- the end-to-end path --
//                  the first conv layer's operand planes (bf16 levels, 32 B/px)
//
// HBM-bound: 3 B/px read twice, 48 B/px (fp32 tensors) or 32 B/px (operand planes) written -- see DESIGN.md.
// Bit-exact with the reference's numpy/OpenCV output (tests/test_gpu_parity.py::test_preprocess_bit_exact_*).
#include <math.h>
#include <string.h>

#include <type_traits>

#include "common.cuh"

namespace wn {

// ---------------------------------------------------------------------------
// Host: constant tables.  Same formulas as OpenCV's initLabTabs (color_lab.cpp)
// and data.py:61-65; checked against the oracle in tests/test_abi_cpu.py.
// ---------------------------------------------------------------------------
void build_tables_host(Tables* t) {
  for (int i = 0; i < 256; i++) {
    double u = i / 255.0;
    double lin = u <= 0.04045 ? u / 12.92 : pow((u + 0.055) / 1.055, 2.4);
    t->gtab[i] = (uint16_t)rint(255.0 * 8.0 * lin);
    t->gamma[i] = (uint8_t)fmin(fmax(255.0 * pow(i / 255.0, 0.7), 0.0), 255.0);
    t->div255[i] = (float)i / 255.0f;
  }
  for (int i = 0; i < 3072; i++) {
    float x = (float)i / (255.0f * 8.0f);
    float f = x < 0.008856f ? x * 7.787f + 0.13793103448275862f : (float)cbrt((double)x);
    t->ctab[i] = (uint16_t)rintf(32768.0f * f);
  }
  // OpenCV builds this table with its own cube-root approximation, which lands one ulp below
  // the correctly rounded value at two arguments where 32768*f sits on a .5 tie.  Entry 324 is
  // reachable from 8-bit RGB (verified against cv2 over all 2^24 colours), 2079 is not.
  t->ctab[324] = 17745;
  t->ctab[2079] = 32975;
  for (int i = 0; i < 256; i++) {
    float li = (float)i * 100.0f / 255.0f;
    float y, fy;
    if (li <= 8.0f) {
      y = li / 903.3f;
      fy = 7.787f * y + 16.0f / 116.0f;
    } else {
      fy = (li + 16.0f) / 116.0f;
      y = fy * fy * fy;
    }
    t->ytab[i] = (int16_t)rintf(y * 16384.0f);
    t->fytab[i] = (int16_t)rintf(fy * 16384.0f);
  }
  for (int i = 0; i < 4096; i++) {
    double x = i / 4096.0;
    double s = x <= 0.0031308 ? 12.92 * x : 1.055 * pow(x, 1.0 / 2.4) - 0.055;
    double v = rint(255.0 * s);
    t->igtab[i] = (uint8_t)fmin(fmax(v, 0.0), 255.0);
  }
}

// ---------------------------------------------------------------------------
// Device helpers: OpenCV 8-bit fixed-point colour conversion
// ---------------------------------------------------------------------------
__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }
__device__ __forceinline__ int clamp255(int v) { return min(max(v, 0), 255); }

// COLOR_RGB2LAB, L only needs fY.
__device__ __forceinline__ int lab_L(const uint16_t* gtab, const uint16_t* ctab, int r, int g,
                                     int b) {
  int R = gtab[r], G = gtab[g], B = gtab[b];
  int fY = ctab[descale(R * 871 + G * 2929 + B * 296, 12)];
  return clamp255(descale(296 * fY - 1336934, 15));
}

__device__ __forceinline__ void rgb2lab(const uint16_t* gtab, const uint16_t* ctab, int r, int g,
                                        int b, int& L, int& A, int& Bv) {
  int R = gtab[r], G = gtab[g], B = gtab[b];
  int fX = ctab[descale(R * 1777 + G * 1541 + B * 778, 12)];
  int fY = ctab[descale(R * 871 + G * 2929 + B * 296, 12)];
  int fZ = ctab[descale(R * 73 + G * 448 + B * 3575, 12)];
  L = clamp255(descale(296 * fY - 1336934, 15));
  A = clamp255(descale(500 * (fX - fY) + 128 * 32768, 15));
  Bv = clamp255(descale(200 * (fY - fZ) + 128 * 32768, 15));
}

// OpenCV's abToXZ_b table as arithmetic (C integer division truncates toward zero).
__device__ __forceinline__ int ab_to_xz(int t) {
  return t <= 3390 ? t * 108 / 841 - 290 : (t * t / 16384) * t / 16384;
}

__device__ __forceinline__ void lab2rgb(const int16_t* ytab, const int16_t* fytab,
                                        const uint8_t* igtab, int L, int A, int Bv, int& r, int& g,
                                        int& b) {
  int y = ytab[L];
  int ify = fytab[L];
  int adiv = ((5 * A * 53687 + 128) >> 13) - 4194;
  int bdiv = ((Bv * 41943 + 16) >> 9) - 10485 + 1;
  int x = ab_to_xz(ify + adiv);
  int z = ab_to_xz(ify - bdiv);
  int ro = descale(12615 * x - 6296 * y - 2223 * z, 14);
  int go = descale(-3773 * x + 7684 * y + 185 * z, 14);
  int bo = descale(217 * x - 836 * y + 4715 * z, 14);
  r = igtab[min(max(ro, 0), 4095)];
  g = igtab[min(max(go, 0), 4095)];
  b = igtab[min(max(bo, 0), 4095)];
}

// BORDER_REFLECT_101 index (cv::borderInterpolate), p >= 0.
__device__ __forceinline__ int reflect101(int p, int len) {
  if (len == 1) return 0;
  while (p >= len) {
    p = 2 * (len - 1) - p;
    if (p < 0) p = -p;
  }
  return p;
}

// ---------------------------------------------------------------------------
// Pass 1: histograms.  grid = (64 tiles, slabs, N), 256 threads.
// ---------------------------------------------------------------------------
constexpr int kStatsThreads = 256;

// RAG (ragged batches): image n = blockIdx.z takes its pointer and geometry from imgs[n]; the grid is sized for the
// image with the most slabs, and the surplus slabs of the others exit
template <bool RAG = false>
__global__ void __launch_bounds__(kStatsThreads)
stats_kernel(const uint8_t* __restrict__ rgb, int H, int W, int th, int tw, int rows_per_slab,
             const Tables* __restrict__ tables, uint32_t* __restrict__ tile_hist,
             uint32_t* __restrict__ rgb_hist, const RaggedImage* __restrict__ imgs) {
  __shared__ uint32_t s_hist[4][256];  // 0: L of this tile, 1..3: R, G, B
  __shared__ uint16_t s_gtab[256];
  __shared__ uint16_t s_ctab[3072];
  if constexpr (RAG) {
    const RaggedImage im = imgs[blockIdx.z];
    if ((int)blockIdx.y >= im.slabs) return;
    rgb = im.rgb;
    H = im.H;
    W = im.W;
    th = im.th;
    tw = im.tw;
    rows_per_slab = im.rows_per_slab;
  }
  const int tid = threadIdx.x;
  for (int i = tid; i < 1024; i += kStatsThreads) (&s_hist[0][0])[i] = 0;
  for (int i = tid; i < 256; i += kStatsThreads) s_gtab[i] = tables->gtab[i];
  for (int i = tid; i < 3072; i += kStatsThreads) s_ctab[i] = tables->ctab[i];
  __syncthreads();

  const int tile = blockIdx.x, ty = tile >> 3, tx = tile & 7;
  const int n = blockIdx.z;
  const int r0 = blockIdx.y * rows_per_slab;
  const int r1 = min(r0 + rows_per_slab, th);
  const uint8_t* img = RAG ? rgb : rgb + (size_t)n * H * W * 3;
  const int count = (r1 - r0) * tw;
  for (int i = tid; i < count; i += kStatsThreads) {
    int rr = i / tw;
    int cc = i - rr * tw;
    int py = ty * th + r0 + rr, px = tx * tw + cc;  // padded-image coordinates
    int sy = reflect101(py, H), sx = reflect101(px, W);
    const uint8_t* p = img + ((size_t)sy * W + sx) * 3;
    int r = p[0], g = p[1], b = p[2];
    atomicAdd(&s_hist[0][lab_L(s_gtab, s_ctab, r, g, b)], 1u);
    if (py < H && px < W) {  // every real pixel lies in exactly one tile
      atomicAdd(&s_hist[1][r], 1u);
      atomicAdd(&s_hist[2][g], 1u);
      atomicAdd(&s_hist[3][b], 1u);
    }
  }
  __syncthreads();
  uint32_t* th_out = tile_hist + ((size_t)n * 64 + tile) * 256;
  uint32_t* rgb_out = rgb_hist + (size_t)n * 768;
  for (int i = tid; i < 256; i += kStatsThreads) {
    uint32_t v = s_hist[0][i];
    if (v) atomicAdd(&th_out[i], v);
  }
  for (int i = tid; i < 768; i += kStatsThreads) {
    uint32_t v = (&s_hist[1][0])[i];
    if (v) atomicAdd(&rgb_out[i], v);
  }
}

// ---------------------------------------------------------------------------
// Pass 2: LUTs.  grid = (65, N), 256 threads: blocks 0..63 CLAHE tiles, 64 = WB.
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t block_inclusive_scan_256(uint32_t v, uint32_t* s_warp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  if (lane == 31) s_warp[warp] = v;
  __syncthreads();
  uint32_t add = 0;
  for (int wi = 0; wi < warp; wi++) add += s_warp[wi];
  __syncthreads();
  return v + add;
}

// numpy's np.quantile(..., method="linear") on the sorted multiset described by an
// inclusive cumulative histogram; `n` elements.  Mirrors numpy/lib/_function_base_impl.py
// (_compute_virtual_index, _get_indexes, _lerp) operation for operation in float64.
__device__ double np_quantile_from_cum(const uint32_t* cum, int n, double q) {
  double vi = __dmul_rn((double)(n - 1), q);  // method "linear": virtual index = (n - 1) * q
  double prev_f = floor(vi);
  long long prev = (long long)prev_f, next = prev + 1;
  if (vi >= (double)(n - 1)) prev = next = n - 1;
  if (vi < 0.0) prev = next = 0;
  if (prev < 0) prev = 0;
  if (next > n - 1) next = n - 1;
  double gamma = __dsub_rn(vi, prev_f);
  int a = 0, b = 0;
  for (int u = 0; u < 256; u++) {
    if (cum[u] > (uint32_t)prev) { a = u; break; }
  }
  for (int u = a; u < 256; u++) {
    if (cum[u] > (uint32_t)next) { b = u; break; }
  }
  double da = (double)a, db = (double)b, diff = __dsub_rn(db, da);
  double res = __dadd_rn(da, __dmul_rn(diff, gamma));
  if (gamma >= 0.5) res = __dsub_rn(db, __dmul_rn(diff, __dsub_rn(1.0, gamma)));
  return res;
}

// RAG: image n = blockIdx.y takes its pixel count, clip limit and LUT scale from imgs[n]
template <bool RAG = false>
__global__ void __launch_bounds__(256)
luts_kernel(const uint32_t* __restrict__ tile_hist, const uint32_t* __restrict__ rgb_hist,
            int npix, int clip, float lut_scale, uint8_t* __restrict__ clahe_lut,
            uint8_t* __restrict__ wb_lut, int gray, const RaggedImage* __restrict__ imgs) {
  __shared__ uint32_t s_warp[8];
  __shared__ uint32_t s_cum[3][256];
  __shared__ unsigned long long s_sum[3];
  __shared__ uint32_t s_red;
  const int tid = threadIdx.x, n = blockIdx.y;
  if constexpr (RAG) {
    npix = imgs[n].H * imgs[n].W;
    clip = imgs[n].clip;
    lut_scale = imgs[n].lut_scale;
  }
  if (blockIdx.x < 64) {
    // OpenCV CLAHE_CalcLut_Body: clip, redistribute the excess, prefix-sum, scale.
    const int tile = blockIdx.x;
    int hv = (int)tile_hist[((size_t)n * 64 + tile) * 256 + tid];
    if (tid == 0) s_red = 0;
    __syncthreads();
    int over = max(hv - clip, 0);
    if (over) atomicAdd(&s_red, (uint32_t)over);
    __syncthreads();
    int excess = (int)s_red;
    hv = min(hv, clip);
    int batch = excess / 256;
    int residual = excess - batch * 256;
    hv += batch;
    if (residual != 0) {
      int step = max(256 / residual, 1);
      if (tid % step == 0 && tid / step < residual) hv += 1;
    }
    uint32_t cum = block_inclusive_scan_256((uint32_t)hv, s_warp);
    float f = rintf(__fmul_rn((float)cum, lut_scale));
    clahe_lut[((size_t)n * 64 + tile) * 256 + tid] = (uint8_t)fminf(fmaxf(f, 0.f), 255.f);
    return;
  }
  // White balance LUT: data.py:15-23 (saturation levels), :38-48 (quantiles, stretch).
  const uint32_t* hist = rgb_hist + (size_t)n * 768;
  if (tid < 3) s_sum[tid] = 0ull;
  __syncthreads();
  for (int c = 0; c < 3; c++) {
    uint32_t hv = hist[c * 256 + tid];
    atomicAdd(&s_sum[c], (unsigned long long)hv * (unsigned long long)tid);
    uint32_t cum = block_inclusive_scan_256(hv, s_warp);
    s_cum[c][tid] = cum;
  }
  __syncthreads();
  __shared__ double s_q[3][2];
  if (tid < 3) {
    const int c = tid;
    unsigned long long mx = max(s_sum[0], max(s_sum[1], s_sum[2]));
    double lo = 0.0, hi = 255.0;
    if (gray) {
      // grayscale branch (data.py:30-36): fixed saturation levels 0.001 / 0.005, no channel ratios; its flat array
      // stays uint8, so the clipping assignments (data.py:43-44) store the TRUNCATED quantiles
      lo = floor(np_quantile_from_cum(s_cum[c], npix, 0.001));
      hi = floor(np_quantile_from_cum(s_cum[c], npix, __dsub_rn(1.0, 0.005)));
    } else if (s_sum[c] != 0ull) {
      double ratio = __ddiv_rn((double)mx, (double)s_sum[c]);
      double sat = __dmul_rn(0.005, ratio);
      double qlo = sat, qhi = __dsub_rn(1.0, sat);
      if (qlo >= 0.0 && qlo <= 1.0 && qhi >= 0.0 && qhi <= 1.0) {
        lo = np_quantile_from_cum(s_cum[c], npix, qlo);
        hi = np_quantile_from_cum(s_cum[c], npix, qhi);
      }
    }
    s_q[c][0] = lo;
    s_q[c][1] = hi;
  }
  __syncthreads();
  for (int c = 0; c < 3; c++) {
    double lo = s_q[c][0], hi = s_q[c][1];
    double v = fmin(fmax((double)tid, lo), hi);
    double span = __dsub_rn(hi, lo);
    double o = 0.0;
    if (span > 0.0) o = __ddiv_rn(__dmul_rn(__dsub_rn(v, lo), 255.0), span);
    int oi = (int)o;  // astype(uint8): truncate
    wb_lut[(size_t)n * 768 + c * 256 + tid] = (uint8_t)min(max(oi, 0), 255);
  }
}

// ---------------------------------------------------------------------------
// Pass 3: per-pixel apply.  grid = (ceil(H*W/256), N), 256 threads.
// ---------------------------------------------------------------------------
// pixels per CTA = 256 * iters (x 4 in the vector path): amortises the ~30 KB of LUT/table staging per CTA.  16 for big
// launches; fewer when the launch is small (one pass of 4 images), so that the grid still has ~8 CTAs per SM and the
// single wave is balanced
constexpr int kApplyItersMax = 16;
static int apply_iters(long long pixels_per_thread_slot, int sm_count) {
  long long it = pixels_per_thread_slot / (256ll * 8 * sm_count);
  return it < 4 ? 4 : it > kApplyItersMax ? kApplyItersMax : (int)it;
}

struct ApplyOut {
  float* f32[4];    // x, wb, he, gc  -- NCHW planes, may be null
  uint8_t* u8[3];   // wb, he, gc     -- NHWC, may be null
  uint4* planes;    // may be null: [n][2][H*W] x 16 B, the first conv layer's operand planes (8 bf16 levels each):
                    // torch.cat([x, wb, he, gc], 1) (net.py:46) as plane 0 = x.rgb wb.rgb he.rg, plane 1 = he.b gc.rgb 0 0 0 0
};
// bf16 bit patterns of two integer levels 0..255 (exact: 8 significant bits), first level in the low half
__device__ __forceinline__ uint32_t bf16_levels2(int a, int b) {
  return (__float_as_uint((float)a) >> 16) | (__float_as_uint((float)b) & 0xffff0000u);
}
__device__ __forceinline__ void store_level_planes(uint4* planes, size_t n, size_t plane, size_t pix, const int* lv) {
  uint4* p = planes + n * 2 * plane + pix;
  p[0] = make_uint4(bf16_levels2(lv[0], lv[1]), bf16_levels2(lv[2], lv[3]), bf16_levels2(lv[4], lv[5]),
                    bf16_levels2(lv[6], lv[7]));
  p[plane] = make_uint4(bf16_levels2(lv[8], lv[9]), bf16_levels2(lv[10], lv[11]), 0u, 0u);
}

// The image data of slot image `img`: one record for every image of a grid call (image i at rgb + i * H * W * 3), or
// the ragged call's device table
__device__ __forceinline__ RaggedImage slot_image(const RaggedImage& one, int img) {
  RaggedImage r = one;
  r.rgb += (size_t)img * one.H * one.W * 3;
  return r;
}
__device__ __forceinline__ RaggedImage slot_image(const RaggedImage* imgs, int img) { return imgs[img]; }

// Whole images (Geom = WholeImages): blockIdx.y is image blockIdx.y of rgb, H x W; the kernel writes any of `out`.
// The slot form (Geom = GridGeom or TableGeom, tiling.cuh): blockIdx.y is slot blockIdx.y of geo, whose pixels take
// their image and coordinates from geo.at and their image data from slot_image(imgs, ...); the kernel writes that
// slot's operand planes (out.planes only), zeros beyond its valid extent, interpolating the CLAHE tiles at image
// coordinates.
struct WholeImages {};
template <bool VEC4, class Geom = WholeImages, class Img = WholeImages>
__global__ void __launch_bounds__(256)
apply_kernel(const uint8_t* __restrict__ rgb, int H, int W, int th, int tw,
             const Tables* __restrict__ tables, const uint8_t* __restrict__ clahe_lut,
             const uint8_t* __restrict__ wb_lut, ApplyOut out, int iters, Geom geo, Img imgs) {
  constexpr bool SLOT = !std::is_same<Geom, WholeImages>::value;
  static_assert(!(VEC4 && SLOT), "the slot form has no vector path");
  __shared__ __align__(16) uint8_t s_clahe[64 * 256];
  __shared__ __align__(16) uint8_t s_wb[768];
  __shared__ __align__(16) uint8_t s_gamma[256];
  __shared__ __align__(16) uint8_t s_igtab[4096];
  __shared__ uint16_t s_gtab[256];
  __shared__ uint16_t s_ctab[3072];
  __shared__ int16_t s_ytab[256];
  __shared__ int16_t s_fytab[256];
  __shared__ float s_div[256];
  int n = blockIdx.y;
  if constexpr (SLOT) {
    n = geo.at(blockIdx.y, 0).img;
    const RaggedImage im = slot_image(imgs, n);
    rgb = im.rgb;
    H = im.H;
    W = im.W;
    th = im.th;
    tw = im.tw;
  }
  const int tid = threadIdx.x;
  // a slot's image index comes from memory: as unsigned, its LUT offset needs no sign extension (which ptxas spills)
  const size_t lut = SLOT ? (size_t)(unsigned)n : (size_t)n;
  {
    const uint4* src = reinterpret_cast<const uint4*>(clahe_lut + lut * 64 * 256);
    uint4* dst = reinterpret_cast<uint4*>(s_clahe);
    for (int i = tid; i < 1024; i += 256) dst[i] = src[i];
    const uint32_t* wsrc = reinterpret_cast<const uint32_t*>(wb_lut + lut * 768);
    for (int i = tid; i < 192; i += 256) reinterpret_cast<uint32_t*>(s_wb)[i] = wsrc[i];
    const uint4* isrc = reinterpret_cast<const uint4*>(tables->igtab);
    for (int i = tid; i < 256; i += 256) reinterpret_cast<uint4*>(s_igtab)[i] = isrc[i];
    s_gamma[tid] = tables->gamma[tid];
    s_gtab[tid] = tables->gtab[tid];
    s_ytab[tid] = tables->ytab[tid];
    s_fytab[tid] = tables->fytab[tid];
    s_div[tid] = tables->div255[tid];
    for (int i = tid; i < 3072; i += 256) s_ctab[i] = tables->ctab[i];
  }
  __syncthreads();
  const int plane = H * W;
  const float inv_tw = __fdiv_rn(1.0f, (float)tw), inv_th = __fdiv_rn(1.0f, (float)th);

  // one pixel: levels of the raw, white-balanced, hist-equalised and gamma-corrected images
  auto one_pixel = [&](int pix, int r, int g, int b, int* lv /* [4][3] */) {
    const int y = pix / W, x = pix - y * W;
    // hist-eq: RGB -> Lab, CLAHE bilinear blend of the four neighbouring tile LUTs, Lab -> RGB
    int L, A, Bv;
    rgb2lab(s_gtab, s_ctab, r, g, b, L, A, Bv);
    float txf = __fsub_rn(__fmul_rn((float)x, inv_tw), 0.5f);
    float tyf = __fsub_rn(__fmul_rn((float)y, inv_th), 0.5f);
    int tx1 = (int)floorf(txf), ty1 = (int)floorf(tyf);
    float xa = __fsub_rn(txf, (float)tx1), ya = __fsub_rn(tyf, (float)ty1);
    float xa1 = __fsub_rn(1.0f, xa), ya1 = __fsub_rn(1.0f, ya);
    int tx2 = min(tx1 + 1, 7), ty2 = min(ty1 + 1, 7);
    tx1 = max(tx1, 0);
    ty1 = max(ty1, 0);
    float l11 = (float)s_clahe[(ty1 * 8 + tx1) * 256 + L];
    float l12 = (float)s_clahe[(ty1 * 8 + tx2) * 256 + L];
    float l21 = (float)s_clahe[(ty2 * 8 + tx1) * 256 + L];
    float l22 = (float)s_clahe[(ty2 * 8 + tx2) * 256 + L];
    float top = __fadd_rn(__fmul_rn(l11, xa1), __fmul_rn(l12, xa));
    float bot = __fadd_rn(__fmul_rn(l21, xa1), __fmul_rn(l22, xa));
    float res = __fadd_rn(__fmul_rn(top, ya1), __fmul_rn(bot, ya));
    int Leq = (int)fminf(fmaxf(rintf(res), 0.f), 255.f);
    lv[0] = r; lv[1] = g; lv[2] = b;
    lv[3] = s_wb[r]; lv[4] = s_wb[256 + g]; lv[5] = s_wb[512 + b];
    lab2rgb(s_ytab, s_fytab, s_igtab, Leq, A, Bv, lv[6], lv[7], lv[8]);
    lv[9] = s_gamma[r]; lv[10] = s_gamma[g]; lv[11] = s_gamma[b];
  };

  if constexpr (VEC4) {
    // four consecutive pixels per thread: 12 input bytes as three 32-bit loads, one float4 store per plane
    for (int it = 0; it < iters; it++) {
      const int pix = ((blockIdx.x * iters + it) * 256 + tid) * 4;
      if (pix >= plane) break;
      const uint32_t* p32 = reinterpret_cast<const uint32_t*>(rgb + ((size_t)n * plane + pix) * 3);
      const uint32_t w0 = p32[0], w1 = p32[1], w2 = p32[2];
      const int px[4][3] = {{(int)(w0 & 255), (int)((w0 >> 8) & 255), (int)((w0 >> 16) & 255)},
                            {(int)(w0 >> 24), (int)(w1 & 255), (int)((w1 >> 8) & 255)},
                            {(int)((w1 >> 16) & 255), (int)(w1 >> 24), (int)(w2 & 255)},
                            {(int)((w2 >> 8) & 255), (int)((w2 >> 16) & 255), (int)(w2 >> 24)}};
      int lv[4][12];
#pragma unroll
      for (int k = 0; k < 4; k++) one_pixel(pix + k, px[k][0], px[k][1], px[k][2], lv[k]);
      const size_t o = (size_t)n * 3 * plane + pix;
#pragma unroll
      for (int t = 0; t < 4; t++) {
        if (!out.f32[t]) continue;
#pragma unroll
        for (int c = 0; c < 3; c++)
          *reinterpret_cast<float4*>(out.f32[t] + o + (size_t)c * plane) =
              make_float4(s_div[lv[0][t * 3 + c]], s_div[lv[1][t * 3 + c]], s_div[lv[2][t * 3 + c]], s_div[lv[3][t * 3 + c]]);
      }
      if (out.planes) {
#pragma unroll
        for (int k = 0; k < 4; k++) store_level_planes(out.planes, n, plane, pix + k, lv[k]);
      }
      const size_t o8 = ((size_t)n * plane + pix) * 3;
#pragma unroll
      for (int t = 0; t < 3; t++) {
        if (!out.u8[t]) continue;
        uint32_t* q = reinterpret_cast<uint32_t*>(out.u8[t] + o8);
        const int* a0 = lv[0] + (t + 1) * 3; const int* a1 = lv[1] + (t + 1) * 3;
        const int* a2 = lv[2] + (t + 1) * 3; const int* a3 = lv[3] + (t + 1) * 3;
        q[0] = (uint32_t)a0[0] | ((uint32_t)a0[1] << 8) | ((uint32_t)a0[2] << 16) | ((uint32_t)a1[0] << 24);
        q[1] = (uint32_t)a1[1] | ((uint32_t)a1[2] << 8) | ((uint32_t)a2[0] << 16) | ((uint32_t)a2[1] << 24);
        q[2] = (uint32_t)a2[2] | ((uint32_t)a3[0] << 8) | ((uint32_t)a3[1] << 16) | ((uint32_t)a3[2] << 24);
      }
    }
  } else if constexpr (SLOT) {
    // planes [slot][2][slot pixels]
    const int wplane = geo.slot_hw();
    for (int it = 0; it < iters; it++) {
      const int pix = (blockIdx.x * iters + it) * 256 + tid;
      if (pix >= wplane) break;
      const SlotPixel p = geo.at(blockIdx.y, pix);
      int lv[12] = {};  // zero operands beyond the valid extent: what the tiled call's TMA reads beyond its window
      if (p.valid) {
        const uint8_t* q = rgb + p.o * 3;
        one_pixel((int)p.o, q[0], q[1], q[2], lv);
      }
      store_level_planes(out.planes, blockIdx.y, wplane, pix, lv);
    }
  } else {
    for (int it = 0; it < iters; it++) {
      const int pix = (blockIdx.x * iters + it) * 256 + tid;
      if (pix >= plane) break;
      const uint8_t* p = rgb + ((size_t)n * plane + pix) * 3;
      int lv[12];
      one_pixel(pix, p[0], p[1], p[2], lv);
      const size_t o = (size_t)n * 3 * plane + pix;
#pragma unroll
      for (int t = 0; t < 4; t++) {
        if (!out.f32[t]) continue;
        float* q = out.f32[t] + o;
        q[0] = s_div[lv[t * 3]]; q[plane] = s_div[lv[t * 3 + 1]]; q[2 * (size_t)plane] = s_div[lv[t * 3 + 2]];
      }
      if (out.planes) store_level_planes(out.planes, n, plane, pix, lv);
      const size_t o8 = ((size_t)n * plane + pix) * 3;
#pragma unroll
      for (int t = 0; t < 3; t++) {
        if (!out.u8[t]) continue;
        uint8_t* q = out.u8[t] + o8;
        q[0] = lv[(t + 1) * 3]; q[1] = lv[(t + 1) * 3 + 1]; q[2] = lv[(t + 1) * 3 + 2];
      }
    }
  }
}

// ---------------------------------------------------------------------------
// ten2arr: clip(0,1) * 255 -> truncate, NCHW -> NHWC (hubconf.py:24-34)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
postprocess_kernel(const float* __restrict__ in, uint8_t* __restrict__ out, int plane) {
  const int n = blockIdx.y;
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= plane) return;
  const float* q = in + (size_t)n * 3 * plane + pix;
  uint8_t* o = out + ((size_t)n * plane + pix) * 3;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    float v = fminf(fmaxf(q[(size_t)c * plane], 0.0f), 1.0f);
    o[c] = (uint8_t)(int)__fmul_rn(v, 255.0f);
  }
}

// ---------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------
struct PreGeom {
  int hp, wp, th, tw, clip;
  float lut_scale;
};

static PreGeom geometry(int H, int W) {
  PreGeom g;
  if (H % 8 == 0 && W % 8 == 0) {
    g.hp = H;
    g.wp = W;
  } else {  // cv::copyMakeBorder(0, 8 - H%8, 0, 8 - W%8): a full 8 on an already divisible side
    g.hp = H + (8 - H % 8);
    g.wp = W + (8 - W % 8);
  }
  g.th = g.hp / 8;
  g.tw = g.wp / 8;
  int area = g.th * g.tw;
  int clip = (int)(0.1 * area / 256);  // createCLAHE(clipLimit=0.1): data.py:71
  g.clip = clip < 1 ? 1 : clip;
  g.lut_scale = 255.0f / (float)area;
  return g;
}

// workspace: [tile_hist N*64*256 u32][rgb_hist N*768 u32][clahe_lut N*64*256 u8][wb_lut N*768 u8]
size_t preprocess_workspace_bytes(int n, int, int) {
  size_t b = 0;
  b += align256((size_t)n * 64 * 256 * 4);
  b += align256((size_t)n * 768 * 4);
  b += align256((size_t)n * 64 * 256);
  b += align256((size_t)n * 768);
  return b;
}

static int preprocess_run(wn_handle* h, const uint8_t* rgb, int n, int H, int W, float* x, float* wb,
                          float* he, float* gc, uint8_t* wb_u8, uint8_t* he_u8, uint8_t* gc_u8, uint4* planes,
                          void* workspace, size_t workspace_bytes, cudaStream_t stream, int gray = 0);

// grayscale branch of white_balance_transform (data.py:30-36, 38-58 with p = 1): the 2-D image runs through the RGB
// machinery as r = g = b with the branch's fixed saturation levels; channel 0 of the result is the answer
__global__ void gray_expand_kernel(const uint8_t* __restrict__ g, uint8_t* __restrict__ rgb, size_t npix) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) {
    const uint8_t v = g[i];
    rgb[3 * i] = v; rgb[3 * i + 1] = v; rgb[3 * i + 2] = v;
  }
}
__global__ void gray_extract_kernel(const uint8_t* __restrict__ rgb, uint8_t* __restrict__ g, size_t npix) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) g[i] = rgb[3 * i];
}
size_t white_balance_gray_workspace_bytes(int n, int h, int w) {
  return align256(preprocess_workspace_bytes(n, h, w)) + 2 * align256((size_t)n * h * w * 3);
}
int white_balance_gray_u8(wn_handle* h, const uint8_t* gray, uint8_t* out, int n, int H, int W, void* workspace,
                          size_t workspace_bytes, cudaStream_t stream) {
  if (workspace_bytes < white_balance_gray_workspace_bytes(n, H, W)) {
    set_error("white balance (gray) workspace too small");
    return WN_E_WORKSPACE;
  }
  uint8_t* ws = (uint8_t*)workspace;
  const size_t pre_b = align256(preprocess_workspace_bytes(n, H, W)), img_b = align256((size_t)n * H * W * 3);
  uint8_t* rgb = ws + pre_b;
  uint8_t* wb = rgb + img_b;
  const size_t npix = (size_t)n * H * W;
  gray_expand_kernel<<<1024, 256, 0, stream>>>(gray, rgb, npix);
  WN_LAUNCH_CHECK(h);
  int rc = preprocess_run(h, rgb, n, H, W, nullptr, nullptr, nullptr, nullptr, wb, nullptr, nullptr, nullptr, ws, pre_b, stream, 1);
  if (rc) return rc;
  gray_extract_kernel<<<1024, 256, 0, stream>>>(wb, out, npix);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

int preprocess_u8(wn_handle* h, const uint8_t* rgb, int n, int H, int W, float* x, float* wb,
                  float* he, float* gc, uint8_t* wb_u8, uint8_t* he_u8, uint8_t* gc_u8,
                  void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return preprocess_run(h, rgb, n, H, W, x, wb, he, gc, wb_u8, he_u8, gc_u8, nullptr, workspace, workspace_bytes,
                        stream);
}

int preprocess_u8_planes(wn_handle* h, const uint8_t* rgb, int n, int H, int W, uint4* planes, void* workspace,
                         size_t workspace_bytes, cudaStream_t stream) {
  return preprocess_run(h, rgb, n, H, W, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, planes,
                        workspace, workspace_bytes, stream, 0);
}

struct PreBufs {
  uint32_t* tile_hist;
  uint32_t* rgb_hist;
  uint8_t* clahe_lut;
  uint8_t* wb_lut;
};
static PreBufs pre_carve(void* workspace, int n) {
  PreBufs b;
  uint8_t* ws = (uint8_t*)workspace;
  b.tile_hist = (uint32_t*)ws;
  ws += align256((size_t)n * 64 * 256 * 4);
  b.rgb_hist = (uint32_t*)ws;
  ws += align256((size_t)n * 768 * 4);
  b.clahe_lut = ws;
  ws += align256((size_t)n * 64 * 256);
  b.wb_lut = ws;
  return b;
}

static int preprocess_check(int n, int H, int W, size_t workspace_bytes) {
  if (workspace_bytes < preprocess_workspace_bytes(n, H, W)) {
    set_error("preprocess workspace too small: %zu < %zu", workspace_bytes,
              preprocess_workspace_bytes(n, H, W));
    return WN_E_WORKSPACE;
  }
  if ((size_t)H * W > (size_t)0x7fffffff / 3 || n > 65535) {
    set_error("image too large: n=%d h=%d w=%d", n, H, W);
    return WN_E_UNSUPPORTED;
  }
  return WN_OK;
}

// passes 1 and 2: per-image histograms -> CLAHE and white-balance LUTs in the workspace
static int preprocess_luts(wn_handle* h, const uint8_t* rgb, int n, int H, int W, const PreGeom& g, const PreBufs& b,
                           cudaStream_t stream, int gray) {
  uint32_t* tile_hist = b.tile_hist;
  uint32_t* rgb_hist = b.rgb_hist;
  size_t hist_bytes = align256((size_t)n * 64 * 256 * 4) + (size_t)n * 768 * 4;
  WN_CUDA(cudaMemsetAsync(tile_hist, 0, hist_bytes, stream));
  // ~4K pixels per CTA keeps the grid well above two CTAs per SM even for one 1080p image
  int slabs = (g.th * g.tw + 4095) / 4096;
  if (slabs > g.th) slabs = g.th;
  if (slabs < 1) slabs = 1;
  int rows_per_slab = (g.th + slabs - 1) / slabs;
  slabs = (g.th + rows_per_slab - 1) / rows_per_slab;
  {
  TimedScope ts(h, kSlotStats, stream);
  stats_kernel<<<dim3(64, slabs, n), kStatsThreads, 0, stream>>>(rgb, H, W, g.th, g.tw,
                                                                  rows_per_slab, h->d_tables,
                                                                  tile_hist, rgb_hist, nullptr);
  WN_LAUNCH_CHECK(h);
  }
  {
  TimedScope ts(h, kSlotLuts, stream);
  luts_kernel<<<dim3(65, n), 256, 0, stream>>>(tile_hist, rgb_hist, H * W, g.clip, g.lut_scale,
                                               b.clahe_lut, b.wb_lut, gray, nullptr);
  WN_LAUNCH_CHECK(h);
  }
  return WN_OK;
}

static int preprocess_run(wn_handle* h, const uint8_t* rgb, int n, int H, int W, float* x, float* wb,
                          float* he, float* gc, uint8_t* wb_u8, uint8_t* he_u8, uint8_t* gc_u8, uint4* planes,
                          void* workspace, size_t workspace_bytes, cudaStream_t stream, int gray) {
  int rc = preprocess_check(n, H, W, workspace_bytes);
  if (rc) return rc;
  PreGeom g = geometry(H, W);
  const PreBufs b = pre_carve(workspace, n);
  rc = preprocess_luts(h, rgb, n, H, W, g, b, stream, gray);
  if (rc) return rc;
  const uint8_t* clahe_lut = b.clahe_lut;
  const uint8_t* wb_lut = b.wb_lut;
  ApplyOut ao;
  ao.f32[0] = x; ao.f32[1] = wb; ao.f32[2] = he; ao.f32[3] = gc;
  ao.u8[0] = wb_u8; ao.u8[1] = he_u8; ao.u8[2] = gc_u8;
  ao.planes = planes;
  TimedScope ts(h, kSlotApply, stream);
  // vector path: 4 pixels per thread needs 4-pixel groups that do not straddle images (and aligned bases)
  const bool vec4 = (H * W) % 4 == 0 && ((uintptr_t)rgb % 4) == 0 && ((uintptr_t)x % 16) == 0 &&
                    ((uintptr_t)wb % 16) == 0 && ((uintptr_t)he % 16) == 0 && ((uintptr_t)gc % 16) == 0 &&
                    ((uintptr_t)wb_u8 % 4) == 0 && ((uintptr_t)he_u8 % 4) == 0 && ((uintptr_t)gc_u8 % 4) == 0;
  if (vec4) {
    const int iters = apply_iters((long long)n * H * W / 4, h->sm_count);
    const int per_cta = 256 * iters * 4;
    apply_kernel<true><<<dim3((H * W + per_cta - 1) / per_cta, n), 256, 0, stream>>>(rgb, H, W, g.th, g.tw, h->d_tables,
                                                                                   clahe_lut, wb_lut, ao, iters,
                                                                                   WholeImages(), WholeImages());
  } else {
    const int iters = apply_iters((long long)n * H * W, h->sm_count);
    const int per_cta = 256 * iters;
    apply_kernel<false><<<dim3((H * W + per_cta - 1) / per_cta, n), 256, 0, stream>>>(rgb, H, W, g.th, g.tw, h->d_tables,
                                                                                    clahe_lut, wb_lut, ao, iters,
                                                                                    WholeImages(), WholeImages());
  }
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

int preprocess_u8_luts(wn_handle* h, const uint8_t* rgb, int n, int H, int W, void* workspace, size_t workspace_bytes,
                       cudaStream_t stream) {
  const int rc = preprocess_check(n, H, W, workspace_bytes);
  if (rc) return rc;
  return preprocess_luts(h, rgb, n, H, W, geometry(H, W), pre_carve(workspace, n), stream, 0);
}

// the stats grid of one image, as preprocess_luts sizes it
RaggedImage ragged_image(const uint8_t* rgb, int H, int W) {
  const PreGeom g = geometry(H, W);
  RaggedImage r;
  r.rgb = rgb;
  r.H = H;
  r.W = W;
  r.th = g.th;
  r.tw = g.tw;
  r.clip = g.clip;
  r.lut_scale = g.lut_scale;
  int slabs = (g.th * g.tw + 4095) / 4096;
  if (slabs > g.th) slabs = g.th;
  if (slabs < 1) slabs = 1;
  r.rows_per_slab = (g.th + slabs - 1) / slabs;
  r.slabs = (g.th + r.rows_per_slab - 1) / r.rows_per_slab;
  return r;
}

int preprocess_u8_ragged_luts(wn_handle* h, int n, const RaggedImage* imgs, int max_slabs, void* workspace,
                              cudaStream_t stream) {
  const PreBufs b = pre_carve(workspace, n);
  WN_CUDA(cudaMemsetAsync(b.tile_hist, 0, align256((size_t)n * 64 * 256 * 4) + (size_t)n * 768 * 4, stream));
  {
  TimedScope ts(h, kSlotStats, stream);
  stats_kernel<true><<<dim3(64, max_slabs, n), kStatsThreads, 0, stream>>>(nullptr, 0, 0, 0, 0, 0, h->d_tables,
                                                                          b.tile_hist, b.rgb_hist, imgs);
  WN_LAUNCH_CHECK(h);
  }
  TimedScope ts(h, kSlotLuts, stream);
  luts_kernel<true><<<dim3(65, n), 256, 0, stream>>>(b.tile_hist, b.rgb_hist, 0, 0, 0.f, b.clahe_lut, b.wb_lut, 0,
                                                     imgs);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

template <class Geom, class Img>
int preprocess_u8_slot_planes(wn_handle* h, const Geom& geo, const Img& imgs, int n, int count, uint4* planes,
                              void* workspace, cudaStream_t stream) {
  const PreBufs b = pre_carve(workspace, n);
  ApplyOut ao;
  memset(&ao, 0, sizeof(ao));
  ao.planes = planes;
  TimedScope ts(h, kSlotApply, stream);
  const int wplane = geo.slot_hw();
  const int iters = apply_iters((long long)count * wplane, h->sm_count);
  const int per_cta = 256 * iters;
  apply_kernel<false><<<dim3((wplane + per_cta - 1) / per_cta, count), 256, 0, stream>>>(
      nullptr, 0, 0, 0, 0, h->d_tables, b.clahe_lut, b.wb_lut, ao, iters, geo, imgs);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}
template int preprocess_u8_slot_planes(wn_handle*, const GridGeom&, const RaggedImage&, int, int, uint4*, void*,
                                       cudaStream_t);
template int preprocess_u8_slot_planes(wn_handle*, const TableGeom&, const RaggedImage* const&, int, int, uint4*,
                                       void*, cudaStream_t);

// ---------------------------------------------------------------------------
// cv2.resize(img, (w, h)) of 8-bit images, default INTER_LINEAR (training_utils.py:94-103), batched: every source
// image has its own size, all land in one (N, dh, dw, 3) batch.  OpenCV imgproc/src/resize.cpp arithmetic, bit
// exact (oracle/preprocess.py::resize_linear_u8 is the CPU restatement):
//   fx = (float)((dx + 0.5) * scale - 0.5), scale = 1 / ((double)dsize / ssize); sx = floor(fx); fx -= sx;
//   x: an index outside [0, ssize-1) is clamped with weights (1, 0); y: only the row index is clamped;
//   weights = saturate_cast<short>(w * 2048) (round half to even); horizontal pass in int32,
//   vertical pass (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2;
//   an exact 2x reduction in both directions is INTER_AREA ((a + b + c + d + 2) >> 2); equal sizes copy.
// swap_rb folds the BGR -> RGB conversion that follows the resize in the reference (a per-channel permutation
// commutes with a per-channel resize).
// ---------------------------------------------------------------------------
constexpr int kResizeGroup = 96;
struct ResizeBatch {
  const uint8_t* src[kResizeGroup];
  int h[kResizeGroup], w[kResizeGroup];
};
__device__ __forceinline__ void resize_coeff(int d, int ssize, int dsize, bool clamp, int& idx, int& w0, int& w1) {
  const double scale = __ddiv_rn(1.0, __ddiv_rn((double)dsize, (double)ssize));
  float f = (float)__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5);
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (clamp) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= ssize - 1) { f = 0.f; s = ssize - 1; }
  }
  idx = s;
  w0 = (int)rintf(__fmul_rn(__fsub_rn(1.0f, f), 2048.0f));
  w1 = (int)rintf(__fmul_rn(f, 2048.0f));
}
__global__ void __launch_bounds__(256)
resize_linear_u8_kernel(const ResizeBatch batch, uint8_t* __restrict__ dst, int dh, int dw, int swap_rb, int n0) {
  const int i = blockIdx.y;
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= dh * dw) return;
  const int dy = pix / dw, dx = pix - dy * dw;
  const uint8_t* __restrict__ src = batch.src[i];
  const int sh = batch.h[i], sw = batch.w[i];
  uint8_t* o = dst + ((size_t)(n0 + i) * dh * dw + pix) * 3;
  int v[3];
  if (sh == dh && sw == dw) {
    const uint8_t* p = src + (size_t)pix * 3;
    v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
  } else if (sh == 2 * dh && sw == 2 * dw) {
    const uint8_t* p = src + ((size_t)(2 * dy) * sw + 2 * dx) * 3;
    const uint8_t* q = p + (size_t)sw * 3;
#pragma unroll
    for (int c = 0; c < 3; c++) v[c] = ((int)p[c] + p[3 + c] + q[c] + q[3 + c] + 2) >> 2;
  } else {
    int xi, xa0, xa1, yi, yb0, yb1;
    resize_coeff(dx, sw, dw, true, xi, xa0, xa1);
    resize_coeff(dy, sh, dh, false, yi, yb0, yb1);
    const int xi1 = min(xi + 1, sw - 1);
    const int y0 = min(max(yi, 0), sh - 1), y1 = min(max(yi + 1, 0), sh - 1);
    const uint8_t* r0 = src + (size_t)y0 * sw * 3;
    const uint8_t* r1 = src + (size_t)y1 * sw * 3;
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const int s0 = (int)r0[xi * 3 + c] * xa0 + (int)r0[xi1 * 3 + c] * xa1;
      const int s1 = (int)r1[xi * 3 + c] * xa0 + (int)r1[xi1 * 3 + c] * xa1;
      const int t = (((yb0 * (s0 >> 4)) >> 16) + ((yb1 * (s1 >> 4)) >> 16) + 2) >> 2;
      v[c] = min(max(t, 0), 255);
    }
  }
  if (swap_rb) { const int t = v[0]; v[0] = v[2]; v[2] = t; }
  o[0] = (uint8_t)v[0]; o[1] = (uint8_t)v[1]; o[2] = (uint8_t)v[2];
}

int resize_u8(wn_handle* h, const uint8_t* const* src, const int* src_h, const int* src_w, int n, uint8_t* dst,
              int dh, int dw, int swap_rb, cudaStream_t stream) {
  for (int n0 = 0; n0 < n; n0 += kResizeGroup) {
    const int cur = n - n0 < kResizeGroup ? n - n0 : kResizeGroup;
    ResizeBatch b;
    for (int i = 0; i < cur; i++) {
      if (!src[n0 + i] || src_h[n0 + i] <= 0 || src_w[n0 + i] <= 0) {
        set_error("wn_resize_u8: image %d is null or empty", n0 + i);
        return WN_E_INVALID;
      }
      b.src[i] = src[n0 + i]; b.h[i] = src_h[n0 + i]; b.w[i] = src_w[n0 + i];
    }
    resize_linear_u8_kernel<<<dim3((dh * dw + 255) / 256, cur), 256, 0, stream>>>(b, dst, dh, dw, swap_rb, n0);
    WN_LAUNCH_CHECK(h);
  }
  return WN_OK;
}

int postprocess_u8(wn_handle* h, const float* out_nchw, uint8_t* out_nhwc, int n, int H, int W,
                   cudaStream_t stream) {
  TimedScope ts(h, kSlotPost, stream);
  postprocess_kernel<<<dim3((H * W + 255) / 256, n), 256, 0, stream>>>(out_nchw, out_nhwc, H * W);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

}  // namespace wn
