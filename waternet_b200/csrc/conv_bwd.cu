// Backward pass of WaterNet on the tensor cores (SURVEY.md section 8f.1): the training hot loop
// of the reference's train.py:100-133 (loss.backward() through waternet/net.py:99-108).
//
//   seed_kernel          d(out)/d(refined), d(out)/d(cm) and sigmoid'/ReLU' -> gradient planes
//   conv_umma_kernel     data gradient = the forward implicit-GEMM kernel run on flipped,
//   <..., kEpiDgrad>     transposed weights; the epilogue applies ReLU' from the saved activation
//   wgrad_umma_kernel    weight gradient: dW[co][ci][tap] = sum_px g[px][co] * a[px+tap][ci], a
//                        GEMM whose K dimension is PIXELS.  Both operands are read straight from
//                        the activation-plane layout act[plane][y][x][8ch], which is exactly the
//                        no-swizzle MN-major wgmma layout (8 channels contiguous, 16 consecutive
//                        pixels of a row = one K=16 step); a tap is again only a start-address
//                        shift of the B operand.  Every CTA stores its fp32 partial sums; a second kernel adds
//                        them in a fixed order (bit-reproducible gradients, no atomics).
//   bias_grad_kernel     db[co] = sum_px g[px][co]
//
// All three GEMM-shaped pieces use the same bf16x3 split as the forward (gradient error ~1e-5), or, when the handle
// trains in WN_MODE_BF16 (wn_set_train_mode), one bf16 product each: the kFmtHi data gradient, the HI weight gradient
// (g_hi x a_hi) and seeds whose lo planes are 0.
#include <assert.h>

#include "umma_conv.cuh"

namespace wn {

// ------------------------------------------------------------------------------------------
// Weight-gradient kernel
// ------------------------------------------------------------------------------------------
template <int KS, int NCI, int TPG>
struct WgradCfg {
  static constexpr int TX = 16;  // one K=16 step = 16 consecutive pixels of a row
  static constexpr int HALO_W = TX + KS - 1;
  static constexpr int A_PLANES = NCI / 8;
  static constexpr int stage_bytes(int ty) {
    return (2 * 16 * ty * TX * 16 + 2 * A_PLANES * (ty + KS - 1) * HALO_W * 16 + 1023) / 1024 * 1024;
  }
  // two pipeline stages (the TMA of the next tile overlaps the MMAs of this one): 8 rows per tile
  // when that fits in shared memory, else 4
  static constexpr int TY = 2 * stage_bytes(8) + 2048 <= 227 * 1024 ? 8 : 4;
  static constexpr int HALO_H = TY + KS - 1;
  static constexpr int G_PLANE = TY * TX * 16;            // one 8-channel plane of the gradient tile
  static constexpr int G_HALF = 16 * G_PLANE;             // M = 128 output channels = 16 planes
  static constexpr int G_BYTES = 2 * G_HALF;              // hi | lo
  static constexpr int A_PLANE = HALO_W * HALO_H * 16;
  static constexpr int A_HALF = A_PLANES * A_PLANE;
  static constexpr int STAGE = stage_bytes(TY);
  static constexpr int NSTAGE = 2;
  static constexpr int SMEM_BYTES = NSTAGE * STAGE + 1024 + 1024;
  static constexpr int NGROUPS = (KS * KS + TPG - 1) / TPG;
  static constexpr int ACC = TPG * NCI / 2;  // fp32 accumulator registers per thread (M = 64 per warpgroup)
  static_assert(ACC <= 128, "tap group does not fit in registers");
  static_assert(NCI % 16 == 0 && NCI <= 256, "invalid wgmma N");
  static_assert(SMEM_BYTES <= 227 * 1024, "tiles do not fit in shared memory");
};

struct WgradArgs {
  float* partial;  // [CTA = split * NGROUPS + group][TPG][128][NCI] fp32 partial sums (reduced by reduce_wgrad_kernel)
  int N, H, W;
  int co_planes;    // 8-channel planes of the gradient to load (per hi/lo half)
  int planes_half;  // planes per half in the gradient buffer (lo parts start there)
  int co_valid;     // valid output channels
  int tiles_x, tiles_y;
};

constexpr int kWgradThreads = 288;  // warps 0-7: two consumer warpgroups (64 output channels each), 8: TMA producer

// HI: single-pass bf16 (WN_MODE_BF16): only the hi halves are loaded and only g_hi x a_hi is issued
template <int KS, int NCI, int TPG, bool HI = false>
__global__ void __launch_bounds__(kWgradThreads, 1)
wgrad_umma_kernel(const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_a,
                  const WgradArgs g) {
  using C = WgradCfg<KS, NCI, TPG>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  // stage s: [gradient tile hi | lo][activation halo hi | lo]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::NSTAGE * C::STAGE);
  uint64_t* full = bars;                 // [NSTAGE]
  uint64_t* empty = bars + C::NSTAGE;    // [NSTAGE]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int group = blockIdx.x;
  const int num_tiles = g.tiles_x * g.tiles_y * g.N;
  const int my_tiles = num_tiles > (int)blockIdx.y ? (num_tiles - 1 - (int)blockIdx.y) / (int)gridDim.y + 1 : 0;
  if (my_tiles == 0) return;
  const int tap0 = group * TPG;
  const int ntaps = min(TPG, KS * KS - tap0);

  // planes the TMA never writes (output channels beyond co_planes*8) must read as zero
  for (int st = 0; st < C::NSTAGE; st++)
    for (int i = tid; i < C::G_BYTES / 16; i += kWgradThreads)
      reinterpret_cast<uint4*>(smem + st * C::STAGE)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    for (int st = 0; st < C::NSTAGE; st++) { mbar_init(&full[st], 1); mbar_init(&empty[st], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      int st = 0;
      uint32_t phase = 0;
      for (int i = 0; i < my_tiles; i++) {
        const int tile = blockIdx.y + i * gridDim.y;
        const int n = tile / (g.tiles_x * g.tiles_y);
        const int rem = tile - n * g.tiles_x * g.tiles_y;
        const int ty = rem / g.tiles_x, tx = rem - ty * g.tiles_x;
        const int x0 = tx * C::TX, y0 = ty * C::TY;
        uint8_t* g_tile = smem + st * C::STAGE;
        uint8_t* a_tile = g_tile + C::G_BYTES;
        mbar_wait(&empty[st], phase ^ 1);
        mbar_expect_tx(&full[st], (uint32_t)((HI ? 1 : 2) * g.co_planes * C::G_PLANE + (HI ? 1 : 2) * C::A_HALF));
        tma_load_5d(g_tile, &tmap_g, &full[st], 0, x0, y0, 0, n);
        if constexpr (!HI) tma_load_5d(g_tile + C::G_HALF, &tmap_g, &full[st], 0, x0, y0, g.planes_half, n);
        tma_load_5d(a_tile, &tmap_a, &full[st], 0, x0 - KS / 2, y0 - KS / 2, 0, n);
        if constexpr (!HI) tma_load_5d(a_tile + C::A_HALF, &tmap_a, &full[st], 0, x0 - KS / 2, y0 - KS / 2, C::A_PLANES, n);
        if (++st == C::NSTAGE) { st = 0; phase ^= 1; }
      }
    }
    return;
  }
  // consumers: warpgroup wg owns output channels 64wg..64wg+63 (gradient planes 8wg..8wg+7).  Both operands are
  // MN-major: K = pixels along x (LBO = 128 B between the two 8-pixel halves), SBO = one 8-channel plane.
  const int wg = warp >> 2;
  float acc[C::ACC];
#pragma unroll
  for (int i = 0; i < C::ACC; i++) acc[i] = 0.f;
  int st = 0;
  uint32_t phase = 0;
  for (int i = 0; i < my_tiles; i++) {
    mbar_wait(&full[st], phase);
    const uint32_t g_base = smem_u32(smem + st * C::STAGE) + (uint32_t)(wg * 8 * C::G_PLANE);
    const uint32_t a_base = smem_u32(smem + st * C::STAGE + C::G_BYTES);
    wg_fence();
#pragma unroll
    for (int tl = 0; tl < TPG; tl++) {
      if (tl >= ntaps) break;
      const int tap = tap0 + tl;
      const int ky = tap / KS, kx = tap - ky * KS;
      float* d = acc + tl * NCI / 2;
#pragma unroll 1
      for (int y = 0; y < C::TY; y++) {
        const uint32_t g_row = g_base + (uint32_t)(y * C::TX * 16);
        const uint32_t a_row = a_base + (uint32_t)(((y + ky) * C::HALO_W + kx) * 16);
        const uint64_t gh = make_desc(g_row, 128, C::G_PLANE), gl = make_desc(g_row + C::G_HALF, 128, C::G_PLANE);
        const uint64_t ah = make_desc(a_row, 128, C::A_PLANE), al = make_desc(a_row + C::A_HALF, 128, C::A_PLANE);
        wgmma_bf16_mn<NCI>(d, gh, ah);  // g_hi x a_hi
        if constexpr (!HI) {
          wgmma_bf16_mn<NCI>(d, gl, ah);  // g_lo x a_hi
          wgmma_bf16_mn<NCI>(d, gh, al);  // g_hi x a_lo
        }
      }
    }
    wg_commit();
    wg_wait<0>();
    if (lane == 0) mbar_arrive(&empty[st]);
    if (++st == C::NSTAGE) { st = 0; phase ^= 1; }
  }
  // accumulator fragment: row = output channel, two consecutive columns (input channels) per 8-column group
  const int co = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c0 = (lane & 3) * 2;
  float* base = g.partial + (size_t)(blockIdx.y * gridDim.x + blockIdx.x) * (TPG * 128 * NCI);
#pragma unroll
  for (int tl = 0; tl < TPG; tl++) {
    if (tl >= ntaps) break;
#pragma unroll
    for (int j = 0; j < NCI / 8; j++) {
      const float* v = acc + tl * NCI / 2 + 4 * j;
      float* p = base + ((size_t)tl * 128 + co) * NCI + 8 * j + c0;
      *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
      *reinterpret_cast<float2*>(p + 8 * NCI) = make_float2(v[2], v[3]);
    }
  }
}

// dense[tap][co][c] = sum over the pixel splits, in split order, of the CTAs' partial sums (deterministic)
__global__ void __launch_bounds__(256)
reduce_wgrad_kernel(const float* __restrict__ partial, float* __restrict__ dense, int kk, int tpg, int ngroups,
                    int splits, int nci, int co_valid) {
  const int per_tap = 128 * nci;
  const long long total = (long long)kk * per_tap;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int tap = (int)(i / per_tap);
    const int rem = (int)(i - (long long)tap * per_tap);
    const int grp = tap / tpg, tl = tap - grp * tpg;
    float acc = 0.f;
    if (rem / nci < co_valid) {
      const float* p = partial + ((size_t)grp * tpg + tl) * per_tap + rem;
      for (int s = 0; s < splits; s++) acc += p[(size_t)s * ngroups * tpg * per_tap];
    }
    dense[i] = acc;
  }
}
// db[c] = sum of the per-block partial sums, in block order
__global__ void reduce_bias_kernel(const float* __restrict__ part, float* __restrict__ db, int nsplit, int stride,
                                   int co_valid) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= co_valid) return;
  float acc = 0.f;
  for (int s = 0; s < nsplit; s++) acc += part[(size_t)s * stride + c];
  db[c] = acc;
}

// part[split][c] = sum over this block's images and pixels of (hi + lo).  grid = (planes, splits), 256 threads.
__global__ void __launch_bounds__(256)
bias_grad_kernel(const uint4* __restrict__ gplanes, float* __restrict__ db, int planes_half, int n_img, int hw,
                 int co_valid) {
  __shared__ float s_part[8][256];
  const int plane = blockIdx.x;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const long long total = (long long)n_img * hw;
  for (long long i = (long long)blockIdx.y * 256 + threadIdx.x; i < total; i += (long long)gridDim.y * 256) {
    const int n = (int)(i / hw);
    const int pix = (int)(i - (long long)n * hw);
    const uint4 h4 = gplanes[((size_t)n * 2 * planes_half + plane) * hw + pix];
    const uint4 l4 = gplanes[((size_t)n * 2 * planes_half + planes_half + plane) * hw + pix];
    const uint32_t hs[4] = {h4.x, h4.y, h4.z, h4.w}, ls[4] = {l4.x, l4.y, l4.z, l4.w};
#pragma unroll
    for (int j = 0; j < 8; j++) {
      acc[j] += __uint_as_float(((hs[j >> 1] >> ((j & 1) * 16)) & 0xffffu) << 16) +
                __uint_as_float(((ls[j >> 1] >> ((j & 1) * 16)) & 0xffffu) << 16);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; j++) s_part[j][threadIdx.x] = acc[j];
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o)
#pragma unroll
      for (int j = 0; j < 8; j++) s_part[j][threadIdx.x] += s_part[j][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x < 8) db[(size_t)blockIdx.y * gridDim.x * 8 + plane * 8 + threadIdx.x] = s_part[threadIdx.x][0];
}

// dense [kk][128][nci] -> OIHW gradient tensor:  dst[o][c][t] = scale * dense[t][row_off + o][cd(c)]
__global__ void extract_wgrad_kernel(const float* __restrict__ dense, float* __restrict__ dst, int co, int ci, int kk,
                                     int nci, int row_off, int split, int base0, int base1, float scale) {
  const int total = co * ci * kk;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int t = i % kk;
    int c = (i / kk) % ci;
    int o = i / (kk * ci);
    int cd = c < split ? base0 + c : base1 + (c - split);
    dst[i] = scale * dense[((size_t)t * 128 + row_off + o) * nci + cd];
  }
}

// Backward of out = sum_r refined_r * cm_r, refined = relu(z_r3), cm = sigmoid(z_8)   (net.py:100-108)
//   g_zr3[3r+c] = g_out[c] * cm[r]            where refined[3r+c] > 0
//   g_z8[r]     = (sum_c g_out[c] * refined[3r+c]) * cm[r] * (1 - cm[r])
// Both are written as 16-channel gradient planes (bf16 hi/lo), unused channels zero.
// 16 gradient values of pixel pix of image n -> a 16-channel gradient buffer (planes hi0, hi1, lo0, lo1); HI: the
// single-pass bf16 seed, bf16(v) and lo = 0
template <bool HI>
__device__ __forceinline__ void store_grad16(uint4* base, const float* v, int n, int pix, int hw) {
  uint32_t hi[8], lo[8];
#pragma unroll
  for (int j = 0; j < 16; j += 2) {
    if constexpr (HI) {
      const __nv_bfloat162 hb = __floats2bfloat162_rn(v[j], v[j + 1]);
      hi[j >> 1] = *reinterpret_cast<const uint32_t*>(&hb);
      lo[j >> 1] = 0u;
    } else {
      split_bf16x2(v[j], v[j + 1], hi[j >> 1], lo[j >> 1]);
    }
  }
  uint4* o = base + (size_t)n * 4 * hw + pix;
  o[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  o[hw] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
  o[2 * (size_t)hw] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  o[3 * (size_t)hw] = make_uint4(lo[4], lo[5], lo[6], lo[7]);
}

// go: d(loss)/d(out) at pixel pix of image n of the batch
template <bool HI>
__device__ __forceinline__ void gate_bwd_pixel(const float* go, const float* __restrict__ cm,
                                               const float* __restrict__ refined, uint4* __restrict__ g8,
                                               uint4* __restrict__ gr3, int n, int pix, int hw) {
  float c[3], v8[16], v9[16];
#pragma unroll
  for (int k = 0; k < 3; k++) c[k] = cm[((size_t)n * 3 + k) * hw + pix];
#pragma unroll
  for (int j = 0; j < 16; j++) v8[j] = v9[j] = 0.f;
#pragma unroll
  for (int r = 0; r < 3; r++) {
    float dot = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const float rf = refined[((size_t)n * 9 + 3 * r + k) * hw + pix];
      dot += go[k] * rf;
      v9[3 * r + k] = rf > 0.f ? go[k] * c[r] : 0.f;
    }
    v8[r] = dot * c[r] * (1.0f - c[r]);
  }
  store_grad16<HI>(g8, v8, n, pix, hw);
  store_grad16<HI>(gr3, v9, n, pix, hw);
}

// data-gradient weights: dense_d[row_off + c][col(o)][kk-1-t] = W[o][c][t]   (transpose + spatial flip)
// input channel c lands in row  row_off + c  (c < split)  or  row_off + c + shift  (c >= split)
__global__ void scatter_weights_T_kernel(const float* __restrict__ src, float* __restrict__ dense, int co, int ci,
                                         int kk, int kpad, int row_off, int col_off, int split, int shift) {
  const int total = co * ci * kk;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int t = i % kk;
    int c = (i / kk) % ci;
    int o = i / (kk * ci);
    int row = row_off + c + (c >= split ? shift : 0);
    dense[((size_t)row * kpad + col_off + o) * kk + (kk - 1 - t)] = src[i];
  }
}

// ---- where a slot pixel of a backward pass sits in its image ------------------------------------------------------
// A backward pass runs a batch of slots, each holding one window (or one whole image) at its top-left.  The per-pixel
// kernels below (the seed, the input-gradient copy and the fold) are written once against the slot geometry of
// tiling.cuh (GridGeom, TableGeom: where does pixel pix of slot s sit in its image?), each paired here with the
// images' d(out) and input-gradient tensors.  Only the kept pixels are seeded from d(out).
//
// Per image: d(loss)/d(out) and the four input-gradient tensors (any may be null), fp32 contiguous (1,3,H,W).
struct RaggedGrads {
  const float* g_out;
  float* in[4];
};

// d_out(p): the image's d(out) or d(maps), 3 planes; d_in(p, t): its input gradient t, 3 planes (NULL: not wanted)
// Grid slots: d(out) and the input gradients are contiguous (N,3,H,W) tensors.
struct GridSlots : GridGeom {
  const float* g_out;
  float* in[4];
  __device__ void check_plan() const {}
  __device__ const float* d_out(const SlotPixel& p) const { return g_out + (size_t)p.img * 3 * p.ihw; }
  __device__ float* d_in(const SlotPixel& p, int t) const {
    return in[t] ? in[t] + (size_t)p.img * 3 * p.ihw : nullptr;
  }
};

// Table slots: per image, one RaggedGrads entry of a device table.
struct TableSlots : TableGeom {
  const RaggedGrads* imgs;
  const int* plan;  // wn_backward_ragged: n, slot_h, slot_w as the forward call wrote them; NULL otherwise
  // a backward with sizes other than the forward's stops instead of reading the wrong activations
  __device__ void check_plan() const {
    assert(!plan || (plan[0] == (int)gridDim.y && plan[1] == slot_h && plan[2] == slot_w));
  }
  __device__ const float* d_out(const SlotPixel& p) const { return imgs[p.img].g_out; }
  __device__ float* d_in(const SlotPixel& p, int t) const { return imgs[p.img].in[t]; }
};

// The seed of a backward pass, from go = d(out) at kept pixels and 0 everywhere else (so every window
// back-propagates only the output pixels it owns):
//   kStackAll       the gate (gate_bwd_pixel) -> g8 and gr3
//   kStackCmg       maps = sigmoid(z_8):  g_z8[r] = d(map_r) * cm_r * (1 - cm_r) -> g8
//   kStackRefiners  refiner `which` alone, out = relu(z_r3) of its three columns:  g_zr3[3 which + c] = d(out_c)
//                   where refined[3 which + c] > 0; the other refiners' six columns are exactly 0 -> gr3
// HI: the planes of the single-pass bf16 backward (lo = 0)
template <class Geom, bool HI = false>
__global__ void __launch_bounds__(256)
seed_kernel(Geom geo, int stack, int which, const float* __restrict__ cm, const float* __restrict__ refined,
            uint4* __restrict__ g8, uint4* __restrict__ gr3) {
  geo.check_plan();
  const int hw = geo.slot_hw();
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= hw) return;
  const int s = blockIdx.y;
  const SlotPixel p = geo.at(s, pix);
  const float* g = geo.d_out(p);
  float go[3];
#pragma unroll
  for (int k = 0; k < 3; k++) go[k] = p.kept ? g[k * p.ihw + p.o] : 0.f;
  if (stack == kStackAll) {
    gate_bwd_pixel<HI>(go, cm, refined, g8, gr3, s, pix, hw);
    return;
  }
  float v[16];
#pragma unroll
  for (int j = 0; j < 16; j++) v[j] = 0.f;
  if (stack == kStackCmg) {
#pragma unroll
    for (int r = 0; r < 3; r++) {
      const float c = cm[((size_t)s * 3 + r) * hw + pix];
      v[r] = go[r] * c * (1.0f - c);
    }
  } else {
    float gz[3];  // refiner `which`'s three columns
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const float rf = refined[((size_t)s * 9 + 3 * which + c) * hw + pix];
      gz[c] = rf > 0.f ? go[c] : 0.f;
    }
#pragma unroll
    for (int r = 0; r < 3; r++)  // constant indices into v
#pragma unroll
      for (int c = 0; c < 3; c++) v[3 * r + c] = r == which ? gz[c] : 0.f;
  }
  store_grad16<HI>(stack == kStackCmg ? g8 : gr3, v, s, pix, hw);
}

// d(loss)/d(input images) from the 32-channel buffers of the first layers (12 real channels: packed input k is
// channels 3k..3k+2 of cat[x, wb, he, gc]): a = gin_a (cmg.conv1), b = gin_b (the refiners' conv1), NULL: not part
// of the call.  Input t of the call receives packed input slot[t]: {0, 1, 2, 3} for the whole network (a and b) and
// the cmg (a); {0, which + 1} for refiner `which` (b), which reads cat[x, input which+1] (the forward handed xbar to
// all three refiners; the other refiners' seeds are zero, so their rows of the data gradient add exact zeros).
struct FirstLayerGrads {
  const uint4* a;
  const uint4* b;
  int slot[4];
};

// v[3k + c] = d(loss)/d(packed input k, channel c) at pixel pix of slot n: the buffers given, hi + lo each, summed
// in the order a_hi, a_lo, b_hi, b_lo.  A NULL buffer is skipped.
__device__ __forceinline__ void first_layer_grads_pixel(const uint4* __restrict__ ga, const uint4* __restrict__ gb,
                                                        int n, int pix, int hw, float* v) {
#pragma unroll
  for (int j = 0; j < 16; j++) v[j] = 0.f;
  const uint4* bufs[2] = {ga, gb};
#pragma unroll
  for (int b = 0; b < 2; b++) {
    if (!bufs[b]) continue;
#pragma unroll
    for (int plane = 0; plane < 2; plane++) {
#pragma unroll
      for (int half = 0; half < 2; half++) {  // 32-channel buffers: 4 planes per half
        const uint4 q = bufs[b][((size_t)n * 8 + half * 4 + plane) * hw + pix];
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 8; j++)
          v[plane * 8 + j] += __uint_as_float(((w[j >> 1] >> ((j & 1) * 16)) & 0xffffu) << 16);
      }
    }
  }
}

// channel c of packed input s in v (constant indices into v)
__device__ __forceinline__ float packed_input(const float* v, int s, int c) {
  return s == 0 ? v[c] : s == 1 ? v[3 + c] : s == 2 ? v[6 + c] : v[9 + c];
}

// The untiled calls: each slot's valid extent is copied into its image.  Only the valid extent is read: the first
// layer's data gradient has no ReLU mask and is not zero beyond it.
template <class Geom>
__global__ void __launch_bounds__(256) extract_input_grads_kernel(Geom geo, FirstLayerGrads f) {
  const int hw = geo.slot_hw();
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= hw) return;
  const SlotPixel p = geo.at(blockIdx.y, pix);
  if (!p.valid) return;
  float v[16];
  first_layer_grads_pixel(f.a, f.b, blockIdx.y, pix, hw, v);
#pragma unroll
  for (int t = 0; t < 4; t++) {
    float* d = geo.d_in(p, t);
    if (!d) continue;
#pragma unroll
    for (int c = 0; c < 3; c++) d[c * p.ihw + p.o] = packed_input(v, f.slot[t], c);
  }
}

// The windowed calls: the pass holds windows [w0, w0 + count).  Of the windows of the pass that contain a valid
// pixel's image pixel (tile_cover), only the first does the work: it adds their contributions one at a time in
// ascending window index to what earlier passes left there.  No atomics, and the order of the additions at a pixel
// is the window order whatever the pass size.
template <class Geom>
__global__ void __launch_bounds__(256) fold_input_grads_kernel(Geom geo, FirstLayerGrads f, int count) {
  const int hw = geo.slot_hw();
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= hw) return;
  const SlotPixel p = geo.at(blockIdx.y, pix);
  if (!p.valid) return;
  const long long w0 = geo.w0;
  const TileCover c = tile_cover(p.tiles, p.y, p.x);
  long long first = -1;
  for (int i = c.i0; i <= c.i1 && first < 0; i++)
    for (int j = c.j0; j <= c.j1; j++) {
      const long long k = p.k0 + (long long)i * p.tiles.nx + j;
      if (k >= w0 && k < w0 + count) {
        first = k;
        break;
      }
    }
  if (first != w0 + blockIdx.y) return;
  float acc[12];
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const float* d = geo.d_in(p, q);
#pragma unroll
    for (int ch = 0; ch < 3; ch++) acc[q * 3 + ch] = d ? d[p.o + ch * p.ihw] : 0.f;
  }
  for (int i = c.i0; i <= c.i1; i++)
    for (int j = c.j0; j <= c.j1; j++) {
      const long long k = p.k0 + (long long)i * p.tiles.nx + j;
      if (k < w0 || k >= w0 + count) continue;
      int ys, xs;
      geo.origin(k, &ys, &xs);
      float v[16];
      first_layer_grads_pixel(f.a, f.b, (int)(k - w0), (p.y - ys) * geo.slot_width() + (p.x - xs), hw, v);
#pragma unroll
      for (int q = 0; q < 4; q++)
#pragma unroll
        for (int ch = 0; ch < 3; ch++) acc[q * 3 + ch] += packed_input(v, f.slot[q], ch);
    }
#pragma unroll
  for (int q = 0; q < 4; q++) {
    float* d = geo.d_in(p, q);
    if (!d) continue;
#pragma unroll
    for (int ch = 0; ch < 3; ch++) d[p.o + ch * p.ihw] = acc[q * 3 + ch];
  }
}
// dst.p[k][i] += src.p[k][i] for the 34 parameter gradients; blockIdx.y = k
struct ParamGrads {
  float* p[WN_NUM_PARAMS];
  int size[WN_NUM_PARAMS];
};
__global__ void __launch_bounds__(256) add_param_grads_kernel(ParamGrads dst, ParamGrads src) {
  const int k = blockIdx.y;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < dst.size[k]; i += gridDim.x * 256) dst.p[k][i] += src.p[k][i];
}

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
// The backward of each forward convolution (the refiners' side by side).
enum DgradLayer { kD8 = 0, kD7, kD6, kD5, kD4, kD3, kD2, kDR3, kDR2, kD1, kDR1, kNumDgrad };
// Data gradient (UmmaCfg): ks, kpad = K = forward Cout (padded), npad = N per block = forward Cin, nblk, concat, tps.
// Weight gradient (WgradCfg): nci = forward input channels (padded), tpg = taps per CTA group.  conv = the cmg
// convolution (-1: refiner conv2 / conv3, -2: refiner conv1).
struct DgradSpec {
  int ks, kpad, npad, nblk, concat, tps, nci, tpg, conv;
};
static constexpr DgradSpec kDSpecs[kNumDgrad] = {
    // ks kpad npad nblk concat tps nci tpg conv
    {3, 16, 64, 1, 1, 9, 64, 4, 7},       // kD8
    {3, 64, 64, 1, 1, 9, 64, 4, 6},       // kD7
    {5, 64, 64, 1, 1, 5, 64, 4, 5},       // kD6
    {7, 64, 64, 1, 1, 7, 64, 4, 4},       // kD5
    {1, 64, 128, 1, 0, 1, 128, 1, 3},     // kD4
    {3, 128, 128, 1, 0, 3, 128, 2, 2},    // kD3
    {5, 128, 128, 1, 0, 5, 128, 2, 1},    // kD2
    {3, 16, 96, 1, 0, 9, 96, 2, -1},      // kDR3
    {5, 96, 32, 3, 1, 5, 96, 2, -1},      // kDR2
    // data gradients with respect to the packed 16-channel input (only when an input image requires grad):
    // from cmg.conv1 (K = 128) and from the three refiner conv1 (K = 96); 32 rows, 12 real
    {7, 128, 32, 1, 1, 7, 16, 16, 0},     // kD1
    {7, 96, 32, 1, 1, 7, 16, 16, -2}};    // kDR1

struct UmmaBwd {
  uint8_t* stages[kNumDgrad];
  float* zero_bias;  // 256 zeros: the dgrad epilogue has no bias
  float* dense;      // packing scratch
};

static size_t dgrad_stage_bytes(const DgradSpec& s) {
  return (size_t)(s.kpad / 16) * s.ks * s.ks * s.npad * 64;
}

int bwd_pack_weights(wn_handle* h, const float* const* params, cudaStream_t stream) {
  if (!h->bwd) h->bwd = (UmmaBwd*)calloc(1, sizeof(UmmaBwd));
  for (int i = 0; i < kNumDgrad; i++)
    if (!h->bwd->stages[i]) WN_CUDA(cudaMalloc(&h->bwd->stages[i], dgrad_stage_bytes(kDSpecs[i])));
  if (!h->bwd->zero_bias) WN_CUDA(cudaMalloc(&h->bwd->zero_bias, 256 * sizeof(float)));
  if (!h->bwd->dense) WN_CUDA(cudaMalloc(&h->bwd->dense, (size_t)128 * 128 * 49 * sizeof(float)));
  UmmaBwd* u = h->bwd;
  WN_CUDA(cudaMemsetAsync(u->zero_bias, 0, 256 * sizeof(float), stream));
  for (int li = 0; li < kNumDgrad; li++) {
    const DgradSpec& s = kDSpecs[li];
    const int kk = s.ks * s.ks, rows = s.npad * s.nblk;
    WN_CUDA(cudaMemsetAsync(u->dense, 0, (size_t)rows * s.kpad * kk * sizeof(float), stream));
    if (s.conv >= 0) {
      const LayerDesc& d = kCmg[s.conv];
      scatter_weights_T_kernel<<<128, 256, 0, stream>>>(params[2 * s.conv], u->dense, d.cout, d.cin, kk, s.kpad, 0, 0,
                                                        d.cin, 0);
      WN_LAUNCH_CHECK(h);
    } else if (s.conv == -2) {
      for (int r = 0; r < 3; r++) {  // refiner r reads cat[x, input r+1]: rows 0..2 and 3(r+1)..3(r+1)+2
        scatter_weights_T_kernel<<<128, 256, 0, stream>>>(params[2 * (8 + 3 * r)], u->dense, 32, 6, kk, s.kpad, 0, 32 * r,
                                                          3, 3 * (r + 1) - 3);
        WN_LAUNCH_CHECK(h);
      }
    } else {
      for (int r = 0; r < 3; r++) {
        const int conv = 8 + 3 * r + (li == kDR3 ? 2 : 1);
        const int co = li == kDR3 ? 3 : 32;
        scatter_weights_T_kernel<<<128, 256, 0, stream>>>(params[2 * conv], u->dense, co, 32, kk, s.kpad, 32 * r,
                                                          (li == kDR3 ? 3 : 32) * r, 32, 0);
        WN_LAUNCH_CHECK(h);
      }
    }
    pack_stages_kernel<<<256, 256, 0, stream>>>(u->dense, (__nv_bfloat16*)u->stages[li], s.npad, s.kpad, kk,
                                                  s.concat, s.nblk);
    WN_LAUNCH_CHECK(h);
  }
  return WN_OK;
}

void bwd_free(wn_handle* h) {
  if (!h->bwd) return;
  for (int i = 0; i < kNumDgrad; i++)
    if (h->bwd->stages[i]) cudaFree(h->bwd->stages[i]);
  if (h->bwd->zero_bias) cudaFree(h->bwd->zero_bias);
  if (h->bwd->dense) cudaFree(h->bwd->dense);
  free(h->bwd);
  h->bwd = nullptr;
}

// ---- training workspace ------------------------------------------------------------------
struct TrainBuffers {
  FwdBuffers f;
  uint4 *ga, *gb, *gra, *grb, *g8, *gr3, *gin_a, *gin_b;
  float* dense;
  float* partial;  // per-CTA partial sums of the weight-gradient GEMM / per-block partial bias sums
};
static constexpr size_t kDenseBytes = (size_t)49 * 128 * 128 * sizeof(float);
// one slot per CTA of a weight-gradient launch (one wave: <= SM count), each TPG * NCI <= 256 accumulator columns
// x 128 rows of fp32
static constexpr size_t kPartialSlotBytes = (size_t)512 * 128 * sizeof(float);
static constexpr int kPartialSlots = 192;
static constexpr size_t kPartialBytes = kPartialSlots * kPartialSlotBytes;
// bytes per pixel: act0 64 | a1..a3 512 each | a4..a7 256 each | r1, r2 384 each | cm 12 | refined 36 |
//                  gradient ping-pong 512 + 512 + 384 + 384 | 16-channel gradients 64 + 64
static constexpr size_t kTrainBytesPerPixel =
    64 + 3 * 512 + 4 * 256 + 2 * 384 + 12 + 36 + 2 * 512 + 2 * 384 + 2 * 64 + 2 * 128;  // + two 32-ch input-gradient buffers

size_t train_workspace_bytes(int n, int h, int w) {
  return (size_t)n * h * w * kTrainBytesPerPixel + kDenseBytes + kPartialBytes + 8192;
}

// The buffers of one training pass of `stack` (FwdStack): kStackAll has all of them; a sub-module called on its own
// (kStackCmg, kStackRefiners) leaves out the other stack's, which stay NULL.  Returns the bytes used from the
// workspace's start, the 1 KiB alignment of the first region included.
static size_t carve(TrainBuffers* t, void* workspace, size_t px, int stack = kStackAll) {
  const uintptr_t start = (uintptr_t)workspace;
  uintptr_t ws = (start + 1023) / 1024 * 1024;
  auto take = [&](size_t bytes) {
    const uintptr_t p = ws;
    ws += (bytes + 1023) / 1024 * 1024;
    return (void*)p;
  };
  const bool cmg = stack != kStackRefiners, ref = stack != kStackCmg;
  memset(t, 0, sizeof(*t));
  t->f.act0 = (uint4*)take(px * 64);
  if (cmg) {
    for (int l = 1; l <= 3; l++) t->f.a[l] = (uint4*)take(px * 512);
    for (int l = 4; l <= 7; l++) t->f.a[l] = (uint4*)take(px * 256);
  }
  if (ref) {
    t->f.r[1] = (uint4*)take(px * 384);
    t->f.r[2] = (uint4*)take(px * 384);
  }
  if (cmg) t->f.cm = (float*)take(px * 12);
  if (ref) t->f.refined = (float*)take(px * 36);
  t->f.exact_flag = (int*)take(256);
  if (cmg) {
    t->ga = (uint4*)take(px * 512);
    t->gb = (uint4*)take(px * 512);
  }
  if (ref) {
    t->gra = (uint4*)take(px * 384);
    t->grb = (uint4*)take(px * 384);
  }
  if (cmg) t->g8 = (uint4*)take(px * 64);
  if (ref) t->gr3 = (uint4*)take(px * 64);
  if (cmg) t->gin_a = (uint4*)take(px * 128);
  if (ref) t->gin_b = (uint4*)take(px * 128);
  t->dense = (float*)take(kDenseBytes);
  t->partial = (float*)take(kPartialBytes);
  return (size_t)(ws - start);
}

// exactly what carve() takes of a workspace of any alignment
size_t submodule_train_workspace_bytes(int n, int h, int w, int stack) {
  TrainBuffers t;
  return carve(&t, nullptr, (size_t)n * h * w, stack) + 1023;
}

static int check_train_args(int n, int H, int W, size_t bytes) {
  if ((long long)n * H * W > kTrainMaxPixels) {
    set_error("training pass limited to %lld pixels per call (got %lld)", kTrainMaxPixels, (long long)n * H * W);
    return WN_E_UNSUPPORTED;
  }
  // carve() aligns every region to 1 KiB: allow for it
  if (bytes < train_workspace_bytes(n, H, W) + 24 * 1024) {
    set_error("training workspace too small: %zu < %zu", bytes, train_workspace_bytes(n, H, W) + 24 * 1024);
    return WN_E_WORKSPACE;
  }
  return WN_OK;
}

size_t train_workspace_bytes_padded(int n, int h, int w) { return train_workspace_bytes(n, h, w) + 24 * 1024; }

int forward_train(wn_handle* h, const float* const in[4], const int64_t st[4][4], float* out, int n, int H, int W,
                  void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  int rc = check_train_args(n, H, W, workspace_bytes);
  if (rc) return rc;
  TrainBuffers t;
  carve(&t, workspace, (size_t)n * H * W);
  FwdOpts o;
  o.scheme = train_scheme(h);
  return umma_forward_layers(h, in, st, out, n, H, W, t.f, stream, o);
}

static int make_plane_tmap(CUtensorMap* tm, void* base, int planes_total, int N, int H, int W, int box_w, int box_h,
                           int box_planes) {
  cuuint64_t dims[5] = {8, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)planes_total, (cuuint64_t)N};
  cuuint64_t strides[4] = {16, (cuuint64_t)W * 16, (cuuint64_t)H * W * 16, (cuuint64_t)planes_total * H * W * 16};
  cuuint32_t box[5] = {8, (cuuint32_t)box_w, (cuuint32_t)box_h, (cuuint32_t)box_planes, 1};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = g_encode(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with %d (wgrad planes=%d box=%dx%dx%d)", (int)r, planes_total, box_w,
              box_h, box_planes);
    return WN_E_CUDA;
  }
  return WN_OK;
}

// dense[tap][128][nci] += sum_px g[px][co] * a[px + tap][ci]
template <int LI>
static int launch_wgrad(wn_handle* h, uint4* gplanes, int co_valid, uint4* aplanes, float* dense, float* partial, int n,
                        int H, int W, cudaStream_t stream) {
  constexpr DgradSpec s = kDSpecs[LI];
  using C = WgradCfg<s.ks, s.nci, s.tpg>;
  const int co_planes = (co_valid + 7) / 8;
  const int planes_half = (co_valid + 15) / 16 * 2;  // gradient buffers hold a multiple of 16 channels
  CUtensorMap tg, ta;
  int rc = make_plane_tmap(&tg, gplanes, 2 * planes_half, n, H, W, C::TX, C::TY, co_planes);
  if (rc) return rc;
  rc = make_plane_tmap(&ta, aplanes, 2 * C::A_PLANES, n, H, W, C::HALO_W, C::HALO_H, C::A_PLANES);
  if (rc) return rc;
  WgradArgs a;
  a.partial = partial;
  a.N = n; a.H = H; a.W = W;
  a.co_planes = co_planes;
  a.planes_half = planes_half;
  a.co_valid = co_valid;
  a.tiles_x = (W + C::TX - 1) / C::TX;
  a.tiles_y = (H + C::TY - 1) / C::TY;
  const long long tiles = (long long)a.tiles_x * a.tiles_y * n;
  long long splits = h->sm_count / C::NGROUPS;  // one wave: every CTA owns an SM (shared memory footprint)
  if (splits > tiles) splits = tiles;
  if (splits < 1) splits = 1;
  if (splits * C::NGROUPS > kPartialSlots) splits = kPartialSlots / C::NGROUPS;
  static_assert((size_t)s.tpg * 128 * s.nci * sizeof(float) <= kPartialSlotBytes, "partial-sum slot");
  auto kern = h->train_bf16 ? wgrad_umma_kernel<s.ks, s.nci, s.tpg, true> : wgrad_umma_kernel<s.ks, s.nci, s.tpg>;
  WN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
  kern<<<dim3(C::NGROUPS, (unsigned)splits), kWgradThreads, C::SMEM_BYTES, stream>>>(tg, ta, a);
  WN_LAUNCH_CHECK(h);
  reduce_wgrad_kernel<<<256, 256, 0, stream>>>(partial, dense, s.ks * s.ks, s.tpg, C::NGROUPS, (int)splits, s.nci,
                                               co_valid);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

static int extract(wn_handle* h, const float* dense, float* dst, int co, int ci, int ks, int nci, int row_off,
                   int split, int base0, int base1, float scale, cudaStream_t stream) {
  extract_wgrad_kernel<<<64, 256, 0, stream>>>(dense, dst, co, ci, ks * ks, nci, row_off, split, base0, base1, scale);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

static int bias_grad(wn_handle* h, const uint4* gplanes, int planes_half, int co_valid, float* db, float* partial, int n,
                     int hw, cudaStream_t stream) {
  const int planes = (co_valid + 7) / 8;
  bias_grad_kernel<<<dim3(planes, 64), 256, 0, stream>>>(gplanes, partial, planes_half, n, hw, co_valid);
  WN_LAUNCH_CHECK(h);
  reduce_bias_kernel<<<(co_valid + 127) / 128, 128, 0, stream>>>(partial, db, 64, planes * 8, co_valid);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

template <int LI>
static int launch_dgrad(wn_handle* h, uint4* g_in, uint4* g_out, const uint4* saved, int n, int H, int W,
                        cudaStream_t stream) {
  constexpr DgradSpec s = kDSpecs[LI];
  constexpr int out_channels = s.npad * s.nblk;
  ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.N = n; a.H = H; a.W = W;
  a.dst0.base = g_out;
  a.dst0.planes_half = out_channels / 8;
  a.split_c = out_channels;
  a.cout = out_channels;
  a.mask_base = saved;  // nullptr: no ReLU in front (network input)
  a.mask_planes_half = out_channels / 8;
  if (h->train_bf16)
    return launch_conv<s.ks, s.kpad, s.npad, kEpiDgrad, s.concat, s.nblk, s.tps, kFmtHi>(
        h, kSlotGate, h->bwd->stages[LI], h->bwd->zero_bias, g_in, a, stream);
  return launch_conv<s.ks, s.kpad, s.npad, kEpiDgrad, s.concat, s.nblk, s.tps>(h, kSlotGate, h->bwd->stages[LI],
                                                                              h->bwd->zero_bias, g_in, a, stream);
}

// wn_debug_backward_layer: the backward pass stops after the seed (buffer kDebugG8 or kDebugGr3) or after
// data-gradient launch li (buffer kDebugDgrad + li) and decodes that buffer into dst (the gradient buffers ping-pong,
// so it cannot be read afterwards).  buffer = -1: the normal path, never stops.
static constexpr int kDebugG8 = 12, kDebugGr3 = 13, kDebugDgrad = 14;
struct BwdStop {
  int buffer = -1;
  float* dst = nullptr;
};
static constexpr int kBwdStopped = 1;  // returned up the call chain once the buffer asked for has been decoded

static int stop_after(wn_handle* h, const BwdStop& stop, int li, const uint4* g_out, int n, int hw,
                      cudaStream_t stream) {
  if (stop.buffer != kDebugDgrad + li) return WN_OK;
  const int rc = decode_planes(h, g_out, stop.dst, kDSpecs[li].npad * kDSpecs[li].nblk / 8, n, hw, stream);
  return rc ? rc : kBwdStopped;
}

// Backward of one cmg convolution from g, the gradient with respect to its output: its weight and bias gradients,
// then, when g_dst is given, the gradient with respect to its input into g_dst.  Its input is the saved activation
// a[conv], whose zeros gate that gradient (ReLU'); conv 0 reads act0 instead, the images * 255 with no ReLU.
template <int LI>
static int cmg_conv_backward(wn_handle* h, const TrainBuffers& t, float* const* grads, uint4* g, uint4* g_dst, int n,
                             int H, int W, cudaStream_t stream, const BwdStop& stop) {
  constexpr DgradSpec s = kDSpecs[LI];
  static_assert(s.conv >= 0, "not a cmg convolution");
  const LayerDesc& d = kCmg[s.conv];
  uint4* act = s.conv ? t.f.a[s.conv] : t.f.act0;
  int rc;
  if ((rc = launch_wgrad<LI>(h, g, d.cout, act, t.dense, t.partial, n, H, W, stream))) return rc;
  if ((rc = extract(h, t.dense, grads[2 * s.conv], d.cout, d.cin, s.ks, s.nci, 0, d.cin, 0, 0,
                    s.conv ? 1.f : 1.f / 255.f, stream)))
    return rc;
  if ((rc = bias_grad(h, g, (d.cout + 15) / 16 * 2, d.cout, grads[2 * s.conv + 1], t.partial, n, H * W, stream)))
    return rc;
  if (!g_dst) return WN_OK;
  if ((rc = launch_dgrad<LI>(h, g, g_dst, s.conv ? act : nullptr, n, H, W, stream))) return rc;
  return stop_after(h, stop, LI, g_dst, n, H * W, stream);
}

// The two halves of the backward pass of a batch whose forward activations are in t.  The confidence-map half starts
// from the gradient planes t.g8, the refiner half from t.gr3 (seed_kernel).  Each
// overwrites its stack's parameter gradients in grads (state-dict order) and, when want_input_grads, writes the data
// gradient of the packed 16-channel input into t.gin_a (cmg.conv1) or t.gin_b (the refiners' conv1).
static int backward_cmg(wn_handle* h, const TrainBuffers& t, float* const* grads, bool want_input_grads, int n, int H,
                        int W, cudaStream_t stream, const BwdStop& stop = BwdStop()) {
  int rc;
  // conv8 ... conv1, the gradient ping-ponging between ga and gb.  conv8's output gradient g8 has 16-channel planes,
  // 3 valid; conv1's input gradient only when asked for
  if ((rc = cmg_conv_backward<kD8>(h, t, grads, t.g8, t.ga, n, H, W, stream, stop))) return rc;
  if ((rc = cmg_conv_backward<kD7>(h, t, grads, t.ga, t.gb, n, H, W, stream, stop))) return rc;
  if ((rc = cmg_conv_backward<kD6>(h, t, grads, t.gb, t.ga, n, H, W, stream, stop))) return rc;
  if ((rc = cmg_conv_backward<kD5>(h, t, grads, t.ga, t.gb, n, H, W, stream, stop))) return rc;
  if ((rc = cmg_conv_backward<kD4>(h, t, grads, t.gb, t.ga, n, H, W, stream, stop))) return rc;
  if ((rc = cmg_conv_backward<kD3>(h, t, grads, t.ga, t.gb, n, H, W, stream, stop))) return rc;
  if ((rc = cmg_conv_backward<kD2>(h, t, grads, t.gb, t.ga, n, H, W, stream, stop))) return rc;
  return cmg_conv_backward<kD1>(h, t, grads, t.ga, want_input_grads ? t.gin_a : nullptr, n, H, W, stream, stop);
}

// conv3, conv2, conv1 of the three refiners side by side.  which = -1: the gradients of all three; 0..2: of refiner
// `which` alone (the launches are the same, only its weight and bias gradients are extracted)
static int backward_refiners(wn_handle* h, const TrainBuffers& t, float* const* grads, int which,
                             bool want_input_grads, int n, int H, int W, cudaStream_t stream,
                             const BwdStop& stop = BwdStop()) {
  int rc;
  const int hw = H * W;
  const int r0 = which < 0 ? 0 : which, r1 = which < 0 ? 3 : which + 1;
  auto gw = [&](int conv) { return grads[2 * conv]; };
  auto gb = [&](int conv) { return grads[2 * conv + 1]; };
  if ((rc = launch_wgrad<kDR3>(h, t.gr3, 9, t.f.r[2], t.dense, t.partial, n, H, W, stream))) return rc;
  for (int r = r0; r < r1; r++) {
    if ((rc = extract(h, t.dense, gw(8 + 3 * r + 2), 3, 32, 3, 96, 3 * r, 32, 32 * r, 0, 1.f, stream))) return rc;
  }
  {
    // the nine bias gradients sit in one 16-channel buffer: reduce once, then split per refiner
    float* tmp = t.dense + (size_t)9 * 128 * 96;
    if ((rc = bias_grad(h, t.gr3, 2, 9, tmp, t.partial, n, hw, stream))) return rc;
    for (int r = r0; r < r1; r++)
      WN_CUDA(cudaMemcpyAsync(gb(8 + 3 * r + 2), tmp + 3 * r, 3 * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  }
  if ((rc = launch_dgrad<kDR3>(h, t.gr3, t.gra, t.f.r[2], n, H, W, stream))) return rc;
  if ((rc = stop_after(h, stop, kDR3, t.gra, n, hw, stream))) return rc;
  if ((rc = launch_wgrad<kDR2>(h, t.gra, 96, t.f.r[1], t.dense, t.partial, n, H, W, stream))) return rc;
  {
    float* tmp = t.dense + (size_t)25 * 128 * 96;
    if ((rc = bias_grad(h, t.gra, 12, 96, tmp, t.partial, n, hw, stream))) return rc;
    for (int r = r0; r < r1; r++) {
      if ((rc = extract(h, t.dense, gw(8 + 3 * r + 1), 32, 32, 5, 96, 32 * r, 32, 32 * r, 0, 1.f, stream))) return rc;
      WN_CUDA(cudaMemcpyAsync(gb(8 + 3 * r + 1), tmp + 32 * r, 32 * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    }
  }
  if ((rc = launch_dgrad<kDR2>(h, t.gra, t.grb, t.f.r[1], n, H, W, stream))) return rc;
  if ((rc = stop_after(h, stop, kDR2, t.grb, n, hw, stream))) return rc;
  if ((rc = launch_wgrad<kDR1>(h, t.grb, 96, t.f.act0, t.dense, t.partial, n, H, W, stream))) return rc;
  {
    float* tmp = t.dense + (size_t)49 * 128 * 16;
    if ((rc = bias_grad(h, t.grb, 12, 96, tmp, t.partial, n, hw, stream))) return rc;
    for (int r = r0; r < r1; r++) {
      // refiner r reads cat[x, input r+1]: channels 0..2 and 3(r+1)..3(r+1)+2 of the packed input
      if ((rc = extract(h, t.dense, gw(8 + 3 * r), 32, 6, 7, 16, 32 * r, 3, 0, 3 * (r + 1), 1.f / 255.f, stream))) return rc;
      WN_CUDA(cudaMemcpyAsync(gb(8 + 3 * r), tmp + 32 * r, 32 * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    }
  }
  if (!want_input_grads) return WN_OK;
  if ((rc = launch_dgrad<kDR1>(h, t.grb, t.gin_b, nullptr, n, H, W, stream))) return rc;
  return stop_after(h, stop, kDR1, t.gin_b, n, hw, stream);
}

// The whole network: the 34 parameter gradients into grads (overwritten) and, when want_input_grads, t.gin_a and
// t.gin_b
static int backward_layers(wn_handle* h, const TrainBuffers& t, float* const* grads, bool want_input_grads, int n,
                           int H, int W, cudaStream_t stream, const BwdStop& stop = BwdStop()) {
  int rc = backward_cmg(h, t, grads, want_input_grads, n, H, W, stream, stop);
  return rc ? rc : backward_refiners(h, t, grads, -1, want_input_grads, n, H, W, stream, stop);
}

// One backward pass over n slots of H x W whose training forward is in t, at the slots of geo: the seed of `stack`
// (seed_kernel), that stack's backward (its parameter gradients into grads, overwritten), then, when want_in, the
// input gradients of the first layer, copied into the images (untiled calls) or folded into them (windowed calls).
template <class Geom>
static int backward_pass(wn_handle* h, const Geom& geo, int stack, int which, const TrainBuffers& t,
                         float* const* grads, bool want_in, bool fold, int n, int H, int W, cudaStream_t stream,
                         const BwdStop& stop = BwdStop()) {
  const dim3 grid((unsigned)(((size_t)H * W + 255) / 256), n);
  if (h->train_bf16)
    seed_kernel<Geom, true><<<grid, 256, 0, stream>>>(geo, stack, which, t.f.cm, t.f.refined, t.g8, t.gr3);
  else
    seed_kernel<<<grid, 256, 0, stream>>>(geo, stack, which, t.f.cm, t.f.refined, t.g8, t.gr3);
  WN_LAUNCH_CHECK(h);
  int rc;
  if (stop.buffer == kDebugG8 || stop.buffer == kDebugGr3) {
    rc = decode_planes(h, stop.buffer == kDebugG8 ? t.g8 : t.gr3, stop.dst, 2, n, H * W, stream);
    return rc ? rc : kBwdStopped;
  }
  rc = stack == kStackAll   ? backward_layers(h, t, grads, want_in, n, H, W, stream, stop)
       : stack == kStackCmg ? backward_cmg(h, t, grads, want_in, n, H, W, stream, stop)
                            : backward_refiners(h, t, grads, which, want_in, n, H, W, stream, stop);
  if (rc || !want_in) return rc;
  // carve() leaves the other stack's buffer of a sub-module NULL
  FirstLayerGrads f = {t.gin_a, t.gin_b, {0, 1, 2, 3}};
  if (stack == kStackRefiners) f.slot[1] = which + 1;
  if (fold)
    fold_input_grads_kernel<<<grid, 256, 0, stream>>>(geo, f, n);
  else
    extract_input_grads_kernel<<<grid, 256, 0, stream>>>(geo, f);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

static int check_bwd_packed(const wn_handle* h) {
  if (h->bwd && h->umma) return WN_OK;
  set_error("backward weights have not been packed");
  return WN_E_STATE;
}

static int check_submodule_args(int n, int H, int W, int stack, size_t bytes);

// The training buffers of an untiled call of `stack`, as its training forward left them in the workspace
static int untiled_buffers(TrainBuffers* t, int stack, int n, int H, int W, void* workspace, size_t workspace_bytes) {
  int rc = stack == kStackAll ? check_train_args(n, H, W, workspace_bytes)
                              : check_submodule_args(n, H, W, stack, workspace_bytes);
  if (rc) return rc;
  if ((rc = get_encoder())) return rc;
  carve(t, workspace, (size_t)n * H * W, stack);
  return WN_OK;
}

// The slots of geo; g: d(out) or d(maps); in: NULL or n_in input gradients
static GridSlots grid_slots(const GridGeom& geo, const float* g, float* const* in, int n_in) {
  GridSlots s = {geo, g, {nullptr, nullptr, nullptr, nullptr}};
  for (int i = 0; in && i < n_in; i++) s.in[i] = in[i];
  return s;
}

static bool any_of4(float* const* p, int count) {
  if (!p) return false;
  for (int i = 0; i < count; i++)
    if (p[i]) return true;
  return false;
}

// wn_backward, wn_confidence_maps_backward, wn_refine_backward: the backward of what the stack's training forward
// left in the workspace
static int untiled_backward(wn_handle* h, int stack, int which, const float* grad, float* const* grads,
                            float* const* input_grads, int n, int H, int W, void* workspace, size_t workspace_bytes,
                            cudaStream_t stream) {
  int rc = check_bwd_packed(h);
  if (rc) return rc;
  TrainBuffers t;
  if ((rc = untiled_buffers(&t, stack, n, H, W, workspace, workspace_bytes))) return rc;
  const int n_in = stack == kStackRefiners ? 2 : 4;
  return backward_pass(h, grid_slots(whole_images(H, W), grad, input_grads, n_in), stack, which, t, grads,
                       any_of4(input_grads, n_in), false, n, H, W, stream);
}

int backward(wn_handle* h, const float* grad_out, float* const* grads, float* const* input_grads, int n, int H,
             int W, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return untiled_backward(h, kStackAll, -1, grad_out, grads, input_grads, n, H, W, workspace, workspace_bytes, stream);
}

// ---- the ragged training step ------------------------------------------------------------------------------------
// The n images of a call run as one pass of n slots of the per-axis maximum size, image i in slot i at the top-left.
// The forward masks every ReLU activation beyond each image (the RAG layers), and the backward seeds 0 there, so
// every gradient plane a weight-gradient GEMM reads is 0 at masked pixels and adds exact zeros (DESIGN.md 4.10).
// Workspace: [plan: n, slot_h, slot_w | windows | PackInArgs | RaggedGrads, one each per image][the training carve-up
// of n slots].  The backward derives its carve-up from the sizes it is given; its seed asserts that they give the
// plan the forward wrote, so a backward with other sizes stops instead of reading the wrong activations.
static void ragged_slot(const int* hs, const int* ws, int n, int* sh, int* sw) {
  *sh = *sw = 0;
  for (int i = 0; i < n; i++) {
    *sh = hs[i] > *sh ? hs[i] : *sh;
    *sw = ws[i] > *sw ? ws[i] : *sw;
  }
}
// the table: [plan: n, slot_h, slot_w | windows | PackInArgs | RaggedGrads]
static HostTable ragged_train_table(int n) {
  return HostTable({256, (size_t)n * sizeof(RaggedWindow), (size_t)n * sizeof(PackInArgs),
                    (size_t)n * sizeof(RaggedGrads)});
}

size_t train_ragged_workspace_bytes(const int* hs, const int* ws, int n) {
  int sh, sw;
  ragged_slot(hs, ws, n, &sh, &sw);
  return 256 + ragged_train_table(n).bytes() + train_workspace_bytes_padded(n, sh, sw);
}

// The per-image host table of a ragged call: imgs[i] (the four inputs and their strides) when imgs is given, and
// grads[i] (d(out) and the four input gradients, NULL: not wanted) when grads is given.  Returns whether any input
// gradient is wanted.
static bool ragged_table(const wn_ragged_tensors* images, const float* const* grad_out, float* const* input_grads,
                         int n, PackInArgs* imgs, RaggedGrads* grads) {
  bool want_in = false;
  for (int i = 0; i < n; i++) {
    if (imgs) {
      const wn_ragged_tensors& d = images[i];
      const float* p[4] = {d.x, d.wb, d.he, d.gc};
      imgs[i] = pack_args(p, d.in_strides);
    }
    if (grads) {
      grads[i].g_out = grad_out[i];
      for (int t = 0; t < 4; t++) {
        grads[i].in[t] = input_grads ? input_grads[4 * i + t] : nullptr;
        want_in = want_in || grads[i].in[t];
      }
    }
  }
  return want_in;
}

// the table's parts and the training buffers of a workspace of any alignment
struct RaggedTrainLayout {
  HostTable table;
  uint8_t* base;  // the device table
  int* plan;      // n, slot_h, slot_w of the forward call
  RaggedWindow* wins;
  PackInArgs* imgs;
  RaggedGrads* grads;
  TrainBuffers t;
};
static RaggedTrainLayout ragged_train_layout(void* workspace, int n, int sh, int sw) {
  RaggedTrainLayout l = {ragged_train_table(n), (uint8_t*)align256((uintptr_t)workspace)};
  l.plan = l.table.dev<int>(l.base, 0);
  l.wins = l.table.dev<RaggedWindow>(l.base, 1);
  l.imgs = l.table.dev<PackInArgs>(l.base, 2);
  l.grads = l.table.dev<RaggedGrads>(l.base, 3);
  carve(&l.t, l.base + l.table.bytes(), (size_t)n * sh * sw);
  return l;
}

int forward_train_ragged(wn_handle* h, const wn_ragged_tensors* images, int n, void* workspace, size_t workspace_bytes,
                         cudaStream_t stream) {
  std::vector<int> hs, ws;
  ragged_sizes(images, n, &hs, &ws);
  const size_t need = train_ragged_workspace_bytes(hs.data(), ws.data(), n);
  if (workspace_bytes < need) {
    set_error("ragged training workspace too small: %zu < %zu", workspace_bytes, need);
    return WN_E_WORKSPACE;
  }
  int sh, sw;
  ragged_slot(hs.data(), ws.data(), n, &sh, &sw);
  RaggedTrainLayout l = ragged_train_layout(workspace, n, sh, sw);
  // the plan, the windows and the PackInArgs; the backward writes the RaggedGrads
  int* plan = l.table.part<int>(0);
  plan[0] = n;
  plan[1] = sh;
  plan[2] = sw;
  RaggedWindow* wins = l.table.part<RaggedWindow>(1);
  for (int i = 0; i < n; i++) {
    RaggedWindow r = {};
    r.out_f32 = images[i].out;
    r.img = i;
    r.H = r.vh = r.ky1 = images[i].height;
    r.W = r.vw = r.kx1 = images[i].width;
    wins[i] = r;
  }
  ragged_table(images, nullptr, nullptr, n, l.table.part<PackInArgs>(2), nullptr);
  int rc = l.table.upload(l.base, stream, 0, 3);
  if (rc) return rc;
  WN_CUDA(cudaMemsetAsync(l.t.f.exact_flag, 1, sizeof(int), stream));  // nonzero = "all inputs are 8-bit levels"
  const TableGeom geo = {l.wins, 0, sh, sw, sh, sw};  // every image is one window of its own size
  if ((rc = pack_inputs(h, geo, l.imgs, n, nullptr, l.t.f.exact_flag, stream))) return rc;
  FwdOpts o;
  o.scheme = train_scheme(h);
  if ((rc = pack_inputs(h, geo, l.imgs, n, l.t.f.act0, nullptr, stream, o.scheme == kSchemeBf16))) return rc;
  o.packed = true;
  o.rwin = l.wins;
  const int64_t none[4][4] = {};
  const float* no_in[4] = {nullptr, nullptr, nullptr, nullptr};
  return umma_forward_layers(h, no_in, none, nullptr, n, sh, sw, l.t.f, stream, o);
}

int backward_ragged(wn_handle* h, const int* hs, const int* ws, const float* const* grad_out, float* const* grads,
                    float* const* input_grads, int n, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  int rc = check_bwd_packed(h);
  if (rc) return rc;
  const size_t need = train_ragged_workspace_bytes(hs, ws, n);
  if (workspace_bytes < need) {
    set_error("ragged training workspace too small: %zu < %zu", workspace_bytes, need);
    return WN_E_WORKSPACE;
  }
  if ((rc = get_encoder())) return rc;
  int sh, sw;
  ragged_slot(hs, ws, n, &sh, &sw);
  RaggedTrainLayout l = ragged_train_layout(workspace, n, sh, sw);
  const bool want_in = ragged_table(nullptr, grad_out, input_grads, n, nullptr, l.table.part<RaggedGrads>(3));
  if ((rc = l.table.upload(l.base, stream, 3, 4))) return rc;
  // every image is one window of its own size
  const TableSlots geo = {{l.wins, 0, sh, sw, sh, sw}, l.grads, l.plan};
  return backward_pass(h, geo, kStackAll, -1, l.t, grads, want_in, false, n, sh, sw, stream);
}

// ---- the sub-modules under autograd (wn_confidence_maps_train / _backward, wn_refine_train / _backward) -----------
// The training forward of one stack (bf16x3 and the exact-levels flag, as forward_train; a refiner's first layer is
// kRL1, the refiners' conv1 without cmg.conv1) keeps its activations in a workspace carved for that stack.  The
// backward seeds that stack's half of the backward pass from d(maps) or d(out) and writes the sub-module's own
// parameter gradients and, on request, the gradients of its own inputs.
static int check_submodule_args(int n, int H, int W, int stack, size_t bytes) {
  if ((long long)n * H * W > kTrainMaxPixels) {
    set_error("training pass limited to %lld pixels per call (got %lld)", kTrainMaxPixels, (long long)n * H * W);
    return WN_E_UNSUPPORTED;
  }
  const size_t need = submodule_train_workspace_bytes(n, H, W, stack);
  if (bytes < need) {
    set_error("sub-module training workspace too small: %zu < %zu", bytes, need);
    return WN_E_WORKSPACE;
  }
  return WN_OK;
}

int confidence_maps_train(wn_handle* h, const float* const in[4], const int64_t st[4][4], float* out_maps, int n,
                          int H, int W, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  int rc = check_submodule_args(n, H, W, kStackCmg, workspace_bytes);
  if (rc) return rc;
  TrainBuffers t;
  carve(&t, workspace, (size_t)n * H * W, kStackCmg);
  FwdOpts o;
  o.scheme = train_scheme(h);
  o.stack = kStackCmg;
  if ((rc = umma_forward_layers(h, in, st, nullptr, n, H, W, t.f, stream, o))) return rc;
  WN_CUDA(cudaMemcpyAsync(out_maps, t.f.cm, (size_t)n * 3 * H * W * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  return WN_OK;
}

int confidence_maps_backward(wn_handle* h, const float* grad_maps, float* const* grads, float* const* input_grads,
                             int n, int H, int W, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return untiled_backward(h, kStackCmg, 0, grad_maps, grads, input_grads, n, H, W, workspace, workspace_bytes,
                          stream);
}

int refine_train(wn_handle* h, int which, const float* const in[4], const int64_t st[4][4], float* out, int n, int H,
                 int W, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  int rc = check_submodule_args(n, H, W, kStackRefiners, workspace_bytes);
  if (rc) return rc;
  TrainBuffers t;
  carve(&t, workspace, (size_t)n * H * W, kStackRefiners);
  FwdOpts o;
  o.scheme = train_scheme(h);
  o.stack = kStackRefiners;
  o.refiner_l1 = true;
  if ((rc = umma_forward_layers(h, in, st, nullptr, n, H, W, t.f, stream, o))) return rc;
  const size_t img = (size_t)3 * H * W * sizeof(float);
  WN_CUDA(cudaMemcpy2DAsync(out, img, t.f.refined + (size_t)which * 3 * H * W, 3 * img, img, n,
                            cudaMemcpyDeviceToDevice, stream));
  return WN_OK;
}

int refine_backward(wn_handle* h, int which, const float* grad_out, float* const* grads, float* const* input_grads,
                    int n, int H, int W, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return untiled_backward(h, kStackRefiners, which, grad_out, grads, input_grads, n, H, W, workspace, workspace_bytes,
                          stream);
}

// ---- wn_debug_backward_layer (test aid) ---------------------------------------------------------------------------
// Buffer numbers (include/waternet_b200.h): 0 act0, 1..7 a1..a7, 8 cm, 9 r1, 10 r2, 11 refined, 12 g8, 13 gr3,
// 14 + li the output of data-gradient launch li (DgradLayer).  Which of them a stack's training pass has:
static bool debug_buffer_in_stack(int buffer, int stack) {
  if (buffer == 0 || stack == kStackAll) return true;
  const bool cmg_buffer = buffer <= 8 || buffer == kDebugG8 || (buffer >= kDebugDgrad + kD8 && buffer <= kDebugDgrad + kD2) ||
                          buffer == kDebugDgrad + kD1;
  return cmg_buffer == (stack == kStackCmg);
}

int debug_backward_layer(wn_handle* h, int stack, int which, int buffer, const float* grad_out, float* const* grads,
                         int n, int H, int W, float* dst, void* workspace, size_t workspace_bytes,
                         cudaStream_t stream) {
  int rc = check_bwd_packed(h);
  if (rc) return rc;
  if (!debug_buffer_in_stack(buffer, stack)) {
    set_error("wn_debug_backward_layer: the training pass of this stack has no buffer %d", buffer);
    return WN_E_INVALID;
  }
  TrainBuffers t;
  if ((rc = untiled_buffers(&t, stack, n, H, W, workspace, workspace_bytes))) return rc;
  const int hw = H * W;
  // the saved forward activations, as wn_forward_train or the sub-module's *_train call left them
  if (buffer < kDebugG8) {
    static constexpr int kChannels[12] = {16, 128, 128, 128, 64, 64, 64, 64, 3, 96, 96, 9};
    const int c = kChannels[buffer];
    if (buffer == 8 || buffer == 11) {
      WN_CUDA(cudaMemcpyAsync(dst, buffer == 8 ? t.f.cm : t.f.refined, (size_t)n * c * hw * sizeof(float),
                              cudaMemcpyDeviceToDevice, stream));
      return WN_OK;
    }
    const uint4* planes = buffer == 0 ? t.f.act0 : buffer <= 7 ? t.f.a[buffer] : t.f.r[buffer - 8];
    return decode_planes(h, planes, dst, c / 8, n, hw, stream);
  }
  // the seed of the stack's backward, then the backward up to the launch asked for (input gradients included)
  BwdStop stop;
  stop.buffer = buffer;
  stop.dst = dst;
  rc = backward_pass(h, grid_slots(whole_images(H, W), grad_out, nullptr, 0), stack, which, t, grads, true, false, n,
                     H, W, stream, stop);
  return rc == kBwdStopped ? WN_OK : rc;
}

// ---- windowed recompute backward (wn_backward_tiled and the sub-modules' windowed calls, DESIGN.md 4.8, 4.9, 4.11) -
// The windows of tiling.cuh, one pass of them at a time: recompute the training forward of the pass, then run the
// backward pass above on its windows as a batch, each window's output gradient taken from grad_out inside its kept
// rectangle and 0 elsewhere.  Because no pixel more than kTileHalo from a kept pixel gets a gradient, each window's
// contribution equals that of its kept pixels in the untiled backward.  The first pass writes the parameter
// gradients of the stack, every later pass writes them into a scratch copy that add_param_grads_kernel adds in (pass
// order).  Input gradients are zeroed, then folded in window order.  Workspace: [flag | scratch parameter gradients |
// (ragged: the table) | one pass of training buffers].
static void param_grad_sizes(int* size) {
  for (int c = 0; c < 8; c++) {
    size[2 * c] = kCmg[c].cout * kCmg[c].cin * kCmg[c].ks * kCmg[c].ks;
    size[2 * c + 1] = kCmg[c].cout;
  }
  for (int r = 0; r < 3; r++)
    for (int i = 0; i < 3; i++) {
      const int conv = 8 + 3 * r + i;
      size[2 * conv] = kRef[i].cout * kRef[i].cin * kRef[i].ks * kRef[i].ks;
      size[2 * conv + 1] = kRef[i].cout;
    }
}

// the stack's own entries [first, first + count) of the 34 parameter gradients
static void stack_params(int stack, int which, int* first, int* count) {
  *first = stack == kStackRefiners ? 16 + 6 * which : 0;
  *count = stack == kStackAll ? WN_NUM_PARAMS : stack == kStackCmg ? 16 : 6;
}

static size_t param_grads_bytes(int stack) {
  int size[WN_NUM_PARAMS], first, count;
  param_grad_sizes(size);
  stack_params(stack, 0, &first, &count);  // the three refiners have the same shapes
  size_t b = 0;
  for (int k = first; k < first + count; k++) b += align256((size_t)size[k] * sizeof(float));
  return b;
}

// The scratch copy of the stack's parameter gradients, from p on: dst / part are the stack's own entries, compacted
// (add_param_grads_kernel grid y = count); later is the 34-entry layout the backward writes from the second pass
// on, the own entries pointing at the scratch copy.  Returns the end of the copy.
struct ScratchGrads {
  ParamGrads dst, part;
  float* later[WN_NUM_PARAMS];
  int count;
};
static uint8_t* scratch_grads(ScratchGrads* s, uint8_t* p, float* const* grads, int stack, int which) {
  int size[WN_NUM_PARAMS], first;
  param_grad_sizes(size);
  stack_params(stack, which, &first, &s->count);
  for (int k = 0; k < WN_NUM_PARAMS; k++) s->later[k] = nullptr;
  for (int k = 0; k < s->count; k++) {
    s->dst.p[k] = grads[first + k];
    s->part.p[k] = s->later[first + k] = (float*)p;
    s->dst.size[k] = s->part.size[k] = size[first + k];
    p += align256((size_t)size[first + k] * sizeof(float));
  }
  return p;
}

// The pass loop: per pass, the training forward of the stack in the handle's training arithmetic (a refiner's first layer is kRL1, as in
// refine_train; the backward needs cm and refined, not the output), then backward_pass with the fold.  in: the
// four images of a grid call, or the per-image table of a ragged one (pack_inputs).  *exact already holds the
// exact-levels flag of the forward that produced the output (the first layer drops its a_lo pass exactly when that
// forward did).
template <class Geom, class In>
static int recompute_passes(wn_handle* h, Geom geo, const std::vector<RaggedPass>& passes, int stack, int which,
                            const In& in, int* exact, ScratchGrads& s, float* const* grads, bool want_in,
                            void* pass_ws, size_t pass_bytes, cudaStream_t stream) {
  const int64_t none[4][4] = {};
  const float* no_in[4] = {nullptr, nullptr, nullptr, nullptr};
  for (size_t pi = 0; pi < passes.size(); pi++) {
    const RaggedPass& q = passes[pi];
    int rc = stack == kStackAll ? check_train_args(q.count, q.slot_h, q.slot_w, pass_bytes)
                                : check_submodule_args(q.count, q.slot_h, q.slot_w, stack, pass_bytes);
    if (rc) return rc;
    TrainBuffers t;
    carve(&t, pass_ws, (size_t)q.count * q.slot_h * q.slot_w, stack);
    t.f.exact_flag = exact;
    FwdOpts o;
    o.scheme = train_scheme(h);
    o.packed = true;
    o.stack = stack;
    o.refiner_l1 = stack == kStackRefiners;
    geo.set_pass(q);
    o.rwin = geo.rwin();
    if ((rc = pack_inputs(h, geo, in, q.count, t.f.act0, nullptr, stream, o.scheme == kSchemeBf16))) return rc;
    if ((rc = umma_forward_layers(h, no_in, none, nullptr, q.count, q.slot_h, q.slot_w, t.f, stream, o))) return rc;
    if ((rc = backward_pass(h, geo, stack, which, t, pi == 0 ? grads : s.later, want_in, true, q.count, q.slot_h,
                            q.slot_w, stream)))
      return rc;
    if (pi > 0) {
      add_param_grads_kernel<<<dim3(64, s.count), 256, 0, stream>>>(s.dst, s.part);
      WN_LAUNCH_CHECK(h);
    }
  }
  return WN_OK;
}

static long long tiled_train_pass(const TileGeom& g, int n, long long max_pass_pixels) {
  return tile_pass_windows(g, n, max_pass_pixels ? max_pass_pixels : kTiledTrainPassPixels);
}

size_t backward_tiled_workspace_bytes(int n, int H, int W, int tile_h, int tile_w, long long max_pass_pixels) {
  const TileGeom g = tile_geom(H, W, tile_h, tile_w);
  const long long p = tiled_train_pass(g, n, max_pass_pixels);
  return 256 + param_grads_bytes(kStackAll) + train_workspace_bytes_padded((int)p, g.win_h, g.win_w) + 256;
}

// The windows of one stack's call (kTileHalo = 13 for both sub-modules too; a refiner's receptive-field radius is 6)
// once the workspace is checked.  in: the stack's four packed inputs; grad: d(out) or d(maps); input_grads: NULL or
// 4 (kStackAll, kStackCmg) / 2 (kStackRefiners) entries.  Nothing is copied from the host.
static int grid_recompute_backward(wn_handle* h, int stack, int which, const float* const in[4],
                                   const int64_t st[4][4], const float* grad, float* const* grads,
                                   float* const* input_grads, int n, int H, int W, int tile_h, int tile_w,
                                   long long max_pass_pixels, void* workspace, size_t workspace_bytes,
                                   cudaStream_t stream) {
  int rc = get_encoder();
  if (rc) return rc;
  const GridSlots geo =
      grid_slots({tile_geom(H, W, tile_h, tile_w), 0}, grad, input_grads, stack == kStackRefiners ? 2 : 4);
  const TileGeom& g = geo.tiles;
  uint8_t* base = (uint8_t*)align256((uintptr_t)workspace);
  int* exact = (int*)base;
  ScratchGrads s;
  uint8_t* pass_ws = scratch_grads(&s, base + 256, grads, stack, which);
  const size_t pass_bytes = workspace_bytes - (size_t)(pass_ws - (uint8_t*)workspace);
  bool want_in = false;
  for (int i = 0; i < 4; i++)
    if (geo.in[i]) {
      want_in = true;
      WN_CUDA(cudaMemsetAsync(geo.in[i], 0, (size_t)n * 3 * H * W * sizeof(float), stream));
    }
  const PackInArgs pa = pack_args(in, st);
  if ((rc = pack_inputs(h, whole_images(H, W), pa, n, nullptr, exact, stream))) return rc;
  const std::vector<RaggedPass> passes =
      grid_passes((long long)n * g.ny * g.nx, tiled_train_pass(g, n, max_pass_pixels), g.win_h, g.win_w);
  return recompute_passes(h, geo, passes, stack, which, pa, exact, s, grads, want_in, pass_ws, pass_bytes, stream);
}

int backward_tiled(wn_handle* h, const float* const in[4], const int64_t st[4][4], const float* grad_out,
                   float* const* grads, float* const* input_grads, int n, int H, int W, int tile_h, int tile_w,
                   long long max_pass_pixels, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  int rc = check_bwd_packed(h);
  if (rc) return rc;
  const size_t need = backward_tiled_workspace_bytes(n, H, W, tile_h, tile_w, max_pass_pixels);
  if (workspace_bytes < need) {
    set_error("tiled backward workspace too small: %zu < %zu", workspace_bytes, need);
    return WN_E_WORKSPACE;
  }
  return grid_recompute_backward(h, kStackAll, -1, in, st, grad_out, grads, input_grads, n, H, W, tile_h, tile_w,
                                 max_pass_pixels, workspace, workspace_bytes, stream);
}

size_t submodule_backward_tiled_workspace_bytes(int n, int H, int W, int tile_h, int tile_w, long long max_pass_pixels,
                                                int stack) {
  const TileGeom g = tile_geom(H, W, tile_h, tile_w);
  const long long p = tiled_train_pass(g, n, max_pass_pixels);
  return 256 + param_grads_bytes(stack) + submodule_train_workspace_bytes((int)p, g.win_h, g.win_w, stack) + 256;
}

int submodule_backward_tiled(wn_handle* h, int stack, int which, const float* const in[4], const int64_t st[4][4],
                             const float* grad, float* const* grads, float* const* input_grads, int n, int H, int W,
                             int tile_h, int tile_w, long long max_pass_pixels, void* workspace, size_t workspace_bytes,
                             cudaStream_t stream) {
  int rc = check_bwd_packed(h);
  if (rc) return rc;
  const size_t need = submodule_backward_tiled_workspace_bytes(n, H, W, tile_h, tile_w, max_pass_pixels, stack);
  if (workspace_bytes < need) {
    set_error("tiled sub-module backward workspace too small: %zu < %zu", workspace_bytes, need);
    return WN_E_WORKSPACE;
  }
  return grid_recompute_backward(h, stack, which, in, st, grad, grads, input_grads, n, H, W, tile_h, tile_w,
                                 max_pass_pixels, workspace, workspace_bytes, stream);
}

// ---- windowed recompute backward of a ragged batch (wn_backward_ragged_tiled, DESIGN.md 4.11) ---------------------
// The pass loop over the plan of ragged_plan: n images of their own sizes, cut into the windows wn_backward_tiled
// cuts each of them into, sorted by shape and packed into passes of equally sized slots.  Each pass's forward is
// that of forward_train_ragged (every ReLU layer stores zeros beyond each window's valid extent).  The table (one
// PackInArgs and one RaggedGrads per image, then the windows in plan order) sits between the scratch parameter
// gradients and the pass buffers and is copied from pageable host memory once per call.
static HostTable ragged_tiled_table(int n, size_t windows) {
  return HostTable({(size_t)n * sizeof(PackInArgs), (size_t)n * sizeof(RaggedGrads), windows * sizeof(RaggedWindow)});
}

static void ragged_tiled_plan(const int* hs, const int* ws, int n, int tile_h, int tile_w, long long max_pass_pixels,
                              std::vector<RaggedWindow>* wins, std::vector<RaggedPass>* passes) {
  ragged_plan(hs, ws, n, tile_h, tile_w, max_pass_pixels ? max_pass_pixels : kTiledTrainPassPixels, wins, passes);
}

static size_t ragged_tiled_workspace(int n, const std::vector<RaggedWindow>& wins,
                                     const std::vector<RaggedPass>& passes) {
  return 256 + param_grads_bytes(kStackAll) + ragged_tiled_table(n, wins.size()).bytes() +
         train_workspace_bytes_padded(1, 1, (int)largest_pass_pixels(passes)) + 256;
}

size_t backward_ragged_tiled_workspace_bytes(const int* hs, const int* ws, int n, int tile_h, int tile_w,
                                             long long max_pass_pixels) {
  std::vector<RaggedWindow> wins;
  std::vector<RaggedPass> passes;
  ragged_tiled_plan(hs, ws, n, tile_h, tile_w, max_pass_pixels, &wins, &passes);
  return ragged_tiled_workspace(n, wins, passes);
}

int backward_ragged_tiled(wn_handle* h, const wn_ragged_tensors* images, const float* const* grad_out,
                          float* const* grads, float* const* input_grads, int n, int tile_h, int tile_w,
                          long long max_pass_pixels, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  int rc = check_bwd_packed(h);
  if (rc) return rc;
  std::vector<int> hs, ws;
  ragged_sizes(images, n, &hs, &ws);
  std::vector<RaggedWindow> wins;
  std::vector<RaggedPass> passes;
  ragged_tiled_plan(hs.data(), ws.data(), n, tile_h, tile_w, max_pass_pixels, &wins, &passes);
  const size_t need = ragged_tiled_workspace(n, wins, passes);
  if (workspace_bytes < need) {
    set_error("ragged tiled backward workspace too small: %zu < %zu", workspace_bytes, need);
    return WN_E_WORKSPACE;
  }
  // the fold's precondition: every image's windows are contiguous in the plan, in ascending tile order
  std::vector<long long> first(n, -1);
  for (size_t p = 0; p < wins.size(); p++) {
    const int i = wins[p].img;
    if (first[i] < 0) first[i] = (long long)p;
    if (wins[p].tile != (long long)p - first[i]) {
      set_error("ragged plan: the windows of image %d are not contiguous in tile order", i);
      return WN_E_STATE;
    }
  }
  if ((rc = get_encoder())) return rc;
  uint8_t* base = (uint8_t*)align256((uintptr_t)workspace);
  int* exact = (int*)base;
  ScratchGrads s;
  uint8_t* table = scratch_grads(&s, base + 256, grads, kStackAll, -1);
  HostTable t = ragged_tiled_table(n, wins.size());
  RaggedGrads* rg = t.part<RaggedGrads>(1);
  const bool want_in = ragged_table(images, grad_out, input_grads, n, t.part<PackInArgs>(0), rg);
  for (int i = 0; i < n; i++)
    for (int t = 0; t < 4; t++)
      if (rg[i].in[t])
        WN_CUDA(cudaMemsetAsync(rg[i].in[t], 0, (size_t)3 * hs[i] * ws[i] * sizeof(float), stream));
  memcpy(t.part<RaggedWindow>(2), wins.data(), wins.size() * sizeof(RaggedWindow));
  if ((rc = t.upload(table, stream))) return rc;
  const PackInArgs* d_imgs = t.dev<PackInArgs>(table, 0);
  TableSlots geo = {{t.dev<RaggedWindow>(table, 2), 0, 0, 0, tile_h, tile_w}, t.dev<RaggedGrads>(table, 1), nullptr};
  uint8_t* pass_ws = table + t.bytes();
  const size_t pass_bytes = workspace_bytes - (size_t)(pass_ws - (uint8_t*)workspace);
  // the exact-levels flag over every pass, as wn_forward_ragged takes it
  WN_CUDA(cudaMemsetAsync(exact, 1, sizeof(int), stream));  // nonzero = "all inputs are 8-bit levels"
  for (const RaggedPass& q : passes) {
    geo.set_pass(q);
    if ((rc = pack_inputs(h, geo, d_imgs, q.count, nullptr, exact, stream))) return rc;
  }
  return recompute_passes(h, geo, passes, kStackAll, -1, d_imgs, exact, s, grads, want_in, pass_ws, pass_bytes,
                          stream);
}

}  // namespace wn
