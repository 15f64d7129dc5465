// Tensor-core path of WaterNet.forward (WN_MODE_BF16X3, WN_MODE_BF16_FP8): wgmma implicit-GEMM convolutions.
//
// Replaces the reference's waternet/net.py:45-56, :75-80, :99-108.  Every
// convolution is a dense contraction (SURVEY.md 2.1), so it runs on the tensor
// cores -- but the 1e-3 parity bar rules out single-pass bf16/tf32 operands
// (SURVEY.md section 0).  Each fp32 operand is split into bf16 hi + lo and
// hi*hi + lo*w + hi*w_lo accumulates in fp32 registers: as three bf16 MMAs ("bf16x3",
// ~2^-16 relative operand error), or -- the default for the tensor-bound layers -- as
// one bf16 MMA plus ONE fp8 (e4m3) MMA of K = 32 for both correction terms, all of a tile's e4m3 MMAs first, into
// the one accumulator (UmmaCfg FMT in umma_conv.cuh; DESIGN.md 4.2).
//
// Data layout in HBM: activations are bf16 planes of 8 channels,
//     act[n][plane][y][x][8]   planes [0, C/8) = hi parts, [C/8, 2C/8) = lo parts,
// so that ONE 5-D TMA box (8 ch, x, y, planes, n) drops a halo tile into shared
// memory as [plane][y][x][16 B] -- exactly the no-swizzle K-major wgmma operand
// layout with "8 consecutive pixels of a row" as the 8x16B core matrix.  A filter
// tap (ky,kx) is then just a different descriptor start address into the SAME halo
// tile: the activations are read from L2/HBM once per tile, not once per tap, and
// out-of-image pixels come back as zeros from the TMA (padding="same").
//
// One persistent CTA per SM, warp-specialised:
//   warps 0-7  two consumer warpgroups (kSpecs wgs 2; wgs 3: warps 0-11, three): each issues the m64 wgmmas of its
//              8 rows of the 8x16-, 16x16-, 8x24- or 16x24-pixel tile (accumulators in registers; kSpecs mw, ng) and then
//              runs the epilogue of those pixels
//              (registers -> shared-memory transpose -> bias/act -> bf16 hi/lo planes or fp32)
//   warp 8     A producer (TMA halo tiles, one 16-channel chunk per stage); wgs 3: warp 12
//   warp 9     B producer (bulk copies of pre-packed weight stages, 1-9 taps of a chunk per stage); wgs 3: warp 13
#include <type_traits>

#include "umma_conv.cuh"

namespace wn {

// torch.cat([x, wb, ce, gc], 1) (net.py:46) -> act planes: 16 channels (12 + 4 zero), bf16 hi/lo of
// v*255.  Inputs that came from 8-bit images (arr2ten: u/255) give integers 0..255, exact in the
// 8-bit bf16 significand: then lo == 0 and the first layer can drop its a_lo pass (flag stays set).
// v[3t + c] = input t, channel c at (n, y, x), times 255; false unless all twelve are 8-bit levels
__device__ __forceinline__ bool pack_pixel(const PackInArgs& a, int n, int y, int x, float* v) {
  bool exact = true;
#pragma unroll
  for (int t = 0; t < 4; t++)
#pragma unroll
    for (int c = 0; c < 3; c++) {
      float f = __fmul_rn(a.p[t][n * a.s[t][0] + c * a.s[t][1] + y * a.s[t][2] + x * a.s[t][3]], 255.0f);
      float r = rintf(f);
      // (u/255)*255 lands within ~2e-5 of u; anything within 2^-14 of a level is treated as that level
      if (fabsf(f - r) <= 6.103515625e-5f && r >= 0.f && r <= 255.f) f = r; else exact = false;
      v[t * 3 + c] = f;
    }
  return exact;
}
// 16 channels -> the four operand planes hi0, hi1, lo0, lo1 of pixel o[0] (planes hw apart); HI: lo = 0
template <bool HI>
__device__ __forceinline__ void store_packed(uint4* o, int hw, float* v) {
  v[12] = v[13] = v[14] = v[15] = 0.f;
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
  o[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  o[hw] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
  o[2 * (size_t)hw] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  o[3 * (size_t)hw] = make_uint4(lo[4], lo[5], lo[6], lo[7]);
}
// The operands of one slot pixel: a grid geometry reads image p.img of one set of four tensors, a table geometry the
// tensors of image p.img (one PackInArgs per image, read through its strides with 64-bit offsets)
__device__ __forceinline__ bool pack_slot_pixel(const PackInArgs& a, const SlotPixel& p, float* v) {
  return pack_pixel(a, p.img, p.y, p.x, v);
}
__device__ __forceinline__ bool pack_slot_pixel(const PackInArgs* __restrict__ imgs, const SlotPixel& p, float* v) {
  return pack_pixel(imgs[p.img], 0, p.y, p.x, v);
}

// Slot pixel blockIdx.x * 256 + tid of slot blockIdx.y of geo (tiling.cuh), read at image coordinates.  PLANES: the
// slot's act0 planes (zeros beyond the valid extent).  FLAG: *exact_flag is cleared unless every valid pixel is an
// 8-bit level.  Whole images (GridGeom tile = image size) take both in one launch; the windowed calls take the flag
// once per call over whole images (or over every pass of a ragged plan) and then the planes per pass.  HI: the planes
// of the single-pass bf16 training forward, lo = 0.  SLOT: the flag is one per slot, exact_flag[blockIdx.y].
template <class Geom, class In, bool PLANES, bool FLAG, bool HI = false, bool SLOT = false>
__global__ void __launch_bounds__(256)
pack_inputs_kernel(Geom geo, In in, uint4* __restrict__ out, int* __restrict__ exact_flag) {
  const int pix = blockIdx.x * 256 + threadIdx.x;
  const int hw = geo.slot_hw();
  bool exact = true;
  if (pix < hw) {
    const SlotPixel p = geo.at(blockIdx.y, pix);
    float v[16];
#pragma unroll
    for (int j = 0; j < 12; j++) v[j] = 0.f;
    if (p.valid) exact = pack_slot_pixel(in, p, v);
    if constexpr (PLANES) store_packed<HI>(out + (size_t)blockIdx.y * 4 * hw + pix, hw, v);
  }
  if constexpr (FLAG)
    if (!__syncthreads_and(exact) && threadIdx.x == 0) atomicExch(exact_flag + (SLOT ? blockIdx.y : 0), 0);
}

// reset: *flag is set to 1 ("all inputs are 8-bit levels") first, inside the packing's timing slot
template <bool PLANES, bool FLAG, class Geom, class In>
static int launch_pack(wn_handle* h, const Geom& geo, const In& in, int count, uint4* act0, int* flag, bool reset,
                       cudaStream_t stream, bool hi = false) {
  TimedScope ts(h, kSlotPack, stream);
  if (reset) WN_CUDA(cudaMemsetAsync(flag, 1, sizeof(int), stream));
  const dim3 grid((unsigned)(((size_t)geo.slot_hw() + 255) / 256), count);
  if (PLANES && hi)
    pack_inputs_kernel<Geom, In, PLANES, FLAG, true><<<grid, 256, 0, stream>>>(geo, in, act0, flag);
  else
    pack_inputs_kernel<Geom, In, PLANES, FLAG><<<grid, 256, 0, stream>>>(geo, in, act0, flag);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}
int pack_inputs(wn_handle* h, const GridGeom& geo, const PackInArgs& in, int count, uint4* act0, int* flag,
                cudaStream_t stream, bool hi) {
  if (!act0) return launch_pack<false, true>(h, geo, in, count, nullptr, flag, true, stream);
  if (flag) return launch_pack<true, true>(h, geo, in, count, act0, flag, true, stream, hi);
  return launch_pack<true, false>(h, geo, in, count, act0, nullptr, false, stream, hi);
}
// a ragged call takes its flag over every pass before the first, so it never asks for both in one launch, and the
// caller sets the flag once before the first of those launches.  slot_flags (fp8-correction scheme): with the planes,
// one flag per slot, set to 1 here and cleared unless the slot holds 8-bit levels only
int pack_inputs(wn_handle* h, const TableGeom& geo, const PackInArgs* imgs, int count, uint4* act0, int* flag,
                cudaStream_t stream, bool hi, int* slot_flags) {
  if (!act0) return launch_pack<false, true>(h, geo, imgs, count, nullptr, flag, false, stream);
  if (slot_flags) {
    TimedScope ts(h, kSlotPack, stream);
    WN_CUDA(cudaMemsetAsync(slot_flags, 1, (size_t)count * sizeof(int), stream));
    const dim3 grid((unsigned)(((size_t)geo.slot_hw() + 255) / 256), count);
    pack_inputs_kernel<TableGeom, const PackInArgs*, true, true, false, true><<<grid, 256, 0, stream>>>(geo, imgs, act0,
                                                                                                      slot_flags);
    WN_LAUNCH_CHECK(h);
    return WN_OK;
  }
  return launch_pack<true, false>(h, geo, imgs, count, act0, nullptr, false, stream, hi);
}

// Sub-modules of the tiled forward: slot blockIdx.y of geo holds `cs` fp32 planes; channels [c0, c0 + c) of its kept
// rectangle are stored into dst, contiguous NCHW (N, c, H, W), at image coordinates.
__global__ void __launch_bounds__(256) store_kept_kernel(const float* __restrict__ src, int cs, int c0, int c,
                                                         float* __restrict__ dst, GridGeom geo) {
  const int pix = blockIdx.x * 256 + threadIdx.x;
  const int hw = geo.slot_hw();
  if (pix >= hw) return;
  const SlotPixel p = geo.at(blockIdx.y, pix);
  if (!p.kept) return;
  const float* s = src + ((size_t)blockIdx.y * cs + c0) * hw + pix;
  float* d = dst + (size_t)p.img * c * p.ihw + p.o;
  for (int k = 0; k < c; k++) d[k * p.ihw] = s[(size_t)k * hw];
}

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
// The ten tensor-core launches of one forward (fused layer list).
enum UmmaLayer {
  kL1 = 0,    // cmg.conv1 (12->128) + the three refiner conv1 (6->32 each): 16 -> 224, 7x7
  kC2, kC3, kC4, kC5, kC6, kC7,
  kC8,        // 64 -> 3 (pad 16), sigmoid
  kR2,        // three refiner conv2 as one block-diagonal 96 -> 96, 5x5
  kR3,        // three refiner conv3 as block-diagonal 96 -> 9 (pad 16), ReLU, gated sum
  kRL1,       // the three refiner conv1 alone (16 -> 96, 7x7): the training forward of a refiner
  kNumUmmaLayers
};
// Everything a layer's launches and packed weights depend on (UmmaCfg in umma_conv.cuh).  npad = output columns
// per diagonal block; concat = CONCAT of the bf16x3 form, set where the a_hi x [w_hi | w_lo] product fits one wgmma
// (N = 2 * NPAD <= 256); slot = timing slot, the state-dict index of the layer's (first) convolution; f8 = the layer
// has an fp8-correction form (UmmaCfg FMT bit 0, the tensor-bound layers), which uses CONCAT 0.  mw = m64 blocks per
// warpgroup (2: 16-pixel-wide tiles, which halve the weight bytes streamed per pixel) and ng = column groups of npad /
// ng channels each (UmmaCfg MW, NG): at mw = 2 the accumulators of both blocks must fit in 128 registers per thread
// in every form (R2's bf16x3 form, CONCAT over three blocks, holds 96 per block).
// wgs = consumer warpgroups (UmmaCfg WGS): 3 gives 24-row tiles, which cut the weight bytes streamed per pixel by a
// third; a layer takes it where its kernels stay free of spills at 160 registers and measure faster.
// Every layer also has a single-pass bf16 form (UmmaCfg FMT kFmtHi, the WN_MODE_BF16 training forward, kRL1 included):
// the bf16x3 weight images, hi rows only, at the layer's own mw, ng and wgs.  It needs no more registers than the
// bf16x3 form (a CONCAT layer's accumulators halve: N = npad instead of 2 * npad).
struct UmmaLayerSpec {
  int ks, cinpad, npad, epi, concat, nblk, tps, slot;
  bool f8;
  int mw, ng, wgs;
};
static constexpr UmmaLayerSpec kSpecs[kNumUmmaLayers] = {
    // ks cinpad npad epi       concat nblk tps slot f8  mw ng wgs
    {7, 16, 224, kEpiAct, 0, 1, 1, 0, false, 1, 1, 2},     // kL1
    {5, 128, 128, kEpiAct, 0, 1, 5, 1, true, 1, 1, 3},     // kC2
    {3, 128, 128, kEpiAct, 0, 1, 3, 2, true, 1, 1, 3},     // kC3
    {1, 128, 64, kEpiAct, 1, 1, 1, 3, false, 1, 1, 3},     // kC4
    {7, 64, 64, kEpiAct, 1, 1, 7, 4, true, 2, 1, 2},       // kC5
    {5, 64, 64, kEpiAct, 1, 1, 5, 5, true, 2, 1, 3},       // kC6
    {3, 64, 64, kEpiAct, 1, 1, 9, 6, true, 2, 1, 3},       // kC7
    {3, 64, 16, kEpiSigmoid, 1, 1, 9, 7, false, 1, 1, 3},  // kC8
    {5, 96, 32, kEpiAct, 1, 3, 5, 9, true, 1, 1, 3},       // kR2
    {3, 96, 16, kEpiGate, 1, 1, 9, 10, false, 1, 1, 3},    // kR3
    {7, 16, 96, kEpiAct, 0, 1, 1, 8, false, 1, 1, 3}};     // kRL1 (CONCAT 0 as kL1: the same sums per channel)
// WN_UMMA_WGS2 builds every layer with two consumer warpgroups (16-row tiles), for A/B runs against the table
#ifdef WN_UMMA_WGS2
static constexpr int layer_wgs(int) { return 2; }
#else
static constexpr int layer_wgs(int li) { return kSpecs[li].wgs; }
#endif

// The first layer's fp8-correction form is its tap-pair form (UmmaCfg kFmtPair8): one e4m3 wgmma for the w_lo
// corrections of two taps, for 8-bit-level inputs; other inputs run its bf16x3 form in the same launch.
static constexpr bool pairs_taps(int li) { return li == kL1; }
static constexpr size_t kPairImageBytes = (size_t)((49 + 1) / 2 + 49) * 224 * 32;  // kL1's tap-pair weight image
static constexpr size_t kPairScaleBytes = 2 * 224 * sizeof(float);                // s_c, then 2^-9 / s_c

// In the fp8-correction scheme a layer writes the hi + fp8-planes format (FMT bit 1) when its consumers read it with
// their fp8 form.  L1 feeds C2 and R2; every other layer feeds the next one, except the last layer of each stack.
static_assert(kSpecs[kC2].f8 == kSpecs[kR2].f8, "L1 writes one format for both of its consumers");
static constexpr bool writes_f8(int li) { return li < kR3 && li != kC8 && kSpecs[li + 1].f8; }

// out -> every peer address (the uint8 output of the last launch, the range guard's re-run -- then conditional on
// *run_if like every launch of that chain)
static __global__ void __launch_bounds__(256)
mirror_u8_kernel(const uint8_t* __restrict__ src, PeerOut peers, size_t bytes, const int* __restrict__ run_if) {
  if (run_if && *run_if == 0) return;
  const size_t stride = (size_t)gridDim.x * blockDim.x, i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
#pragma unroll
  for (int k = 0; k < WN_MAX_PEERS; k++) {
    if (k >= peers.n) continue;
    uint8_t* dst = peers.p[k];
    // 16-byte copies where source and destination allow it (the batches of a 16-byte aligned buffer); bytes otherwise
    const size_t vecs = (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0) ? bytes / 16 : 0;
    for (size_t i = i0; i < vecs; i += stride) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
    for (size_t i = vecs * 16 + i0; i < bytes; i += stride) dst[i] = src[i];
  }
}
int mirror_u8(wn_handle* h, const uint8_t* src, const PeerOut& peers, size_t bytes, const int* run_if, cudaStream_t stream) {
  if (peers.n <= 0 || bytes == 0) return WN_OK;
  mirror_u8_kernel<<<4 * h->sm_count, 256, 0, stream>>>(src, peers, bytes, run_if);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

struct UmmaWeights {
  uint8_t* stages8[kNumUmmaLayers];  // fp8-correction weight images (layers with an fp8 form; kL1: tap pairs)
  float* scale8[kNumUmmaLayers];     // {ws, 2^-9 / ws, max|w|, -}; kL1: per-column scales (pair_scale_kernel)
  int* overflow_dev;                 // sticky: an activation left the e4m3 range in the fp8-correction mode
  int* overflow_host;                // pinned mirror, refreshed at the end of every forward of that mode
  unsigned* live_dev;                // per launch: the low-end record of its fp8 planes (ConvArgs::f8_live)
  uint8_t* stages[kNumUmmaLayers];
  float* bias[kNumUmmaLayers];
  float* dense;  // scratch for packing
};

// one block's rows per (chunk, tap): 64 B per output channel in the bf16x3 and the fp8-correction layouts alike
static size_t stage_bytes_total(const UmmaLayerSpec& s) { return (size_t)(s.cinpad / 16) * s.ks * s.ks * s.npad * 64; }

int umma_pack_weights(wn_handle* h, const float* const* params, cudaStream_t stream) {
  if (!h->umma) h->umma = (UmmaWeights*)calloc(1, sizeof(UmmaWeights));
  for (int i = 0; i < kNumUmmaLayers; i++) {  // (re)allocate whatever an earlier, failed call left unallocated
    if (!h->umma->stages[i]) WN_CUDA(cudaMalloc(&h->umma->stages[i], stage_bytes_total(kSpecs[i])));
    if (!h->umma->bias[i]) WN_CUDA(cudaMalloc(&h->umma->bias[i], kSpecs[i].npad * kSpecs[i].nblk * sizeof(float)));
    if (kSpecs[i].f8 || pairs_taps(i)) {
      const size_t img = pairs_taps(i) ? kPairImageBytes : stage_bytes_total(kSpecs[i]);
      if (!h->umma->stages8[i]) WN_CUDA(cudaMalloc(&h->umma->stages8[i], img));
      const size_t sc = pairs_taps(i) ? kPairScaleBytes : 4 * sizeof(float);
      if (!h->umma->scale8[i]) WN_CUDA(cudaMalloc(&h->umma->scale8[i], sc));
    }
  }
  if (!h->umma->dense) WN_CUDA(cudaMalloc(&h->umma->dense, (size_t)224 * 128 * 49 * sizeof(float)));
  if (!h->umma->overflow_dev) WN_CUDA(cudaMalloc(&h->umma->overflow_dev, sizeof(int)));
  if (!h->umma->overflow_host) WN_CUDA(cudaHostAlloc(&h->umma->overflow_host, sizeof(int), cudaHostAllocDefault));
  if (!h->umma->live_dev) WN_CUDA(cudaMalloc(&h->umma->live_dev, kNumUmmaLayers * sizeof(unsigned)));
  UmmaWeights* u = h->umma;
  *u->overflow_host = 0;  // new weights: the fp8-correction mode gets a fresh chance
  WN_CUDA(cudaMemsetAsync(u->overflow_dev, 0, sizeof(int), stream));
  WN_CUDA(cudaMemsetAsync(u->live_dev, 0, kNumUmmaLayers * sizeof(unsigned), stream));
  auto W = [&](int conv) { return params[2 * conv]; };
  auto B = [&](int conv) { return params[2 * conv + 1]; };
  for (int li = 0; li < kNumUmmaLayers; li++) {
    const UmmaLayerSpec& s = kSpecs[li];
    const int kk = s.ks * s.ks;
    const int rows = s.npad * s.nblk;
    WN_CUDA(cudaMemsetAsync(u->dense, 0, (size_t)rows * s.cinpad * kk * sizeof(float), stream));
    WN_CUDA(cudaMemsetAsync(u->bias[li], 0, rows * sizeof(float), stream));
    auto scatter = [&](int conv, int co, int ci, int row_off, int split, int base0, int base1) -> int {
      // the first layer consumes image levels 0..255 (see pack_inputs_kernel): fold the /255 into its weights
      scatter_weights_kernel<<<128, 256, 0, stream>>>(W(conv), u->dense, co, ci, kk, s.cinpad, row_off, split,
                                                      base0, base1, li == kL1 || li == kRL1 ? 255.0f : 1.0f);
      WN_LAUNCH_CHECK(h);
      scatter_bias_kernel<<<1, 256, 0, stream>>>(B(conv), u->bias[li], co, row_off);
      WN_LAUNCH_CHECK(h);
      return WN_OK;
    };
    int rc = WN_OK;
    if (li == kL1) {
      rc = scatter(0, 128, 12, 0, 12, 0, 0);
      for (int r = 0; r < 3 && !rc; r++)  // refiner r sees cat[x, input r+1]: channels 0..2 and 3(r+1)..3(r+1)+2
        rc = scatter(8 + 3 * r, 32, 6, 128 + 32 * r, 3, 0, 3 * (r + 1));
    } else if (li >= kC2 && li <= kC8) {
      const int conv = li;  // cmg.conv2..conv8 are convs 1..7
      const LayerDesc& d = kCmg[conv];
      rc = scatter(conv, d.cout, d.cin, 0, d.cin, 0, 0);
    } else if (li == kR2) {
      for (int r = 0; r < 3 && !rc; r++) rc = scatter(8 + 3 * r + 1, 32, 32, 32 * r, 32, 32 * r, 0);
    } else if (li == kRL1) {  // kL1's refiner rows, from row 0
      for (int r = 0; r < 3 && !rc; r++) rc = scatter(8 + 3 * r, 32, 6, 32 * r, 3, 0, 3 * (r + 1));
    } else {
      for (int r = 0; r < 3 && !rc; r++) rc = scatter(8 + 3 * r + 2, 3, 32, 3 * r, 32, 32 * r, 0);
    }
    if (rc) return rc;
    // each column group's stages are contiguous: group g holds dense rows [g * gw, (g + 1) * gw)
    const int gw = s.npad / s.ng;
    const size_t group_bytes = stage_bytes_total(s) / s.ng;
    for (int g = 0; g < s.ng; g++) {
      pack_stages_kernel<<<256, 256, 0, stream>>>(u->dense, (__nv_bfloat16*)(u->stages[li] + g * group_bytes), gw,
                                                  s.cinpad, kk, s.concat, s.nblk, g * gw);
      WN_LAUNCH_CHECK(h);
    }
    if (pairs_taps(li)) {
      static_assert(kSpecs[kL1].cinpad == 16 && kSpecs[kL1].ng == 1 && kSpecs[kL1].nblk == 1 && kSpecs[kL1].npad == 224 &&
                    kSpecs[kL1].ks == 7, "kPairImageBytes");
      pair_scale_kernel<<<s.npad, 256, 0, stream>>>(u->dense, u->scale8[li], s.npad, s.cinpad * kk);
      WN_LAUNCH_CHECK(h);
      pack_stages_pair_kernel<<<64, 256, 0, stream>>>(u->dense, u->stages8[li], u->scale8[li], s.npad, kk);
      WN_LAUNCH_CHECK(h);
    }
    if (s.f8) {
      WN_CUDA(cudaMemsetAsync(u->scale8[li], 0, 4 * sizeof(float), stream));
      f8_absmax_kernel<<<64, 256, 0, stream>>>(u->dense, (size_t)rows * s.cinpad * kk, u->scale8[li]);
      WN_LAUNCH_CHECK(h);
      f8_scale_finish_kernel<<<1, 1, 0, stream>>>(u->scale8[li]);
      WN_LAUNCH_CHECK(h);
      for (int g = 0; g < s.ng; g++) {
        pack_stages_f8_kernel<<<256, 256, 0, stream>>>(u->dense, u->stages8[li] + g * group_bytes, u->scale8[li], gw,
                                                       s.cinpad, kk, s.tps, s.nblk, g * gw);
        WN_LAUNCH_CHECK(h);
      }
    }
  }
  return WN_OK;
}

void umma_free(wn_handle* h) {
  if (!h->umma) return;
  for (int i = 0; i < kNumUmmaLayers; i++) {
    if (h->umma->stages[i]) cudaFree(h->umma->stages[i]);
    if (h->umma->bias[i]) cudaFree(h->umma->bias[i]);
    if (h->umma->stages8[i]) cudaFree(h->umma->stages8[i]);
    if (h->umma->scale8[i]) cudaFree(h->umma->scale8[i]);
  }
  if (h->umma->dense) cudaFree(h->umma->dense);
  if (h->umma->overflow_dev) cudaFree(h->umma->overflow_dev);
  if (h->umma->overflow_host) cudaFreeHost(h->umma->overflow_host);
  if (h->umma->live_dev) cudaFree(h->umma->live_dev);
  free(h->umma);
  h->umma = nullptr;
}

// bytes per pixel: act0 (16 ch) 64 | cmg ping/pong (128 ch) 512 each | ref ping/pong (96 ch) 384 each | cm 12
static constexpr size_t kUmmaBytesPerPixel = 64 + 512 + 512 + 384 + 384 + 12;

// Images per pass: <= 8 Mi pixels (~15 GB of workspace) by default; wn_set_chunk_pixels lowers the cap
// (tests force the multi-pass path on small batches with it; it never raises the workspace need).
static constexpr long long kDefaultChunkPixels = 8ll << 20;
static int umma_chunk(long long cap, int n, int h, int w) {
  if (cap <= 0 || cap > kDefaultChunkPixels) cap = kDefaultChunkPixels;
  long long per = (long long)h * w;
  long long nb = cap / (per > 0 ? per : 1);
  if (nb < 1) nb = 1;
  return nb < n ? (int)nb : n;
}
int umma_chunk_images(const wn_handle* h, int n, int height, int width) {
  return umma_chunk(h ? h->chunk_pixels : 0, n, height, width);
}

size_t umma_forward_workspace_bytes(int n, int h, int w) {
  const size_t nb = (size_t)umma_chunk(0, n, h, w);
  return nb * h * w * kUmmaBytesPerPixel + nb * h * 64 + 4096;
}

// Launch layer LI in `scheme` (FwdOpts): the fp8-correction scheme (1), single-pass bf16 (kSchemeBf16) or bf16x3 (0).
// A layer's fp8 form reads its own weight images, in the [hi | fp8] layout; the single-pass form reads the hi rows of
// the bf16x3 images.  A pass of a ragged batch (a.rwin) runs the RAG instantiations of the layers that mask (kEpiAct)
// or store per window (kEpiGate); the confidence maps are per pixel and need neither.
// FUSE (inference, fp8-correction and bf16x3 schemes): layer LI + 1, a 1x1 layer, runs in LI's epilogue (UmmaCfg
// kFmtFuse1x1) from its bf16x3 weight image; the launch writes LI + 1's output in LI + 1's format, in LI's timing slot.
template <int LI, bool RAG, bool FUSE = false>
static int launch_layer_as(wn_handle* h, int scheme, void* in_base, ConvArgs a, cudaStream_t stream) {
  constexpr UmmaLayerSpec s = kSpecs[LI];
  constexpr bool R = RAG && s.epi != kEpiSigmoid;
  const UmmaWeights* u = h->umma;
  constexpr int GW = s.npad / s.ng;  // channels per column group
  constexpr int FZ = FUSE ? kFmtFuse1x1 : 0;
  constexpr int OUT_LI = FUSE ? LI + 1 : LI;  // the layer whose output the launch stores
  if constexpr (FUSE) {
    constexpr UmmaLayerSpec f = kSpecs[LI + 1];
    static_assert(f.ks == 1 && f.cinpad == s.npad && f.npad == kFuseNpad && f.concat && f.nblk == 1 && !f.f8 &&
                  f.epi == kEpiAct && s.epi == kEpiAct, "the fused layer: 1x1, CONCAT, bf16x3 weights, activation");
    a.wpk1x1 = u->stages[LI + 1];
    a.bias1x1 = u->bias[LI + 1];
    if (scheme == kSchemeBf16) {
      set_error("the fused 1x1 layer runs in the inference schemes only");
      return WN_E_STATE;
    }
  } else if (scheme == kSchemeBf16) {
    return launch_conv<s.ks, s.cinpad, GW, s.epi, s.concat, s.nblk, s.tps, kFmtHi, R, s.mw, s.ng, layer_wgs(LI)>(
        h, s.slot, u->stages[LI], u->bias[LI], in_base, a, stream);
  }
  if (scheme == 1) {
    constexpr int FMT =
        (s.f8 ? kFmtIn8 : 0) | (writes_f8(OUT_LI) ? kFmtOut8 : 0) | (pairs_taps(LI) ? kFmtPair8 : 0) | FZ;
    if constexpr ((FMT & kFmtOut8) != 0) {
      a.f8_overflow = u->overflow_dev;
      a.f8_live = u->live_dev + OUT_LI;
    }
    if constexpr (s.f8) {
      a.f8_scale = u->scale8[LI] + 1;
      // the planes it reads: L1's refiner blocks for R2, its cmg block for C2, else the launch before (C4: also
      // when it runs in C3's epilogue)
      a.f8_overflow = u->overflow_dev;
      a.f8_live_in = u->live_dev + (LI == kR2 ? kL1 : LI - 1);
      a.f8_live_need = LI == kR2 ? 0x54u : 0x1u;
    }
    if constexpr (pairs_taps(LI)) {
      a.f8_scale = u->scale8[LI] + s.npad;
      a.wpk8 = u->stages8[LI];
    }
    return launch_conv<s.ks, s.cinpad, GW, s.epi, (s.f8 ? 0 : s.concat), s.nblk, s.tps, FMT, R, s.mw, s.ng,
                       layer_wgs(LI)>(h, s.slot, s.f8 ? u->stages8[LI] : u->stages[LI], u->bias[LI], in_base, a, stream);
  }
  return launch_conv<s.ks, s.cinpad, GW, s.epi, s.concat, s.nblk, s.tps, FZ, R, s.mw, s.ng, layer_wgs(LI)>(
      h, s.slot, u->stages[LI], u->bias[LI], in_base, a, stream);
}
template <int LI, bool FUSE = false>
static int launch_layer(wn_handle* h, int scheme, void* in_base, ConvArgs a, cudaStream_t stream) {
  return a.rwin ? launch_layer_as<LI, true, FUSE>(h, scheme, in_base, a, stream)
                : launch_layer_as<LI, false, FUSE>(h, scheme, in_base, a, stream);
}
// WN_UMMA_UNFUSED_C4 runs cmg.conv4 as a launch of its own in every forward, for A/B runs against the fused form
#ifdef WN_UMMA_UNFUSED_C4
static constexpr bool kFuseC4 = false;
#else
static constexpr bool kFuseC4 = true;
#endif

// bf16 hi/lo planes -> fp32 NCHW (test aid)
__global__ void decode_planes_kernel(const uint4* __restrict__ src, float* __restrict__ dst, int planes_half, int hw,
                                     int f8) {
  const int n = blockIdx.z, plane = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= hw) return;
  const uint4 h4 = src[((size_t)n * 2 * planes_half + plane) * hw + pix];
  if (f8) {  // hi planes + per 16 channels {e4m3((v - hi) * 2^9), e4m3(v)}: v ~ hi + lo8 / 512
    const uint4 l4 = src[((size_t)n * 2 * planes_half + planes_half + 2 * (plane >> 1)) * hw + pix];
    const uint32_t hs[4] = {h4.x, h4.y, h4.z, h4.w}, ls[4] = {l4.x, l4.y, l4.z, l4.w};
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const float hi = __uint_as_float(((hs[j >> 1] >> ((j & 1) * 16)) & 0xffffu) << 16);
      const int byte = (plane & 1) * 8 + j;
      const uint32_t b8 = (ls[byte >> 2] >> ((byte & 3) * 8)) & 0xffu;  // e4m3: sign, 4 exponent bits (bias 7), 3 mantissa
      const int e = (int)((b8 >> 3) & 15), m = (int)(b8 & 7);
      const float mag = e == 0 ? ldexpf((float)m, -9) : ldexpf((float)(8 + m), e - 10);
      const float lo = ((b8 & 0x80u) ? -mag : mag) * (1.f / 512.f);
      dst[((size_t)n * planes_half * 8 + plane * 8 + j) * hw + pix] = hi + lo;
    }
    return;
  }
  const uint4 l4 = src[((size_t)n * 2 * planes_half + planes_half + plane) * hw + pix];
  const uint32_t hs[4] = {h4.x, h4.y, h4.z, h4.w}, ls[4] = {l4.x, l4.y, l4.z, l4.w};
#pragma unroll
  for (int j = 0; j < 8; j++) {
    float hi = __uint_as_float(((hs[j >> 1] >> ((j & 1) * 16)) & 0xffffu) << 16);
    float lo = __uint_as_float(((ls[j >> 1] >> ((j & 1) * 16)) & 0xffffu) << 16);
    dst[((size_t)n * planes_half * 8 + plane * 8 + j) * hw + pix] = hi + lo;
  }
}

int decode_planes(wn_handle* h, const uint4* src, float* dst, int planes_half, int n, int hw, cudaStream_t stream) {
  decode_planes_kernel<<<dim3((hw + 255) / 256, planes_half, n), 256, 0, stream>>>(src, dst, planes_half, hw, 0);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

// Where every layer's output lives.  Inference ping-pongs two buffers per stack; the training
// forward (conv_bwd.cu) gives every activation its own buffer because the backward pass needs them.
int umma_forward_layers(wn_handle* h, const float* const in[4], const int64_t st[4][4], float* out, int n, int H,
                        int W, const FwdBuffers& b, cudaStream_t stream, const FwdOpts& o) {
  const int dbg_layer = o.dbg_layer;
  float* const dbg_dst = o.dbg_dst;
  if (!o.packed) {
    const int rc = pack_inputs(h, whole_images(H, W), pack_args(in, st), n, b.act0, b.exact_flag, stream,
                               o.scheme == kSchemeBf16);
    if (rc) return rc;
  }
  ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.N = n; a.H = H; a.W = W;
  a.run_if = o.run_if;
  a.rwin = o.rwin;
  a.f8_live_clear = ~0u;
  int rc;
  // fp8-correction scheme (inference): the tensor-bound layers replace the two bf16 correction passes by one
  // fp8 MMA (UmmaCfg FMT); a layer whose consumer is such a layer writes the hi + fp8-planes format
  const bool f8 = o.scheme == 1;
  const int sc = o.scheme;
  // after layer li's launch: decode its output (a.dst0) when it is the one wn_debug_forward_layer asks for.  That
  // call numbers an output by its convolution in state-dict order, the layer's timing slot; L1's second output
  // (a.dst1) is the refiners' conv1, number 8.
  auto dump = [&](int li) -> bool {
    const bool second = li == kL1 && dbg_layer == 8;
    if (dbg_layer != kSpecs[li].slot && !second) return false;
    const ActDst& d = second ? a.dst1 : a.dst0;
    decode_planes_kernel<<<dim3((H * W + 255) / 256, d.planes_half, n), 256, 0, stream>>>(d.base, dbg_dst, d.planes_half,
                                                                                      H * W, f8 && writes_f8(li));
    h->launches++;
    return true;
  };
  auto act = [&](uint4* d0, int c0, uint4* d1, int c1) {
    a.dst0.base = d0; a.dst0.planes_half = c0 / 8;
    a.dst1.base = d1; a.dst1.planes_half = c1 / 8;
    a.split_c = c0; a.cout = c0 + c1;
  };
  // the last launch: refiner conv3 + ReLU, then (when the maps are given) the gated sum -> fp32 NCHW and/or
  // ten2arr'd uint8 NHWC; refined_out optionally receives the three refined images
  auto last = [&]() {
    a.out_f32 = out;
    a.out_u8 = o.out_u8;
    a.cm = o.stack == kStackRefiners ? nullptr : b.cm;
    a.refined_out = b.refined;
    if (o.tiles) {
      a.tiled = 1;
      a.tiles = *o.tiles;
      a.win0 = o.win0;
    }
  };
  const bool want_cmg = o.stack != kStackRefiners, want_ref = o.stack != kStackCmg;
  a.skip_lo = b.exact_flag;
  a.a_hi_only = o.hi_only ? 1 : 0;
  a.slot_levels = o.slot_levels;
  if (o.refiner_l1) {  // the refiners' conv1 alone, bf16x3 or single-pass bf16 (the sums of kL1's refiner columns)
    constexpr UmmaLayerSpec s = kSpecs[kRL1];
    act(b.r[1], 96, nullptr, 0);
    if (sc == kSchemeBf16)
      rc = launch_conv<s.ks, s.cinpad, s.npad, s.epi, s.concat, s.nblk, s.tps, kFmtHi, false, s.mw, s.ng,
                       layer_wgs(kRL1)>(h, s.slot, h->umma->stages[kRL1], h->umma->bias[kRL1], b.act0, a, stream);
    else
      rc = launch_conv<s.ks, s.cinpad, s.npad, s.epi, s.concat, s.nblk, s.tps, 0, false, s.mw, s.ng, layer_wgs(kRL1)>(
          h, s.slot, h->umma->stages[kRL1], h->umma->bias[kRL1], b.act0, a, stream);
    if (rc) return rc;
  } else {
    // L1: 16 -> 128 (cmg) + 96 (refiners); the training forward of the cmg alone has no r[1] and stores 128
    act(b.a[1], 128, b.r[1], b.r[1] ? 96 : 0);
    if ((rc = launch_layer<kL1>(h, sc, b.act0, a, stream))) return rc;
  }
  a.skip_lo = nullptr;
  a.a_hi_only = 0;
  a.slot_levels = nullptr;
  if (dump(kL1)) return WN_OK;
  if (want_cmg) {
    act(b.a[2], 128, nullptr, 0);
    a.f8_live_clear = want_ref ? 0x3u : ~0u;  // L1's refiner blocks are R2's to check and clear
    if ((rc = launch_layer<kC2>(h, sc, b.a[1], a, stream))) return rc;
    a.f8_live_clear = ~0u;
    if (dump(kC2)) return WN_OK;
    // cmg.conv4 fused into cmg.conv3's launch: its output must not land in b.a[4], the ping-pong buffer of b.a[2]
    // that the same launch's halo loads read, so from cmg.conv4 on every output moves one buffer back (b.a[l - 1])
    const bool fuse = kFuseC4 && o.fuse_c4;
    auto cmg_out = [&](int l) { return b.a[fuse ? l - 1 : l]; };
    if (fuse) {  // one launch: cmg.conv3, and cmg.conv4 in its epilogue
      act(cmg_out(4), 64, nullptr, 0);
      if ((rc = launch_layer<kC3, true>(h, sc, b.a[2], a, stream))) return rc;
    } else {
      act(b.a[3], 128, nullptr, 0);
      if ((rc = launch_layer<kC3>(h, sc, b.a[2], a, stream))) return rc;
      if (dump(kC3)) return WN_OK;
      act(b.a[4], 64, nullptr, 0);
      if ((rc = launch_layer<kC4>(h, sc, b.a[3], a, stream))) return rc;
      if (dump(kC4)) return WN_OK;
    }
    act(cmg_out(5), 64, nullptr, 0);
    if ((rc = launch_layer<kC5>(h, sc, cmg_out(4), a, stream))) return rc;
    if (dump(kC5)) return WN_OK;
    act(cmg_out(6), 64, nullptr, 0);
    if ((rc = launch_layer<kC6>(h, sc, cmg_out(5), a, stream))) return rc;
    if (dump(kC6)) return WN_OK;
    act(cmg_out(7), 64, nullptr, 0);
    if ((rc = launch_layer<kC7>(h, sc, cmg_out(6), a, stream))) return rc;
    if (dump(kC7)) return WN_OK;
    // the confidence maps are fp32: a dump of them is written in place of b.cm
    const bool dump_maps = dbg_layer == kSpecs[kC8].slot;
    a.out_f32 = dump_maps ? dbg_dst : b.cm;
    if ((rc = launch_layer<kC8>(h, sc, cmg_out(7), a, stream))) return rc;
    if (dump_maps) return WN_OK;
  }
  if (!want_ref) return WN_OK;
  act(b.r[2], 96, nullptr, 0);
  if ((rc = launch_layer<kR2>(h, sc, b.r[1], a, stream))) return rc;
  if (dump(kR2)) return WN_OK;
  last();
  // a dump of the refined images (number 10): the same launch with no gate, storing them alone
  const bool dump_refined = dbg_layer == kSpecs[kR3].slot;
  if (dump_refined) {
    a.out_f32 = nullptr;
    a.out_u8 = nullptr;
    a.cm = nullptr;
    a.refined_out = dbg_dst;
  }
  if ((rc = launch_layer<kR3>(h, sc, b.r[2], a, stream))) return rc;
  if (dump_refined) return WN_OK;
  return o.out_u8 ? mirror_u8(h, o.out_u8, o.peers, (size_t)n * H * W * 3, o.run_if, stream) : WN_OK;
}

// Workspace carve-up of one pass (<= umma_chunk images).
static FwdBuffers carve(void* workspace, int n, int H, int W) {
  const size_t px = (size_t)n * H * W;
  uint8_t* ws = (uint8_t*)(((uintptr_t)workspace + 1023) / 1024 * 1024);
  uint4* cmgAB[2];
  uint4* refAB[2];
  FwdBuffers b;
  memset(&b, 0, sizeof(b));
  b.act0 = (uint4*)ws;     ws += px * 64;
  cmgAB[0] = (uint4*)ws;   ws += px * 512;
  cmgAB[1] = (uint4*)ws;   ws += px * 512;
  refAB[0] = (uint4*)ws;   ws += px * 384;
  refAB[1] = (uint4*)ws;   ws += px * 384;
  b.cm = (float*)ws;       ws += px * 12;
  b.exact_flag = (int*)align256((uintptr_t)ws);
  for (int l = 1; l <= 7; l++) b.a[l] = cmgAB[(l - 1) & 1];
  b.r[1] = refAB[0];
  b.r[2] = refAB[1];
  return b;
}

int umma_debug_layer(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], int n, int H, int W,
                     int layer, float* dst, void* workspace, size_t workspace_bytes, cudaStream_t stream, int scheme) {
  if (!h->umma || umma_chunk(0, n, H, W) != n || workspace_bytes < umma_forward_workspace_bytes(n, H, W)) {
    set_error("debug layer dump: weights not packed, batch too large for one pass or workspace too small");
    return WN_E_WORKSPACE;
  }
  int rc = get_encoder();
  if (rc) return rc;
  // a dump stops the chain before the consumers that check and clear the low-end records
  WN_CUDA(cudaMemsetAsync(h->umma->live_dev, 0, kNumUmmaLayers * sizeof(unsigned), stream));
  FwdOpts o;
  o.scheme = scheme;
  o.dbg_layer = layer;
  o.dbg_dst = dst;
  return umma_forward_layers(h, in, in_strides, nullptr, n, H, W, carve(workspace, n, H, W), stream, o);
}

// Where the passes of a forward call store their results beyond their own buffers (FwdBuffers).  Whole images (no
// tiles, no window table) store at the offsets of the pass's first image; windows store their kept rectangles.
struct FwdOut {
  float* f32 = nullptr;        // kStackAll: the images, fp32 NCHW (may be null); kStackCmg: the maps; windowed
                               // kStackRefiners: refiner `which`'s image
  float* refined = nullptr;    // kStackRefiners: whole images [n][9][H][W]; windowed, one pass of windows
  int which = 0;
  uint8_t* u8 = nullptr;       // ten2arr'd uint8 NHWC images (the gate epilogue)
  PeerOut peers = {};          // ... and their peer copies
  const TileGeom* tiles = nullptr;  // the slots are windows of these tiles (grid geometry)
};

// One forward call (WN_MODE_BF16X3, WN_MODE_BF16_FP8): the weights, workspace and encoder checks, the scheme this
// handle runs (once an activation has left the e4m3 range, sticky flag, the handle keeps to bf16x3 until new weights
// are packed), then `start` (the call's LUTs, table and call-wide exact-levels flag), then per pass of geo: its
// buffers, `act0` (the operand planes, the per-pass flag), the ten launches, in the fp8-correction scheme the
// bf16x3 chain of the same pass right behind them, every launch conditional on the range flag (ConvArgs::run_if: a
// pass whose activations left the e4m3 range is recomputed within the call, nobody sees the degraded result), and a
// windowed sub-module's kept-rectangle store.  The range flag is mirrored to the host at the end.  flag: the
// call-wide exact-levels flag, or null when act0 sets one per pass.
template <class Geom, class Start, class Act0>
static int forward_call(wn_handle* h, const char* what, size_t workspace_bytes, size_t need, FwdOpts o, Geom geo,
                        const std::vector<RaggedPass>& passes, void* fwd_ws, int* flag, const FwdOut& f,
                        cudaStream_t stream, Start start, Act0 act0) {
  if (!h->umma) {
    set_error("tensor-core weights have not been packed");
    return WN_E_STATE;
  }
  if (workspace_bytes < need) {
    set_error("%s workspace too small: %zu < %zu", what, workspace_bytes, need);
    return WN_E_WORKSPACE;
  }
  int rc = get_encoder();
  if (rc) return rc;
  if (o.scheme == 1 && *h->umma->overflow_host) o.scheme = 0;
  if ((rc = start())) return rc;
  const int64_t none[4][4] = {};
  const float* no_in[4] = {nullptr, nullptr, nullptr, nullptr};
  o.packed = true;
  o.fuse_c4 = o.scheme != kSchemeBf16;  // nothing reads cmg.conv3's output but cmg.conv4
  for (const RaggedPass& p : passes) {
    geo.set_pass(p);
    FwdBuffers b = carve(fwd_ws, p.count, p.slot_h, p.slot_w);
    if (flag) b.exact_flag = flag;
    FwdOpts po = o;
    po.rwin = geo.rwin();
    if ((rc = act0(geo, p, b, po))) return rc;
    float* out = f.f32;
    if (!f.tiles && !po.rwin) {  // images p.first, p.first + 1, ...
      const size_t n0 = (size_t)p.first, px = (size_t)p.slot_h * p.slot_w;
      if (out) out += n0 * 3 * px;
      if (f.u8) po.out_u8 = f.u8 + n0 * px * 3;
      for (int k = 0; k < f.peers.n; k++) po.peers.p[k] = f.peers.p[k] + n0 * px * 3;
      po.peers.n = f.peers.n;
      if (o.stack == kStackCmg) b.cm = out;  // the maps are the result
      if (o.stack == kStackRefiners) {
        b.refined = f.refined + n0 * 9 * px;
        out = nullptr;
      }
    } else if (o.stack == kStackAll) {
      po.out_u8 = f.u8;
      if (f.tiles) {
        po.tiles = f.tiles;
        po.win0 = p.first;
      }
    } else {  // the sub-modules keep their result in window layout: store_kept_kernel below
      out = nullptr;
      if (o.stack == kStackRefiners) b.refined = f.refined;
    }
    if ((rc = umma_forward_layers(h, no_in, none, out, p.count, p.slot_h, p.slot_w, b, stream, po))) return rc;
    if (po.scheme == 1) {
      po.scheme = 0;
      po.run_if = h->umma->overflow_dev;
      Timing* timing = h->timing;  // the conditional launches are not part of the per-kernel timing record
      h->timing = nullptr;
      rc = umma_forward_layers(h, no_in, none, out, p.count, p.slot_h, p.slot_w, b, stream, po);
      h->timing = timing;
      if (rc) return rc;
    }
    if constexpr (std::is_same<Geom, GridGeom>::value)
      if (f.tiles && o.stack != kStackAll) {  // after the pass and its conditional bf16x3 re-run
        TimedScope ts(h, kSlotGate, stream);
        const bool maps = o.stack == kStackCmg;
        store_kept_kernel<<<dim3((unsigned)(((size_t)geo.slot_hw() + 255) / 256), p.count), 256, 0, stream>>>(
            maps ? b.cm : f.refined, maps ? 3 : 9, maps ? 0 : 3 * f.which, 3, f.f32, geo);
        WN_LAUNCH_CHECK(h);
      }
  }
  if (o.scheme == 1)
    WN_CUDA(cudaMemcpyAsync(h->umma->overflow_host, h->umma->overflow_dev, sizeof(int), cudaMemcpyDeviceToHost, stream));
  return WN_OK;
}

static int no_start() { return WN_OK; }

// uint8 in: the preprocess writes act0 as exact 8-bit levels (hi planes only), so the flag of every pass is set
static FwdOpts u8_opts(int scheme) {
  FwdOpts o;
  o.scheme = scheme;
  o.hi_only = true;
  return o;
}

int umma_forward(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], float* out, int n, int H,
                 int W, void* workspace, size_t workspace_bytes, cudaStream_t stream, int scheme, int stack,
                 float* refined) {
  const int nb = umma_chunk(h->chunk_pixels, n, H, W);
  // Several passes: whether the first layer runs its level form is decided once, over every input pixel of the n
  // images, so that the result does not depend on how the batch is split (the tiled and ragged calls decide so too).
  // The flag sits where a full pass puts it, beyond the buffers of any smaller pass.  One pass takes it in the
  // packing launch.
  int* flag = nb < n ? carve(workspace, nb, H, W).exact_flag : nullptr;
  FwdOpts o;
  o.scheme = scheme;
  o.stack = stack;
  FwdOut f;
  f.f32 = out;
  f.refined = refined;
  return forward_call(
      h, "forward", workspace_bytes, umma_forward_workspace_bytes(n, H, W), o, whole_images(H, W),
      grid_passes(n, nb, H, W), workspace, flag, f, stream,
      [&] { return flag ? pack_inputs(h, whole_images(H, W), pack_args(in, in_strides), n, nullptr, flag, stream) : WN_OK; },
      [&](const GridGeom&, const RaggedPass& p, FwdBuffers& b, FwdOpts& po) {
        const float* sub[4];
        for (int t = 0; t < 4; t++) sub[t] = in[t] + p.first * in_strides[t][0];
        return pack_inputs(h, whole_images(H, W), pack_args(sub, in_strides), p.count, b.act0,
                           flag ? nullptr : b.exact_flag, stream, po.scheme == kSchemeBf16);
      });
}

// preprocess -> forward -> ten2arr without materialising the four fp32 input tensors or the fp32 output:
// the per-pixel preprocess kernel writes the first layer's operand planes (8-bit levels are exact in bf16: hi
// planes only), the last launch's epilogue writes uint8 NHWC (hubconf.py:8-34, SURVEY 8f.2).
size_t umma_enhance_workspace_bytes(int n, int h, int w) {
  const int nb = umma_chunk(0, n, h, w);
  return umma_forward_workspace_bytes(n, h, w) + align256(preprocess_workspace_bytes(nb, h, w)) + 1024;
}

int umma_enhance_u8(wn_handle* h, const uint8_t* rgb, uint8_t* out_u8, float* out_f32, int n, int H, int W,
                    void* workspace, size_t workspace_bytes, cudaStream_t stream, int scheme, const PeerOut& peers) {
  const int nb = umma_chunk(h->chunk_pixels, n, H, W);
  uint8_t* pre_ws = (uint8_t*)align256((uintptr_t)workspace);
  const size_t pre_b = align256(preprocess_workspace_bytes(nb, H, W));
  FwdOut f;
  f.f32 = out_f32;
  f.u8 = out_u8;
  f.peers = peers;
  return forward_call(h, "enhance", workspace_bytes, umma_enhance_workspace_bytes(n, H, W), u8_opts(scheme),
                      whole_images(H, W), grid_passes(n, nb, H, W), pre_ws + pre_b, nullptr, f, stream, no_start,
                      [&](const GridGeom&, const RaggedPass& p, FwdBuffers& b, FwdOpts&) {
                        WN_CUDA(cudaMemsetAsync(b.exact_flag, 1, sizeof(int), stream));
                        return preprocess_u8_planes(h, rgb + (size_t)p.first * H * W * 3, p.count, H, W, b.act0,
                                                    pre_ws, pre_b, stream);
                      });
}

// The tiled form (tiling.cuh): the statistics and LUTs of all n images once, then per pass a batch of equally sized
// windows runs through the same ten launches (and range guard) as a batch of images, and the last launch stores
// each window's kept rectangle into the full-image outputs.  Workspace: one pass of windows plus the per-image
// LUTs, independent of the image size.  The geometry is arithmetic on the window index: nothing is copied from the
// host, so the call stays stream-ordered and can be captured in a graph.  Its callers have applied the shape and
// image-size checks of wn_enhance_u8_tiled (api.cu).
size_t umma_enhance_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels) {
  const TileGeom g = tile_geom(h, w, tile_h, tile_w);
  const long long p = tile_pass_windows(g, n, max_pass_pixels ? max_pass_pixels : kDefaultChunkPixels);
  return (size_t)p * g.win_h * g.win_w * kUmmaBytesPerPixel + 4096 + align256(preprocess_workspace_bytes(n, h, w)) +
         1024;
}

// the passes of the windows of n images of g, as many per pass as fit in max_pass_pixels (0: the default)
static std::vector<RaggedPass> window_passes(const TileGeom& g, int n, long long max_pass_pixels) {
  return grid_passes((long long)n * g.ny * g.nx,
                     tile_pass_windows(g, n, max_pass_pixels ? max_pass_pixels : kDefaultChunkPixels), g.win_h, g.win_w);
}

int umma_enhance_u8_tiled(wn_handle* h, const uint8_t* rgb, uint8_t* out_u8, float* out_f32, int n, int H, int W,
                          int tile_h, int tile_w, long long max_pass_pixels, void* workspace, size_t workspace_bytes,
                          cudaStream_t stream, int scheme) {
  const TileGeom g = tile_geom(H, W, tile_h, tile_w);
  uint8_t* pre_ws = (uint8_t*)align256((uintptr_t)workspace);
  const size_t pre_b = align256(preprocess_workspace_bytes(n, H, W));
  const RaggedImage img = ragged_image(rgb, H, W);
  FwdOut f;
  f.f32 = out_f32;
  f.u8 = out_u8;
  f.tiles = &g;
  return forward_call(
      h, "tiled enhance", workspace_bytes, umma_enhance_tiled_workspace_bytes(n, H, W, tile_h, tile_w, max_pass_pixels),
      u8_opts(scheme), GridGeom{g, 0}, window_passes(g, n, max_pass_pixels), pre_ws + pre_b, nullptr, f, stream,
      [&] { return preprocess_u8_luts(h, rgb, n, H, W, pre_ws, pre_b, stream); },
      [&](const GridGeom& geo, const RaggedPass& p, FwdBuffers& b, FwdOpts&) {
        WN_CUDA(cudaMemsetAsync(b.exact_flag, 1, sizeof(int), stream));
        return preprocess_u8_slot_planes(h, geo, img, n, p.count, b.act0, pre_ws, stream);
      });
}

// The ragged form (tiling.cuh ragged_plan): the statistics and LUTs of all n images in one launch each, then per
// pass a batch of slots runs through the same ten launches (and range guard) as a batch of images; each window's
// valid extent is masked and its kept rectangle stored into its own image.  The plan (per-image geometry and one
// descriptor per window) is copied into the workspace once per call, so the call cannot be captured in a graph.
// Workspace: the largest pass plus the per-image LUTs plus the table, independent of the image sizes.
static HostTable ragged_u8_table(int n, size_t windows) {
  return HostTable({(size_t)n * sizeof(RaggedImage), windows * sizeof(RaggedWindow)});
}
static long long ragged_pass_pixels(long long max_pass_pixels) {
  return max_pass_pixels ? max_pass_pixels : kDefaultChunkPixels;
}
static size_t ragged_workspace(int n, const std::vector<RaggedWindow>& wins, const std::vector<RaggedPass>& passes) {
  return (size_t)largest_pass_pixels(passes) * kUmmaBytesPerPixel + 4096 +
         align256(preprocess_workspace_bytes(n, 1, 1)) + ragged_u8_table(n, wins.size()).bytes() + 1024;
}

size_t umma_enhance_ragged_workspace_bytes(const int* hs, const int* ws, int n, int tile_h, int tile_w,
                                           long long max_pass_pixels) {
  std::vector<RaggedWindow> wins;
  std::vector<RaggedPass> passes;
  ragged_plan(hs, ws, n, tile_h, tile_w, ragged_pass_pixels(max_pass_pixels), &wins, &passes);
  return ragged_workspace(n, wins, passes);
}

int umma_enhance_u8_ragged(wn_handle* h, const wn_ragged_image* images, int n, int tile_h, int tile_w,
                           long long max_pass_pixels, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                           int scheme) {
  std::vector<int> hs, ws;
  ragged_sizes(images, n, &hs, &ws);
  std::vector<RaggedWindow> wins;
  std::vector<RaggedPass> passes;
  ragged_plan(hs.data(), ws.data(), n, tile_h, tile_w, ragged_pass_pixels(max_pass_pixels), &wins, &passes);
  // workspace: [LUTs of the n images][table: n RaggedImage | windows][one pass]
  uint8_t* pre_ws = (uint8_t*)align256((uintptr_t)workspace);
  const size_t pre_b = align256(preprocess_workspace_bytes(n, 1, 1));
  uint8_t* table = pre_ws + pre_b;
  HostTable t = ragged_u8_table(n, wins.size());
  const RaggedImage* d_imgs = t.dev<RaggedImage>(table, 0);
  const TableGeom geo = {t.dev<RaggedWindow>(table, 1), 0, 0, 0, tile_h, tile_w};
  auto start = [&]() {
    RaggedImage* imgs = t.part<RaggedImage>(0);
    int max_slabs = 1;
    for (int i = 0; i < n; i++) {
      imgs[i] = ragged_image(images[i].rgb, images[i].height, images[i].width);
      max_slabs = imgs[i].slabs > max_slabs ? imgs[i].slabs : max_slabs;
    }
    RaggedWindow* rw = t.part<RaggedWindow>(1);
    for (size_t k = 0; k < wins.size(); k++) {
      rw[k] = wins[k];
      rw[k].rgb = images[wins[k].img].rgb;
      rw[k].out_u8 = images[wins[k].img].out_u8;
      rw[k].out_f32 = images[wins[k].img].out_f32;
    }
    const int rc = t.upload(table, stream);
    return rc ? rc : preprocess_u8_ragged_luts(h, n, d_imgs, max_slabs, pre_ws, stream);
  };
  return forward_call(h, "ragged enhance", workspace_bytes, ragged_workspace(n, wins, passes), u8_opts(scheme), geo,
                      passes, table + t.bytes(), nullptr, FwdOut(), stream, start,
                      [&](const TableGeom& pg, const RaggedPass& p, FwdBuffers& b, FwdOpts&) {
                        WN_CUDA(cudaMemsetAsync(b.exact_flag, 1, sizeof(int), stream));
                        return preprocess_u8_slot_planes(h, pg, d_imgs, n, p.count, b.act0, pre_ws, stream);
                      });
}

// The tiled form of umma_forward (fp32 tensors in): the windows of tiling.cuh, one pass of them at a time through
// the same ten launches and range guard.  The windowed packing kernel reads each window's operands at image
// coordinates through the caller's strides.  Whether the first layer drops its a_lo pass is decided once for the
// whole call, over every input pixel of the n images (whole_images), so it takes the path wn_forward takes when that
// runs the batch in one pass.  The flag sits at the start of the workspace, outside the per-pass carve-up (whose
// layout moves with the window count), and stays valid for the bf16x3 re-run of every pass.  kStackAll: the gate
// epilogue stores each kept rectangle into `out`.  The sub-modules keep their result (the maps, or the three refined
// images) in window layout and store_kept_kernel copies the kept rectangle of the wanted planes into `out`.
// Workspace: [flag | refined images of one pass (sub-modules) | one pass], independent of the image size.  Nothing
// is copied from the host: the call can be captured in a graph.
size_t umma_forward_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels,
                                          bool submodule) {
  const TileGeom g = tile_geom(h, w, tile_h, tile_w);
  const size_t px = (size_t)tile_pass_windows(g, n, max_pass_pixels ? max_pass_pixels : kDefaultChunkPixels) *
                    g.win_h * g.win_w;
  return px * kUmmaBytesPerPixel + 4096 + 256 + (submodule ? align256(px * 9 * sizeof(float)) + 256 : 0);
}

int umma_forward_tiled(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], float* out, int n,
                       int H, int W, int tile_h, int tile_w, long long max_pass_pixels, void* workspace,
                       size_t workspace_bytes, cudaStream_t stream, int scheme, int stack, int which) {
  const bool sub = stack != kStackAll;
  const TileGeom g = tile_geom(H, W, tile_h, tile_w);
  const std::vector<RaggedPass> passes = window_passes(g, n, max_pass_pixels);
  uint8_t* base = (uint8_t*)align256((uintptr_t)workspace);
  int* exact = (int*)base;
  FwdOut f;
  f.f32 = out;
  f.refined = (float*)(base + 256);
  f.which = which;
  f.tiles = &g;
  void* fwd_ws = base + 256 + (sub ? align256(largest_pass_pixels(passes) * 9 * sizeof(float)) : 0);
  const PackInArgs pa = pack_args(in, in_strides);
  FwdOpts o;
  o.scheme = scheme;
  o.stack = stack;
  return forward_call(
      h, "tiled forward", workspace_bytes,
      umma_forward_tiled_workspace_bytes(n, H, W, tile_h, tile_w, max_pass_pixels, sub), o, GridGeom{g, 0}, passes,
      fwd_ws, exact, f, stream, [&] { return pack_inputs(h, whole_images(H, W), pa, n, nullptr, exact, stream); },
      [&](const GridGeom& geo, const RaggedPass& p, FwdBuffers& b, FwdOpts&) {
        return pack_inputs(h, geo, pa, p.count, b.act0, nullptr, stream);
      });
}

// The ragged form of umma_forward (fp32 tensors in, wn_forward_ragged): the windows and passes of ragged_plan, as
// umma_enhance_u8_ragged runs them, with the operands read through each image's strides (pack_inputs on the table)
// instead of preprocessed from uint8.  The exact-levels flag is taken once over every input pixel of every image
// before the first pass, as umma_forward_tiled takes it, and stays valid for the bf16x3 re-run of every pass.  The
// gate epilogue stores each window's kept rectangle into its image's `out` (RaggedWindow::out_f32).  The plan (one
// PackInArgs per image, one descriptor per window) is copied into the workspace once per call, so the call cannot be
// captured in a graph.  Workspace: [flag | table | the largest pass].
static HostTable ragged_fp32_table(int n, size_t windows) {
  return HostTable({(size_t)n * sizeof(PackInArgs), windows * sizeof(RaggedWindow)});
}
static size_t ragged_fp32_workspace(int n, const std::vector<RaggedWindow>& wins,
                                    const std::vector<RaggedPass>& passes) {
  return (size_t)largest_pass_pixels(passes) * kUmmaBytesPerPixel + 4096 + 256 +
         ragged_fp32_table(n, wins.size()).bytes() + 1024;
}

size_t umma_forward_ragged_workspace_bytes(const int* hs, const int* ws, int n, int tile_h, int tile_w,
                                           long long max_pass_pixels) {
  std::vector<RaggedWindow> wins;
  std::vector<RaggedPass> passes;
  ragged_plan(hs, ws, n, tile_h, tile_w, ragged_pass_pixels(max_pass_pixels), &wins, &passes);
  return ragged_fp32_workspace(n, wins, passes);
}

int umma_forward_ragged(wn_handle* h, const wn_ragged_tensors* images, int n, int tile_h, int tile_w,
                        long long max_pass_pixels, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                        int scheme) {
  std::vector<int> hs, ws;
  ragged_sizes(images, n, &hs, &ws);
  std::vector<RaggedWindow> wins;
  std::vector<RaggedPass> passes;
  ragged_plan(hs.data(), ws.data(), n, tile_h, tile_w, ragged_pass_pixels(max_pass_pixels), &wins, &passes);
  uint8_t* base = (uint8_t*)align256((uintptr_t)workspace);
  int* exact = (int*)base;
  uint8_t* table = base + 256;
  HostTable t = ragged_fp32_table(n, wins.size());
  const PackInArgs* d_imgs = t.dev<PackInArgs>(table, 0);
  const TableGeom geo = {t.dev<RaggedWindow>(table, 1), 0, 0, 0, tile_h, tile_w};
  auto start = [&]() {
    PackInArgs* imgs = t.part<PackInArgs>(0);
    for (int i = 0; i < n; i++) {
      const wn_ragged_tensors& d = images[i];
      const float* in[4] = {d.x, d.wb, d.he, d.gc};
      imgs[i] = pack_args(in, d.in_strides);
    }
    RaggedWindow* rw = t.part<RaggedWindow>(1);
    for (size_t k = 0; k < wins.size(); k++) {
      rw[k] = wins[k];
      rw[k].out_f32 = images[wins[k].img].out;
    }
    int rc = t.upload(table, stream);
    if (rc) return rc;
    WN_CUDA(cudaMemsetAsync(exact, 1, sizeof(int), stream));  // nonzero = "all inputs are 8-bit levels"
    TableGeom fg = geo;
    for (const RaggedPass& p : passes) {
      fg.set_pass(p);
      if ((rc = pack_inputs(h, fg, d_imgs, p.count, nullptr, exact, stream))) return rc;
    }
    return WN_OK;
  };
  FwdOpts o;
  o.scheme = scheme;
  return forward_call(h, "ragged forward", workspace_bytes, ragged_fp32_workspace(n, wins, passes), o, geo, passes,
                      table + t.bytes(), exact, FwdOut(), stream, start,
                      [&](const TableGeom& pg, const RaggedPass& p, FwdBuffers& b, FwdOpts& po) {
                        // the fp8-correction scheme decides the first layer's form per window (kFmtPair8): its flags
                        // sit in the buffer of cmg.conv2's output, which nothing reads or writes before the first
                        // layer has run
                        int* slot_flags = po.scheme == 1 ? reinterpret_cast<int*>(b.a[2]) : nullptr;
                        po.slot_levels = slot_flags;
                        return pack_inputs(h, pg, d_imgs, p.count, b.act0, nullptr, stream, false, slot_flags);
                      });
}

int umma_f8_overflowed(const wn_handle* h) { return h->umma && h->umma->overflow_host ? *h->umma->overflow_host : 0; }

}  // namespace wn

