// Implicit-GEMM convolution kernel (Hopper wgmma) shared by the forward (conv_umma.cu) and the backward
// data-gradient pass (conv_bwd.cu).  See conv_umma.cu for the design notes.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma_ops.cuh"

namespace wn {

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// Bounded wait: a pipeline bug becomes a trap ("unspecified launch failure"), never a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t it = 0; it < (1u << 26); it++) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) return;
  }
  __trap();
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* tmap, uint64_t* bar, int c0,
                                            int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// wgmma shared-memory matrix descriptor, no swizzle.  K-major: LBO = byte distance between the two 8-element K
// halves of a K = 16 step, SBO = byte distance between 8-row groups.  MN-major: LBO = distance between the 8-deep K
// groups, SBO = distance between 8-element M/N groups.
__device__ __forceinline__ uint64_t make_desc(uint32_t addr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((addr >> 4) & 0x3fff) | ((uint64_t)((lbo >> 4) & 0x3fff) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3fff) << 32);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
// barrier over the 128 threads of one warpgroup (id 1 + warpgroup; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
// four floats -> four e4m3 bytes, f0 at the lowest address
__device__ __forceinline__ uint32_t pack_e4m3x4(float f0, float f1, float f2, float f3) {
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(f1), "f"(f0));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(f3), "f"(f2));
  return (uint32_t)lo | ((uint32_t)hi << 16);
}
__device__ __forceinline__ uint16_t pack_e4m3x2(float f0, float f1) {
  uint16_t v;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(v) : "f"(f1), "f"(f0));
  return v;
}

// ------------------------------------------------------------------------------------------
// Kernel configuration
// ------------------------------------------------------------------------------------------
// kEpiAct: bias + ReLU -> bf16 hi/lo planes.  kEpiSigmoid: bias + sigmoid -> 3 fp32 maps.
// kEpiGate: bias + ReLU, gated sum with the confidence maps -> fp32 NCHW output.
// kEpiDgrad (backward): no bias; zero where the saved forward activation is zero (ReLU'), -> planes.
enum Epilogue { kEpiAct = 0, kEpiSigmoid = 1, kEpiGate = 2, kEpiDgrad = 3 };

// One CTA tile = (8 * MW) x (8 * WGS) pixels: consumer warpgroup w computes pixel rows 8w..8w+7 as MW m64 blocks
// (block b = tile columns 8b..8b+7) with m64nNk16 wgmma, accumulators in registers, and then runs the epilogue of
// those rows itself.  Warps 0 .. 4 WGS - 1 are the consumers; warp 4 WGS is the A producer (TMA halo tiles), warp
// 4 WGS + 1 the B producer (weights).
constexpr int kStageLd = 36;       // epilogue staging: floats per row (32 channels + 4 against bank conflicts)

// NPAD   output channels per diagonal block
// CONCAT weight stage rows are [hi rows | lo rows]: a_hi x [w_hi|w_lo] is ONE MMA of N = 2*NPAD (the
//        activation tile is read from shared memory once for two products), then a_lo x w_hi with
//        N = NPAD.  Pays when NPAD <= 64, where an MMA is bound by the A-operand read.
// NBLK   number of diagonal blocks (the three refiners run as one block-diagonal layer): input
//        chunk c only feeds block c / (NCHUNK / NBLK), so only that block's weights are staged.
// TPS    filter taps per weight stage: small-N layers batch a kernel row (or all taps) per stage so
//        that the per-stage pipeline cost (barrier wait, wgmma commit and wait, bulk-copy latency) is amortised.
// FMT    bit 0 (kFmtIn8): fp8 correction scheme on the input side.  v = hi (bf16) + lo; instead of the two
//        bf16 correction passes (a_lo x w_hi, a_hi x w_lo) ONE e4m3 wgmma of K = 32 multiplies
//        [e4m3(lo * 2^9) | e4m3(v)] (the two fp8 planes the producing layer wrote where the bf16 lo planes
//        used to be) by [e4m3(w * ws) ; e4m3(w_lo * ws * 2^9)]: 2 pass-equivalents instead of 3 at half the
//        operand bytes.  The bf16 weights of such a layer are packed pre-scaled by the power of two ws * 2^9
//        (exact), so the two products carry the same scale and the epilogue multiplies their sum by 2^-9 / ws once.
//        Both products go into ONE accumulator, in two phases per tile: the correction phase issues every chunk's
//        e4m3 wgmmas, then the main phase every chunk's bf16 a_hi x w_hi.  Hopper's fp8 wgmma adds with fewer mantissa
//        bits than fp32; in this order it only ever adds into correction sums (about 2^-8 of the result), never into
//        the main product.  Each phase walks the chunks in pairs: a halo stage holds the two planes of each chunk of
//        a pair that the phase reads, a weight stage the phase's 32-byte-per-channel units of TPS taps of both chunks
//        (pack_stages_f8_kernel), so stages keep the bytes and the wgmma count of the other forms.
//        bit 1 (kFmtOut8): the epilogue writes that hi + fp8-planes format (its consumer has bit 0 set).
//        bit 2 (kFmtHi): single-pass bf16 (WN_MODE_BF16, training only): ONE wgmma per product, a_hi x w_hi of
//        N = NPAD (a CONCAT layer takes the hi rows of its [hi | lo] stage rows), fp32 accumulation.  The a_lo and w_lo
//        products are never issued and the halo loads fetch the two hi planes of a chunk only.  kEpiAct / kEpiDgrad
//        store lo = 0, so every plane buffer of that mode holds exactly the bf16 operand its consumers multiply.
//        bit 3 (kFmtPair8): the first layer's fp8 tap-pair form, for 8-bit-level inputs (*skip_lo set, or the tile's
//        entry of slot_levels; otherwise the tile runs the bf16x3 form of FMT 0 from ConvArgs::wpk).  A level a is exact in bf16, so only a x w_lo has
//        to be added to a x w_hi, and it is ONE e4m3 wgmma of K = 32 per PAIR of taps: the two 16-byte core matrices
//        of a K = 32 row are the 16 channels of two taps of the same halo plane, one descriptor LBO apart (pair table
//        in the consumer).  The consumers convert the halo tile's hi planes to e4m3 in shared memory themselves.
//        Per tile and warpgroup: 25 e4m3 wgmmas (all of them first: the accumulator holds only correction sums while
//        the fp8 MMA, which adds with fewer bits than fp32, adds into it), then 49 bf16 wgmmas a x w_hi; the weights
//        (ConvArgs::wpk8) are scaled by s_c 2^9 per output column c (a power of two) and the epilogue multiplies
//        column c by 2^-9 / s_c (ConvArgs::f8_scale[c]).  74 bf16-pass equivalents instead of 98.
//        bit 4 (kFmtFuse1x1): a 1x1 layer NPAD -> kFuseNpad (cmg.conv4 behind cmg.conv3) runs in the epilogue.  Each
//        warpgroup computes the layer's activation in the accumulator layout with the fp32 operations of the kEpiAct
//        epilogue, splits it into bf16 hi / lo and packs the pairs into the A registers of RS wgmmas (an m64nNk16
//        accumulator fragment's columns [16k, 16k + 16) are the A fragment of K step k); then, per 16-channel chunk,
//        a_hi x [w_hi | w_lo] and a_lo x w_hi as the 1x1 layer's own CONCAT launch issues them, from its bf16x3 image
//        (ConvArgs::wpk1x1), which the B producer sends as kFuseStages more weight stages behind each tile's.  The
//        1x1 layer's output (ConvArgs::bias1x1, dst0, cout, kFmtOut8, f8_overflow) is what the epilogue stores; the
//        layer's own activation never leaves registers.
// MW     m64 blocks per warpgroup: 1 = 8 x 16-pixel tile (M = 128), 2 = 16 x 16 (M = 256).  Every weight stage a
//        CTA streams from L2 then serves twice the pixels.
// NG     column groups: a CTA computes the NPAD output channels [g * NPAD, (g + 1) * NPAD) of column group g; the
//        layer has NG * NPAD channels and each group's weight stages are packed contiguously.  Splitting the columns
//        keeps MW = 2 within the registers of a wide layer, at the price of reading each halo tile once per group.
// WGS    consumer warpgroups: 2 = 16-row tiles, 320 threads (warps 0-7 consumers, 8-9 producers); 3 = 24-row tiles,
//        512 threads (warps 0-11 consumers, 12-13 producers, 14-15 only complete the producer warpgroup).  A third
//        warpgroup serves every weight stage to 192 pixels instead of 128 without more accumulators per thread; at
//        512 threads the register file allows 128 per thread, so the producer warpgroup gives its registers up
//        (setmaxnreg) and the consumers run at kWgs3ConsumerRegs.
constexpr int kFmtIn8 = 1, kFmtOut8 = 2, kFmtHi = 4, kFmtPair8 = 8, kFmtFuse1x1 = 16;
// The low end of e4m3 (DESIGN 4.2): a block of fp8 planes whose largest value is below this is recomputed in bf16x3
constexpr float kF8LowMax = 0.015625f;  // 2^-6, e4m3's smallest normal
// kFmtFuse1x1: output channels of the fused 1x1 layer, and its weight stages per tile (its 16-channel chunks, 4 KB
// each in the CONCAT layout, UmmaCfg::FUSE_CHUNKS to a stage)
constexpr int kFuseNpad = 64, kFuseStages = 2;
constexpr int kWgs3ProducerRegs = 24, kWgs3ConsumerRegs = 160;  // 128 x 24 + 384 x 160 <= 65,536
template <int KS, int CIN_PAD, int NPAD, int CONCAT = 0, int NBLK = 1, int TPS = 1, int FMT = 0, int MW = 1,
          int NG = 1, int WGS = 2>
struct UmmaCfg {
  static constexpr bool F8IN = (FMT & kFmtIn8) != 0;
  static constexpr bool HI = (FMT & kFmtHi) != 0;
  static constexpr bool PAIR = (FMT & kFmtPair8) != 0;
  static constexpr bool FUSE = (FMT & kFmtFuse1x1) != 0;
  static constexpr bool DUAL = CONCAT != 0 && !HI;  // two accumulator halves per block: [a x w_hi | a_hi x w_lo]
  static constexpr int TILE_W = 8 * MW, TILE_H = 8 * WGS;
  static constexpr int CONSUMER_WARPS = 4 * WGS;                  // arrivals per "stage empty"
  static constexpr int WARP_A = CONSUMER_WARPS, WARP_B = CONSUMER_WARPS + 1;
  static constexpr int THREADS = WGS == 2 ? 320 : 512;
  static constexpr int HALO_W = TILE_W + KS - 1, HALO_H = TILE_H + KS - 1;
  static constexpr int NCHUNK = CIN_PAD / 16;
  static constexpr int PLANE_BYTES = HALO_W * HALO_H * 16;
  // hi k0, hi k1, lo k0, lo k1; F8IN: the two planes its phase reads of each chunk of a pair (fp8 or hi planes)
  static constexpr int A_STAGE = (4 * PLANE_BYTES + 1023) / 1024 * 1024;
  // one tap of weights: [hi|lo][k8 0|1][NPAD][16 B] (CONCAT: [k8][hi rows | lo rows]) -- 64 B per output channel;
  // fp8 scheme: one phase's unit of a tap, [k16 half][NPAD][16 B] e4m3 or [k8][NPAD][16 B] bf16 -- 32 B, and a
  // stage holds TPS taps of both chunks of a pair
  static constexpr int B_TAP = NPAD * (F8IN ? 32 : 64);
  static constexpr int B_STAGE = (F8IN ? 2 : 1) * TPS * B_TAP;
  // kFmtFuse1x1: the layer's NPAD outputs are the 1x1 layer's 16-channel chunks; its weight stages are those of a
  // CONCAT launch (64 B per output channel and chunk for [w_hi | w_lo])
  static constexpr int FUSE_CHUNKS = NPAD / 16 / kFuseStages;  // chunks of the 1x1 layer per weight stage
  static constexpr int FUSE_STAGE = FUSE_CHUNKS * kFuseNpad * 64;
  static_assert((KS * KS) % TPS == 0, "taps per weight stage must divide the filter");
  static constexpr int NSTAGE_PER_CHUNK = KS * KS / TPS;
  static constexpr int STAGING = WGS * 64 * kStageLd * 4;
  // barriers (512 B) + the biases of every column group: 2048 B, more for layers over 384 channels (VGG's 512)
  // (kFmtPair8: the per-column dequantisation factors follow the biases)
  // (kFmtFuse1x1: the fused layer's biases follow)
  static constexpr int BIAS_BYTES = NG * NBLK * NPAD * 4 * (PAIR ? 2 : 1) + (FUSE ? kFuseNpad * 4 : 0);
  static constexpr int TAIL = 512 + (BIAS_BYTES > 1536 ? BIAS_BYTES : 1536);
  static constexpr int BUDGET = 227 * 1024 - 1024 - TAIL - STAGING;
  // halo ring: enough stages to prefetch the next chunk (or the next tile when there is one chunk)
  // (a 1x1 layer is HBM-bound and its stages are small: keep more loads in flight)
  static constexpr int NA_WANT = NCHUNK == 1 ? 2 : KS == 1 ? 6 : 3;
  // weight ring: whatever is left after the halo ring, 2..8 stages
  static constexpr int NB_FIT = (BUDGET - NA_WANT * A_STAGE) / B_STAGE;
  static constexpr int NB = NB_FIT > 8 ? 8 : NB_FIT < 2 ? 2 : NB_FIT;
  static constexpr int NA_FIT = (BUDGET - NB * B_STAGE) / A_STAGE;
  static constexpr int NA = NA_FIT > NA_WANT ? NA_WANT : NA_FIT;
  static_assert(!F8IN || !CONCAT, "fp8 corrections: the [hi | second part] weight layout");
  static_assert(!HI || FMT == kFmtHi, "single-pass bf16 reads and writes bf16 planes only");
  // kFmtPair8: one chunk of 16 channels, one tap per bf16x3 stage; warpgroup w converts its halo rows into plane 2 + w
  static_assert(!PAIR || (CIN_PAD == 16 && !CONCAT && NBLK == 1 && TPS == 1 && MW == 1 && NG == 1 && WGS == 2 &&
                          !F8IN && !HI), "the tap-pair form is the first layer's");
  static constexpr int PAIRS = (KS * KS + 1) / 2;           // e4m3 wgmmas per tile (the last tap pairs with a zero)
  static constexpr int PAIR_UNITS = PAIRS + KS * KS;        // units of NPAD * 32 B: e4m3 pairs, then bf16 taps
  static constexpr int PAIR_STAGES = PAIR_UNITS / 2;        // two units per weight stage of B_STAGE bytes
  static_assert(!PAIR || PAIR_UNITS % 2 == 0, "whole weight stages");
  static_assert(!FUSE || (!CONCAT && NBLK == 1 && MW == 1 && NG == 1 && !HI && !PAIR && FUSE_STAGE <= B_STAGE &&
                          NPAD % (16 * kFuseStages) == 0), "the fused 1x1 layer follows a plain layer of one block");
  static constexpr int CPB = NCHUNK / NBLK;                // chunks per diagonal block
  static constexpr int BLK_COLS = DUAL ? 2 * NPAD : NPAD;   // accumulator columns per block
  static constexpr int COLS = NBLK * BLK_COLS;             // accumulator columns of the tile
  static constexpr int ACC = COLS / 2;                     // fp32 accumulator registers per thread (M = 64 per warpgroup)
  static constexpr int SMEM_BYTES = NA * A_STAGE + NB * B_STAGE + STAGING + TAIL + 1024;  // + barriers/bias + align slack
  static_assert(NA >= 1, "halo tile does not fit in shared memory");
  static_assert(NCHUNK % NBLK == 0, "chunks must split evenly over the diagonal blocks");
  static_assert(NPAD % 16 == 0 && (DUAL ? 2 : 1) * NPAD <= 256, "invalid wgmma N");
  static_assert(MW == 1 || MW == 2, "one or two m64 blocks per warpgroup");
  static_assert(WGS == 2 || WGS == 3, "two or three consumer warpgroups");
  static_assert(NG == 1 || NBLK == 1, "column groups of a block-diagonal layer");
  static_assert(MW * ACC <= 128, "accumulators do not fit in registers");
  static_assert(!F8IN || CPB % 2 == 0, "fp8 corrections: chunk pairs of one diagonal block");
  // full weight image of one column group: every (chunk, stage); F8IN: every (phase, chunk pair, stage)
  static constexpr size_t GROUP_BYTES = (size_t)NCHUNK * NSTAGE_PER_CHUNK * B_STAGE;
};

struct ActDst {
  uint4* base;   // [n][2*planes_half][H][W] of 16-byte (8 x bf16) units
  int planes_half;
};

struct ConvArgs {
  const uint8_t* wpk;   // packed weight stages
  const float* bias;    // [NPAD]
  int N, H, W;
  int in_planes_half;   // C_in_pad / 8
  int tiles_x, tiles_y;
  int num_tiles;        // work items: tiles_x * tiles_y * N * NG (one parameter load, never a register kept live)
  // kEpiAct
  ActDst dst0, dst1;
  int split_c;          // channels [0, split_c) -> dst0, [split_c, cout) -> dst1
  int cout;             // valid output channels
  // kEpiSigmoid / kEpiGate
  float* out_f32;       // [n][3][H][W] (gate: optional)
  const float* cm;      // [n][3][H][W] (gate; null = no gated sum, only refined_out is produced)
  uint8_t* out_u8;      // gate, optional: ten2arr of the result (clip [0,1], *255, truncate), uint8 NHWC
  // optional: *skip_lo != 0 means every input value is exactly representable in the hi plane
  // (8-bit image levels), so the a_lo x w_hi pass contributes nothing and is not issued
  const int* skip_lo;
  // the input planes hold exact 8-bit levels and only the hi planes exist (written by the preprocess kernel):
  // the halo loads fetch two planes per chunk instead of four and the a_lo pass is never issued
  int a_hi_only;
  // kEpiGate, training only: also store the three refined images (post-ReLU), fp32 [n][9][H][W]
  float* refined_out;
  // kEpiDgrad: saved forward activation (planes) whose zeros gate the gradient
  const uint4* mask_base;
  int mask_planes_half;
  // fp8 correction scheme (FMT bit 0): dequantisation factor 2^-9 / ws of the accumulator; kFmtPair8: one factor
  // 2^-9 / s_c per output column
  const float* f8_scale;
  // kFmtPair8: the tap-pair weight image (pack_stages_pair_kernel), streamed instead of wpk for level inputs
  const uint8_t* wpk8;
  // kFmtPair8, optional: per image of the launch, nonzero when it holds 8-bit levels only.  A ragged pass decides
  // the form per window with it (its windows come from images of every kind); otherwise *skip_lo decides
  const int* slot_levels;
  // FMT bit 1: sticky device flag raised when an activation leaves the e4m3 range (its correction terms would
  // saturate in the consumer's fp8 pass); the host side then re-runs the batch with the bf16x3 kernels.  FMT bit 0
  // raises it too, for operands at e4m3's low end (f8_live_in)
  int* f8_overflow;
  // FMT bit 1: the low end of the launch's output, per block b of its columns (L1: block 0 the cmg's 128, blocks 1-3
  // the refiners' 32 each; one block elsewhere): bit 2b once a value of the block is nonzero, bit 2b + 1 once one is
  // at least kF8LowMax.  Each consumer warp ORs what it stored into it when it is done
  unsigned* f8_live;
  // FMT bit 0: the f8_live word of the launch whose fp8 planes this one reads.  Before anything else one thread checks
  // the blocks of f8_live_need (their bits 2b): a block that is nonzero with no value of kF8LowMax or more raises
  // f8_overflow; then it clears the bits of f8_live_clear for the next pass
  unsigned* f8_live_in;
  unsigned f8_live_need, f8_live_clear;
  // conditional launch: when non-null and *run_if == 0 the kernel returns at once (the bf16x3 re-run of a
  // batch is enqueued unconditionally behind the fp8-correction pass and only does work if the flag is up)
  const int* run_if;
  // kEpiGate of the tiled forward (tiled != 0): image n of the launch is window win0 + n of `tiles`; only the
  // pixels of its kept rectangle are stored, into out_f32 / out_u8 of the full images at image coordinates
  int tiled;
  long long win0;
  TileGeom tiles;
  // ragged batches (kernel template RAG): image n of the launch is window rwin[n] at the slot's top-left.  kEpiAct
  // stores zeros at slot pixels outside its valid extent; kEpiGate stores its kept rectangle into that window's
  // image (its own out_f32 / out_u8 and width)
  const RaggedWindow* rwin;
  // kFmtFuse1x1: the fused 1x1 layer's bf16x3 CONCAT weight image and its biases
  const uint8_t* wpk1x1;
  const float* bias1x1;
};

__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}
// v = hi + lo with hi = bf16(v), lo = bf16(v - hi), for two values at once: two packed conversions
// (F2FP.BF16.PACK_AB) instead of four scalar F2F, and the back-conversion is a shift.
__device__ __forceinline__ void split_bf16x2(float f0, float f1, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(f0, f1);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  const float h0 = __uint_as_float(hi << 16), h1 = __uint_as_float(hi & 0xffff0000u);
  const __nv_bfloat162 l = __floats2bfloat162_rn(f0 - h0, f1 - h1);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// Epilogue of 16 consecutive output channels [ch, ch + 16) of one pixel; f = the raw sums (scaled in the fp8 scheme).
// RAG: `valid` is false at slot pixels outside the window's valid extent, where kEpiAct stores zeros (hi, lo and
// fp8 planes alike; they cannot raise the e4m3 flag).
// HI (kFmtHi): the planes hold bf16(v) and lo = 0.
// Returns OUT8's ConvArgs::f8_live bits of the 16 values (0 otherwise).
template <int EPI, bool OUT8, bool RAG = false, bool HI = false>
__device__ __forceinline__ unsigned epilogue16(const ConvArgs& g, const float* s_bias, const float* f, int ch, int n,
                                           int gx, int gy, bool valid = true) {
  const size_t hw = (size_t)g.H * g.W;
  const size_t pix = (size_t)gy * g.W + gx;
  if constexpr (EPI == kEpiAct || EPI == kEpiDgrad) {
    if (ch >= g.cout) return 0u;
    if constexpr (OUT8) {
      // hi planes as usual; where the bf16 lo planes would be: per 16 channels one plane of
      // e4m3((v - hi) * 2^9) and one of e4m3(v) -- the K = 32 operand of the consumer's fp8 pass
      uint32_t hi[8], l8[4], h8[4];
      float vmax = 0.f;
#pragma unroll
      for (int j = 0; j < 16; j += 4) {
        float v[4], r[4];
#pragma unroll
        for (int t = 0; t < 4; t++) {
          v[t] = fmaxf(f[j + t] + s_bias[ch + j + t], 0.f);
          if constexpr (RAG) v[t] = valid ? v[t] : 0.f;
          vmax = fmaxf(vmax, v[t]);
        }
#pragma unroll
        for (int t = 0; t < 4; t += 2) {
          const __nv_bfloat162 h = __floats2bfloat162_rn(v[t], v[t + 1]);
          const uint32_t hb = *reinterpret_cast<const uint32_t*>(&h);
          hi[(j + t) >> 1] = hb;
          r[t] = (v[t] - __uint_as_float(hb << 16)) * 512.f;
          r[t + 1] = (v[t + 1] - __uint_as_float(hb & 0xffff0000u)) * 512.f;
        }
        l8[j >> 2] = pack_e4m3x4(r[0], r[1], r[2], r[3]);
        h8[j >> 2] = pack_e4m3x4(v[0], v[1], v[2], v[3]);
      }
      // e4m3 range guard (|v| <= 448).  v is past the ReLU, whose fmaxf has already turned a NaN into 0; +inf raises it
      if (!(vmax <= 448.f) && g.f8_overflow) atomicOr(g.f8_overflow, 1);
      const bool second = ch >= g.split_c;
      const ActDst& d = second ? g.dst1 : g.dst0;
      const int chl = second ? ch - g.split_c : ch;
      const unsigned live = vmax > 0.f ? (vmax >= kF8LowMax ? 3u : 1u) << (second ? 2 + 2 * (chl >> 5) : 0) : 0u;
      uint4* p_hi = d.base + ((size_t)n * 2 * d.planes_half + (chl >> 3)) * hw + pix;
      uint4* p_f8 = d.base + ((size_t)n * 2 * d.planes_half + d.planes_half + 2 * (chl >> 4)) * hw + pix;
      p_hi[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
      p_hi[hw] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
      p_f8[0] = make_uint4(l8[0], l8[1], l8[2], l8[3]);
      p_f8[hw] = make_uint4(h8[0], h8[1], h8[2], h8[3]);
      return live;
    } else {
#pragma unroll
      for (int q = 0; q < 16; q += 8) {  // one 8-channel plane at a time
        const int c = ch + q;
        if (c >= g.cout) break;
        uint32_t hi[4], lo[4];
        uint32_t mask[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
        if constexpr (EPI == kEpiDgrad) {
          if (g.mask_base) {  // no mask: gradient with respect to the network input (no ReLU in front)
            const uint4 m = g.mask_base[((size_t)n * 2 * g.mask_planes_half + (c >> 3)) * hw + pix];
            mask[0] = m.x; mask[1] = m.y; mask[2] = m.z; mask[3] = m.w;
          }
        }
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
          float f0, f1;
          if constexpr (EPI == kEpiDgrad) {  // ReLU': pass the gradient where the activation was > 0
            f0 = (mask[j >> 1] & 0x0000ffffu) ? f[q + j] : 0.f;
            f1 = (mask[j >> 1] & 0xffff0000u) ? f[q + j + 1] : 0.f;
          } else {
            f0 = fmaxf(f[q + j] + s_bias[c + j], 0.f);
            f1 = fmaxf(f[q + j + 1] + s_bias[c + j + 1], 0.f);
            if constexpr (RAG) {
              f0 = valid ? f0 : 0.f;
              f1 = valid ? f1 : 0.f;
            }
          }
          if constexpr (HI) {
            const __nv_bfloat162 hb = __floats2bfloat162_rn(f0, f1);
            hi[j >> 1] = *reinterpret_cast<const uint32_t*>(&hb);
            lo[j >> 1] = 0u;
          } else {
            split_bf16x2(f0, f1, hi[j >> 1], lo[j >> 1]);
          }
        }
        const bool second = c >= g.split_c;
        const ActDst& d = second ? g.dst1 : g.dst0;
        const int plane = (second ? c - g.split_c : c) >> 3;
        uint4* p_hi = d.base + ((size_t)n * 2 * d.planes_half + plane) * hw + pix;
        p_hi[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
        p_hi[(size_t)d.planes_half * hw] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
      }
    }
  } else {
    if (ch != 0) return 0u;
    const size_t o = (size_t)n * 3 * hw + pix;
    if constexpr (EPI == kEpiSigmoid) {
#pragma unroll
      for (int c = 0; c < 3; c++) g.out_f32[o + c * hw] = 1.0f / (1.0f + expf(-(f[c] + s_bias[c])));
    } else {  // kEpiGate: columns 3r+c = refiner r, colour c  (net.py:104-108)
      float r[9];
#pragma unroll
      for (int j = 0; j < 9; j++) r[j] = fmaxf(f[j] + s_bias[j], 0.f);
      if (g.refined_out) {
#pragma unroll
        for (int j = 0; j < 9; j++) g.refined_out[(size_t)n * 9 * hw + pix + j * hw] = r[j];
      }
      if (g.cm) {
        const float c0 = g.cm[o], c1 = g.cm[o + hw], c2 = g.cm[o + 2 * hw];
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; c++)
          v[c] = __fadd_rn(__fadd_rn(__fmul_rn(r[c], c0), __fmul_rn(r[3 + c], c1)), __fmul_rn(r[6 + c], c2));
        size_t oo = o, ohw = hw, o8 = ((size_t)n * hw + pix) * 3;
        float* out_f32 = g.out_f32;
        uint8_t* out_u8 = g.out_u8;
        if constexpr (RAG) {  // slot pixel -> pixel of the window's own image; only the kept rectangle is stored
          const RaggedWindow& t = g.rwin[n];
          const int y = t.ys + gy, x = t.xs + gx;
          if (y < t.ky0 || y >= t.ky1 || x < t.kx0 || x >= t.kx1) return 0u;
          ohw = (size_t)t.H * t.W;
          oo = (size_t)y * t.W + x;
          o8 = oo * 3;
          out_f32 = t.out_f32;
          out_u8 = t.out_u8;
        } else if (g.tiled) {  // window pixel -> image pixel; the halo around the kept rectangle is not stored
          const TileWindow t = tile_window(g.tiles, g.win0 + n);
          const int y = t.ys + gy, x = t.xs + gx;
          if (y < t.ky0 || y >= t.ky1 || x < t.kx0 || x >= t.kx1) return 0u;
          ohw = (size_t)g.tiles.H * g.tiles.W;
          const size_t ipix = (size_t)y * g.tiles.W + x;
          oo = (size_t)t.img * 3 * ohw + ipix;
          o8 = ((size_t)t.img * ohw + ipix) * 3;
        }
        if (out_f32) {
#pragma unroll
          for (int c = 0; c < 3; c++) out_f32[oo + c * ohw] = v[c];
        }
        if (out_u8) {  // ten2arr (hubconf.py:24-34): clip to [0,1], *255, truncate; NHWC
          uint8_t* q = out_u8 + o8;
#pragma unroll
          for (int c = 0; c < 3; c++) q[c] = (uint8_t)(int)__fmul_rn(fminf(fmaxf(v[c], 0.0f), 1.0f), 255.0f);
        }
      }
    }
  }
  return 0u;
}

// RAG: a pass of a ragged batch (ConvArgs::rwin).  Work item t is pixel tile t / NG, column group t % NG, so the
// groups of one pixel tile run on neighbouring CTAs at the same time and share its halo loads in L2.
template <int KS, int CIN_PAD, int NPAD, int EPI, int CONCAT, int NBLK, int TPS, int FMT = 0, bool RAG = false,
          int MW = 1, int NG = 1, int WGS = 2>
__global__ void __launch_bounds__(WGS == 2 ? 320 : 512, 1)
conv_umma_kernel(const __grid_constant__ CUtensorMap tmap_in, const ConvArgs g) {
  using C = UmmaCfg<KS, CIN_PAD, NPAD, CONCAT, NBLK, TPS, FMT, MW, NG, WGS>;
  constexpr bool F8IN = C::F8IN, DUAL = C::DUAL, OUT8 = (FMT & kFmtOut8) != 0;
  static_assert(!OUT8 || EPI == kEpiAct, "fp8 planes are written by the activation epilogue only");
  static_assert(!RAG || EPI == kEpiAct || EPI == kEpiGate, "ragged passes mask activations and store the gate");
  if (g.run_if != nullptr && *reinterpret_cast<const volatile int*>(g.run_if) == 0) return;  // whole grid alike
  if constexpr (F8IN)  // the producer of this launch's fp8 planes has completed (stream order): check its low end
    if (g.f8_live_in != nullptr && blockIdx.x == 0 && threadIdx.x == 0) {
      const unsigned w = atomicAnd(g.f8_live_in, ~g.f8_live_clear);
      if (w & ~(w >> 1) & g.f8_live_need) atomicOr(g.f8_overflow, 1);
    }
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a_stages = smem;
  uint8_t* b_stages = smem + C::NA * C::A_STAGE;
  float* staging = reinterpret_cast<float*>(b_stages + C::NB * C::B_STAGE);
  uint8_t* tail = reinterpret_cast<uint8_t*>(staging) + C::STAGING;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(tail);
  uint64_t* a_empty = a_full + C::NA;
  uint64_t* b_full = a_empty + C::NA;
  uint64_t* b_empty = b_full + C::NB;
  float* s_bias = reinterpret_cast<float*>(tail + 512);
  static_assert((2 * 6 + 2 * 8) * 8 <= 512 && C::BIAS_BYTES <= C::TAIL - 512, "barrier / bias area");

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int num_tiles = g.num_tiles;
  if (tid == 0) {
    for (int i = 0; i < C::NA; i++) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], C::CONSUMER_WARPS); }
    for (int i = 0; i < C::NB; i++) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], C::CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < NG * NBLK * NPAD; i += C::THREADS) s_bias[i] = g.bias[i];
  if constexpr (C::PAIR)
    for (int i = tid; i < NPAD; i += C::THREADS) s_bias[NPAD + i] = g.f8_scale[i];
  if constexpr (C::FUSE)
    for (int i = tid; i < kFuseNpad; i += C::THREADS) s_bias[NPAD + i] = g.bias1x1[i];
  __syncthreads();
  // kFmtPair8: the tap-pair form runs on tiles of 8-bit levels (decided per call on the device, like the a_lo pass,
  // or per image with slot_levels); the B producer and the consumers take the same decision
  const bool levels = (g.skip_lo != nullptr && *g.skip_lo != 0) || g.a_hi_only;
  auto pair_tile = [&](int tile) {
    if (!C::PAIR) return false;
    if (g.a_hi_only || g.slot_levels == nullptr) return levels;
    return g.slot_levels[tile / NG / (g.tiles_x * g.tiles_y)] != 0;
  };
  // WGS = 3: the producer warpgroup gives registers up, the consumer warpgroups take them; each setmaxnreg sits at
  // one place that dominates the code of its role, so that ptxas compiles the consumers for kWgs3ConsumerRegs
  if constexpr (WGS == 3) {
    if (warp >= C::CONSUMER_WARPS) {
      asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kWgs3ProducerRegs));
      if (warp > C::WARP_B) return;  // warps 14-15 only complete the producer warpgroup
    }
  }
  if (warp == C::WARP_A) {
    // ===================== A producer: halo tiles by TMA =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int pt = tile / NG;
        const int n = pt / (g.tiles_x * g.tiles_y);
        const int rem = pt - n * g.tiles_x * g.tiles_y;
        const int ty = rem / g.tiles_x, tx = rem - ty * g.tiles_x;
        const int x0 = tx * C::TILE_W - KS / 2, y0 = ty * C::TILE_H - KS / 2;
        for (int c = 0; c < C::NCHUNK; c++) {
          mbar_wait(&a_empty[stage], phase ^ 1);
          uint8_t* dst = a_stages + stage * C::A_STAGE;
          if constexpr (F8IN) {  // step c < NCHUNK / 2: the fp8 planes of chunks 2c, 2c + 1; then their hi planes
            mbar_expect_tx(&a_full[stage], 4 * C::PLANE_BYTES);
            const int plane = c < C::NCHUNK / 2 ? g.in_planes_half + 4 * c : 4 * (c - C::NCHUNK / 2);
            tma_load_5d(dst, &tmap_in, &a_full[stage], 0, x0, y0, plane, n);
            tma_load_5d(dst + 2 * C::PLANE_BYTES, &tmap_in, &a_full[stage], 0, x0, y0, plane + 2, n);
          } else {
            // kFmtHi never reads the lo planes
            mbar_expect_tx(&a_full[stage], (C::HI || g.a_hi_only ? 2 : 4) * C::PLANE_BYTES);
            tma_load_5d(dst, &tmap_in, &a_full[stage], 0, x0, y0, 2 * c, n);
            if (!C::HI && !g.a_hi_only)
              tma_load_5d(dst + 2 * C::PLANE_BYTES, &tmap_in, &a_full[stage], 0, x0, y0, g.in_planes_half + 2 * c, n);
          }
          if (++stage == C::NA) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }
  if (warp == C::WARP_B) {
    // ===================== B producer: packed weight stages =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      auto send = [&](const uint8_t* src, uint32_t bytes) {
        mbar_wait(&b_empty[stage], phase ^ 1);
        mbar_expect_tx(&b_full[stage], bytes);
        bulk_load(b_stages + stage * C::B_STAGE, src, bytes, &b_full[stage]);
        if (++stage == C::NB) { stage = 0; phase ^= 1; }
      };
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const bool pair = pair_tile(tile);
        const uint8_t* wpk = pair ? g.wpk8 : g.wpk + (size_t)(tile % NG) * C::GROUP_BYTES;
        const int nit = pair ? C::PAIR_STAGES : C::NCHUNK * C::NSTAGE_PER_CHUNK;
        for (int it = 0; it < nit; it++) send(wpk + (size_t)it * C::B_STAGE, C::B_STAGE);
        if constexpr (C::FUSE)  // then the fused 1x1 layer's whole image, kFuseStages more stages through the same ring
          for (int it = 0; it < kFuseStages; it++) send(g.wpk1x1 + (size_t)it * C::FUSE_STAGE, C::FUSE_STAGE);
      }
    }
    return;
  }
  if constexpr (WGS == 3) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kWgs3ConsumerRegs));

  // ===================== consumers: wgmma, then the epilogue of the warpgroup's 64 rows =====================
  const int wg = warp >> 2, wtid = tid & 127;
  const bool skip_lo = levels;
  // A operand: rows of the tile = pixels, 8 consecutive pixels of a halo row = one core matrix; this warpgroup's
  // rows start 8 halo rows further, its second m64 block 8 pixels (128 B) further along the same halo rows.  K halves
  // (channels 0-7 / 8-15 of the chunk) are one plane apart.
  constexpr uint32_t kSboA = C::HALO_W * 16;
  constexpr uint32_t kLboB = (CONCAT ? 2 * NPAD : NPAD) * 16;
  float acc[MW][C::ACC];
  int astage = 0, bstage = 0, pend_a = -1, pend_b = -1;
  uint32_t aphase = 0, bphase = 0;
  // a stage may be refilled once the wgmma groups reading it have completed: the release of a stage waits for
  // the NEXT stage's group to be issued (wait_group 1), so that the tensor core always has one group queued
  auto release = [&]() {
    if (lane == 0) {
      if (pend_b >= 0) mbar_arrive(&b_empty[pend_b]);
      if (pend_a >= 0) mbar_arrive(&a_empty[pend_a]);
    }
    pend_a = pend_b = -1;
  };
  unsigned live = 0u;  // OUT8: ConvArgs::f8_live bits of every value this thread stores
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const bool pair = pair_tile(tile);
#pragma unroll
    for (int mb = 0; mb < MW; mb++) {
#pragma unroll
      for (int i = 0; i < C::ACC; i++) acc[mb][i] = 0.f;
    }
    // unrolled: the diagonal block a chunk feeds (which accumulator registers its wgmmas write) is a constant.
    // F8IN: step c is chunk pair c % (NCHUNK / 2) of the correction phase (c < NCHUNK / 2), then of the main phase:
    // every e4m3 wgmma of the tile comes first, so that while the fp8 MMA, which adds with fewer bits than fp32, adds
    // into the accumulator, it holds only correction sums (about 2^-8 of the result)
#pragma unroll
    for (int c = 0; c < C::NCHUNK; c++) {
      const bool corr = F8IN && c < C::NCHUNK / 2;
      mbar_wait(&a_full[astage], aphase);
      const uint32_t a_base = smem_u32(a_stages + astage * C::A_STAGE) + (uint32_t)(wg * 8 * C::HALO_W * 16);
      const int blk = NBLK > 1 ? (F8IN ? 2 * (c % (C::NCHUNK / 2)) : c) / C::CPB : 0;
      if constexpr (C::PAIR) {
        if (pair) {
          // the e4m3 operand: warpgroup wg converts the two hi planes of its 14 halo rows (8 wg ..) into plane 2 + wg
          // of the stage, at the same offsets (those planes hold lo planes or nothing, unused when the inputs are
          // levels); then the async proxy may read them
          uint8_t* st = a_stages + astage * C::A_STAGE;
          for (int p = wtid; p < (8 + KS - 1) * C::HALO_W; p += 128) {
            const size_t o = (size_t)(wg * 8 * C::HALO_W + p) * 16;
            const uint4 h0 = *reinterpret_cast<const uint4*>(st + o);
            const uint4 h1 = *reinterpret_cast<const uint4*>(st + C::PLANE_BYTES + o);
            const uint32_t hw[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
            uint32_t q[4];
#pragma unroll
            for (int j = 0; j < 4; j++)
              q[j] = pack_e4m3x4(__uint_as_float(hw[2 * j] << 16), __uint_as_float(hw[2 * j] & 0xffff0000u),
                                 __uint_as_float(hw[2 * j + 1] << 16), __uint_as_float(hw[2 * j + 1] & 0xffff0000u));
            *reinterpret_cast<uint4*>(st + (2 + wg) * C::PLANE_BYTES + o) = make_uint4(q[0], q[1], q[2], q[3]);
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          wg_bar(1 + wg);
        }
      }
      // one weight stage: wait for it, issue its wgmmas (body), commit; its release waits for the next stage's group
      auto stage = [&](bool last_of_chunk, auto&& body) {
        mbar_wait(&b_full[bstage], bphase);
        const uint32_t b_base = smem_u32(b_stages + bstage * C::B_STAGE);
        wg_fence();
        body(b_base);
        wg_commit();
        wg_wait<1>();
        release();
        pend_b = bstage;
        if (last_of_chunk) pend_a = astage;
        if (++bstage == C::NB) { bstage = 0; bphase ^= 1; }
      };
      bool issued = false;
      if constexpr (C::PAIR) {
        if (pair) {
          // unrolled, so that each unit's wgmma is known at compile time (ptxas serialises wgmmas behind a branch
          // on the unit index)
#pragma unroll
          for (int tg = 0; tg < C::PAIR_STAGES; tg++) {
            stage(tg == C::PAIR_STAGES - 1, [&](uint32_t b_base) {
              // units 2 tg, 2 tg + 1 of [25 e4m3 pairs | 49 bf16 taps].  Pair p: taps t0 = min(2p, 47) and t0 + 1, one
              // descriptor from tap t0 with LBO = the distance to tap t0 + 1 (16 B along a kernel row, one halo row
              // minus 6 pixels across rows); pair 24 is taps 47 (zero weights) and 48, so that no read leaves the rows
              // of the warpgroup.  Every wgmma has N = NPAD, B = [K half][NPAD rows][16 B], LBO NPAD * 16.
#pragma unroll
              for (int j = 0; j < 2; j++) {
                const int u = 2 * tg + j;
                const uint32_t b_unit = b_base + (uint32_t)(j * NPAD * 32);
                if (u < C::PAIRS) {
                  const int t0 = 2 * u < KS * KS - 2 ? 2 * u : KS * KS - 2, t1 = t0 + 1;
                  const uint32_t o0 = (uint32_t)(((t0 / KS) * C::HALO_W + t0 % KS) * 16);
                  const uint32_t o1 = (uint32_t)(((t1 / KS) * C::HALO_W + t1 % KS) * 16);
                  // (N = 32 where the form is compiled out: the e4m3 shapes other layers need are generated)
                  const uint32_t a_pair = a_base + (2 + wg) * C::PLANE_BYTES + o0;
                  wgmma_e4m3<C::PAIR ? NPAD : 32>(acc[0], make_desc(a_pair, o1 - o0, kSboA), make_desc(b_unit, NPAD * 16, 128));
                } else {
                  const int tap = u - C::PAIRS;
                  const uint32_t a_tap = a_base + (uint32_t)(((tap / KS) * C::HALO_W + tap % KS) * 16);
                  wgmma_bf16<NPAD>(acc[0], make_desc(a_tap, C::PLANE_BYTES, kSboA), make_desc(b_unit, NPAD * 16, 128));
                }
              }
            });
          }
          issued = true;
        }
      }
      if (!issued) {
        for (int tg = 0; tg < C::NSTAGE_PER_CHUNK; tg++) {
          stage(tg == C::NSTAGE_PER_CHUNK - 1, [&](uint32_t b_base) {
#pragma unroll
            for (int t = 0; t < TPS; t++) {
              const int tap = tg * TPS + t;
              const int ky = tap / KS, kx = tap - ky * KS;
              const uint32_t a_tap = a_base + (uint32_t)((ky * C::HALO_W + kx) * 16);
              const uint32_t b_tap = b_base + (uint32_t)(t * C::B_TAP);
              // MW = 2: block mb is the same descriptor 8 pixels further, as an add to the start-address field (that of a
              // shared-memory address never carries into the next field); fewer live descriptors than building each anew
              const uint64_t a_hi0 = make_desc(a_tap, C::PLANE_BYTES, kSboA);
#pragma unroll
              for (int mb = 0; mb < MW; mb++) {
                const uint64_t a_hi = a_hi0 + mb * (128 >> 4);
                const uint64_t a_lo = MW == 1 ? make_desc(a_tap + 2 * C::PLANE_BYTES, C::PLANE_BYTES, kSboA)
                                              : a_hi + ((2 * C::PLANE_BYTES) >> 4);
#pragma unroll
                for (int b = 0; b < NBLK; b++) {
                  if (NBLK > 1 && b != blk) continue;
                  float* d = acc[mb] + b * C::BLK_COLS / 2;
                  if constexpr (C::HI) {
                    wgmma_bf16<NPAD>(d, a_hi, make_desc(b_tap, kLboB, 128));                // a_hi x w_hi
                  } else if constexpr (F8IN) {
                    // chunk 2p (planes 0-1, a_hi) and chunk 2p + 1 (planes 2-3, a_lo) of the pair, each one of the
                    // phase's units: [e4m3(lo*2^9) | e4m3(v)] x [e4m3(w*ws) ; e4m3(w_lo*ws*2^9)] (K = 32), then
                    // a_hi x w_hi * ws * 2^9 (bf16, K = 16)
                    const uint32_t b_odd = b_tap + TPS * C::B_TAP;
                    if (corr) {
                      wgmma_e4m3<NPAD>(d, a_hi, make_desc(b_tap, NPAD * 16, 128));
                      wgmma_e4m3<NPAD>(d, a_lo, make_desc(b_odd, NPAD * 16, 128));
                    } else {
                      wgmma_bf16<NPAD>(d, a_hi, make_desc(b_tap, NPAD * 16, 128));
                      wgmma_bf16<NPAD>(d, a_lo, make_desc(b_odd, NPAD * 16, 128));
                    }
                  } else if constexpr (CONCAT) {
                    wgmma_bf16<2 * NPAD>(d, a_hi, make_desc(b_tap, kLboB, 128));            // a_hi x [w_hi | w_lo]
                    if (!skip_lo) wgmma_bf16<NPAD>(d, a_lo, make_desc(b_tap, kLboB, 128));  // a_lo x w_hi
                  } else {
                    wgmma_bf16<NPAD>(d, a_hi, make_desc(b_tap, kLboB, 128));                // a_hi x w_hi
                    if (!skip_lo) wgmma_bf16<NPAD>(d, a_lo, make_desc(b_tap, kLboB, 128));  // a_lo x w_hi
                    wgmma_bf16<NPAD>(d, a_hi, make_desc(b_tap + 2 * NPAD * 16, kLboB, 128));  // a_hi x w_lo
                  }
                }
              }
            }
          });
        }
      }
      if (++astage == C::NA) { astage = 0; aphase ^= 1; }
    }
    wg_wait<0>();
    release();

    // ---- epilogue: one m64 block at a time, 32 output channels at a time through shared memory.  The accumulator
    // fragment gives a thread two channels of two rows per 8 columns; the epilogue wants a pixel's consecutive
    // channels in one thread.  Row r of block mb is pixel (8 mb + r % 8, 8 wg + r / 8) of the tile.
    const int pt = tile / NG, c0 = (tile % NG) * NPAD;
    const int n = pt / (g.tiles_x * g.tiles_y);
    const int rem = pt - n * g.tiles_x * g.tiles_y;
    const int ty = rem / g.tiles_x, tx = rem - ty * g.tiles_x;
    float* stg = staging + wg * 64 * kStageLd;
    const int frow = (warp & 3) * 16 + (lane >> 2), fcol = (lane & 3) * 2;
    const int r = wtid & 63, half = wtid >> 6;
    const int m = wg * 64 + r;
    const int gy = ty * C::TILE_H + (m >> 3);
    const float dscale = F8IN ? *g.f8_scale : 1.f;
    // kFmtFuse1x1: the fused layer's A operands (hi / lo, 4 registers per K step) and the ring stages of its weights
    static_assert(!C::FUSE || kFuseNpad <= C::ACC, "the fused layer's accumulators take the place of this layer's");
    uint32_t a_hi[C::FUSE ? NPAD / 4 : 1], a_lo[C::FUSE ? NPAD / 4 : 1];
    int fuse_stage[kFuseStages];
    if constexpr (C::FUSE) {
      // This layer's activation in the accumulator layout, with the fp32 operations of its kEpiAct epilogue (max(acc
      // dscale + b, 0), or max(acc + b, 0); __fmul_rn / __fadd_rn so that nothing contracts into an fma),
      // masked as a ragged slot masks it, and split into the bf16 hi / lo the 1x1 layer's own launch reads.  Register
      // 2j + h holds columns 8j + fcol, +1 of row frow + 8h: registers 4k .. 4k + 3 are the A fragment of K step k.
      bool row_valid[2] = {true, true};
      if constexpr (RAG) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int mh = wg * 64 + frow + 8 * h;
          row_valid[h] = tx * C::TILE_W + (mh & 7) < g.rwin[n].vw && ty * C::TILE_H + (mh >> 3) < g.rwin[n].vh;
        }
      }
#pragma unroll
      for (int j = 0; j < NPAD / 8; j++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
          float x[2];
#pragma unroll
          for (int e = 0; e < 2; e++) {
            float s = acc[0][4 * j + 2 * h + e];
            if constexpr (F8IN) s = __fmul_rn(s, dscale);
            x[e] = fmaxf(__fadd_rn(s, s_bias[8 * j + fcol + e]), 0.f);
            if constexpr (RAG) x[e] = row_valid[h] ? x[e] : 0.f;
          }
          split_bf16x2(x[0], x[1], a_hi[2 * j + h], a_lo[2 * j + h]);
        }
      }
      // its weight stages (the B producer sends them behind this tile's): released once the epilogue is done
#pragma unroll
      for (int s = 0; s < kFuseStages; s++) {
        mbar_wait(&b_full[bstage], bphase);
        fuse_stage[s] = bstage;
        if (++bstage == C::NB) { bstage = 0; bphase ^= 1; }
      }
    }
    // the epilogue stores this layer's output, or the fused 1x1 layer's (its biases follow this layer's)
    constexpr bool EDUAL = DUAL || C::FUSE, EF8 = F8IN && !C::FUSE;
    constexpr int ENPAD = C::FUSE ? kFuseNpad : NPAD;
    constexpr int NCH = C::FUSE ? kFuseNpad : NBLK * NPAD;
    const float* e_bias = C::FUSE ? s_bias + NPAD : s_bias;
#pragma unroll
    for (int mb = 0; mb < MW; mb++) {
      const int gx = tx * C::TILE_W + mb * 8 + (m & 7);
      const bool inside = gx < g.W && gy < g.H;
      bool valid = true;
      if constexpr (RAG) valid = gx < g.rwin[n].vw && gy < g.rwin[n].vh;
#pragma unroll
      for (int ch0 = 0; ch0 < NCH; ch0 += 32) {
        if constexpr (C::FUSE) {
          // the fused layer's output channels [ch0, ch0 + 32), into the registers of its columns in a CONCAT launch's
          // accumulators (w_hi products at ch0, w_lo products at kFuseNpad + ch0): per chunk the N = 32 column blocks
          // a_hi x w_hi, a_hi x w_lo, a_lo x w_hi -- per column the products and the order of that launch's
          // a_hi x [w_hi | w_lo], a_lo x w_hi.  32 accumulators at a time beside the 64 A registers.
          float* d_hi = acc[0] + ch0 / 2;
          float* d_lo = acc[0] + (kFuseNpad + ch0) / 2;
#pragma unroll
          for (int i = 0; i < 16; i++) d_hi[i] = d_lo[i] = 0.f;
          wg_fence();
#pragma unroll
          for (int k = 0; k < NPAD / 16; k++) {
            const uint32_t b_hi = smem_u32(b_stages + fuse_stage[k / C::FUSE_CHUNKS] * C::B_STAGE) +
                                  (uint32_t)((k % C::FUSE_CHUNKS) * kFuseNpad * 64 + ch0 * 16);
            const uint32_t b_lo = b_hi + kFuseNpad * 16;
            wgmma_bf16_rs<32>(d_hi, a_hi + 4 * k, make_desc(b_hi, 2 * kFuseNpad * 16, 128));  // a_hi x w_hi
            wgmma_bf16_rs<32>(d_lo, a_hi + 4 * k, make_desc(b_lo, 2 * kFuseNpad * 16, 128));  // a_hi x w_lo
            wgmma_bf16_rs<32>(d_hi, a_lo + 4 * k, make_desc(b_hi, 2 * kFuseNpad * 16, 128));  // a_lo x w_hi
          }
          wg_commit();
          wg_wait<0>();
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const int ch = ch0 + 8 * j;
          if (ch < NCH) {
            const int col = NBLK > 1 ? (ch / NPAD) * C::BLK_COLS + ch % NPAD : ch;
            float v[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
              v[k] = acc[mb][col / 2 + k];
              if constexpr (EDUAL) v[k] += acc[mb][(col + ENPAD) / 2 + k];
              if constexpr (EF8) v[k] = v[k] * dscale;
              if constexpr (C::PAIR) v[k] = pair ? v[k] * s_bias[NPAD + col + fcol + (k & 1)] : v[k];
            }
            float* s = stg + frow * kStageLd + 8 * j + fcol;
            *reinterpret_cast<float2*>(s) = make_float2(v[0], v[1]);
            *reinterpret_cast<float2*>(s + 8 * kStageLd) = make_float2(v[2], v[3]);
          }
        }
        wg_bar(1 + wg);
        const int cb = ch0 + 16 * half;
        if (cb < NCH && inside) {
          float f[16];
          const float4* s = reinterpret_cast<const float4*>(stg + r * kStageLd + 16 * half);
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const float4 x = s[q];
            f[4 * q] = x.x; f[4 * q + 1] = x.y; f[4 * q + 2] = x.z; f[4 * q + 3] = x.w;
          }
          live |= epilogue16<EPI, OUT8, RAG, C::HI>(g, e_bias, f, c0 + cb, n, gx, gy, valid);
        }
        wg_bar(1 + wg);
      }
    }
    if constexpr (C::FUSE)
      if (lane == 0)
#pragma unroll
        for (int s = 0; s < kFuseStages; s++) mbar_arrive(&b_empty[fuse_stage[s]]);
  }
  if constexpr (OUT8) {  // the low-end record of what this warp stored: one atomic per warp
    live = __reduce_or_sync(0xffffffffu, live);
    if (lane == 0 && live != 0u && g.f8_live != nullptr) atomicOr(g.f8_live, live);
  }
}

// ------------------------------------------------------------------------------------------
// Operand packing kernels
// ------------------------------------------------------------------------------------------
// scatter one OIHW fp32 tensor into a dense [npad][cinpad][ks*ks] fp32 block-matrix
static __global__ void scatter_weights_kernel(const float* __restrict__ src, float* __restrict__ dense, int co, int ci,
                                       int kk, int cinpad, int row_off, int split, int base0, int base1,
                                       float divisor) {
  const int total = co * ci * kk;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int t = i % kk;
    int c = (i / kk) % ci;
    int o = i / (kk * ci);
    int cd = c < split ? base0 + c : base1 + (c - split);
    dense[((size_t)(row_off + o) * cinpad + cd) * kk + t] = __fdiv_rn(src[i], divisor);
  }
}
static __global__ void scatter_bias_kernel(const float* __restrict__ src, float* __restrict__ dst, int co, int row_off) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < co; i += gridDim.x * blockDim.x) dst[row_off + i] = src[i];
}
// dense fp32 [nblk*npad][cinpad][kk] -> weight stages, one per (chunk, tap), holding the rows of the
// diagonal block the chunk feeds:  concat ? [k8][hi rows | lo rows][8] : [hi|lo][k8][rows][8]   (bf16)
// row_off: the stages of one column group (UmmaCfg NG) hold dense rows [row_off, row_off + npad)
static __global__ void pack_stages_kernel(const float* __restrict__ dense, __nv_bfloat16* __restrict__ out, int npad,
                                   int cinpad, int kk, int concat, int nblk, int row_off = 0) {
  const int nchunk = cinpad / 16, cpb = nchunk / nblk;
  const size_t total = (size_t)nchunk * kk * 2 * 2 * npad * 8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int e = (int)(i % 8);
    size_t r = i / 8;
    int k8, split, nrow;
    if (concat) {
      int row2 = (int)(r % (2 * npad)); r /= 2 * npad;
      k8 = (int)(r % 2); r /= 2;
      split = row2 >= npad;
      nrow = row2 - split * npad;
    } else {
      nrow = (int)(r % npad); r /= npad;
      k8 = (int)(r % 2); r /= 2;
      split = (int)(r % 2); r /= 2;
    }
    int tap = (int)(r % kk);
    int chunk = (int)(r / kk);
    int cin = chunk * 16 + k8 * 8 + e;
    int row = row_off + (chunk / cpb) * npad + nrow;
    float w = dense[((size_t)row * cinpad + cin) * kk + tap];
    __nv_bfloat16 hi = __float2bfloat16_rn(w);
    out[i] = split == 0 ? hi : __float2bfloat16_rn(w - __bfloat162float(hi));
  }
}


// fp8 correction scheme (UmmaCfg FMT bit 0): units of rows * 32 B in the order the two phases of a tile read them,
//   first one per (chunk, tap):  [k16 0|1][rows][16 fp8 (e4m3)]    w * ws  |  w_lo * ws * 2^9   (K = 32 fp8 MMA)
//   then one per (chunk, tap):   [k8 0|1][rows][8 bf16]            w_hi * ws * 2^9              (K = 16 bf16 MMA)
// Within a phase, unit (chunk, tap) is at ((pair * kk / tps + tap / tps) * 2 + chunk % 2) * tps + tap % tps, pair =
// chunk / 2: a weight stage is tps taps of chunk 2 pair, then the same taps of chunk 2 pair + 1.
// with rows = npad (dense rows from row_off on: one column group).  scale[0] = ws (a power of two placing max|w| in
// [112, 224] over the whole layer),
// scale[1] = 2^-9 / ws (what the epilogue multiplies the accumulator with); scale[2] = max|w|.
// scale[2] (as unsigned bits) accumulates max|w| over the grid (bit patterns of non-negative floats are
// ordered like the floats); f8_scale_finish_kernel turns it into scale[0], scale[1].
static __global__ void f8_absmax_kernel(const float* __restrict__ dense, size_t n, float* __restrict__ scale) {
  __shared__ float smax[256];
  float m = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(dense[i]));
  smax[threadIdx.x] = m;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) smax[threadIdx.x] = fmaxf(smax[threadIdx.x], smax[threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x == 0) atomicMax(reinterpret_cast<unsigned int*>(scale + 2), __float_as_uint(smax[0]));
}
static __global__ void f8_scale_finish_kernel(float* __restrict__ scale) {
  const float mx = fmaxf(scale[2], 1e-30f);
  const float ws = exp2f(floorf(log2f(224.f / mx)));
  scale[0] = ws;
  scale[1] = 1.f / (512.f * ws);
}
static __global__ void pack_stages_f8_kernel(const float* __restrict__ dense, uint8_t* __restrict__ out,
                                             const float* __restrict__ scale, int npad, int cinpad, int kk, int tps,
                                             int nblk, int row_off) {
  const int nchunk = cinpad / 16, cpb = nchunk / nblk, rows = npad;
  const size_t unit_bytes = (size_t)rows * 32;
  const float ws = scale[0];
  // one thread per (chunk, tap, row, channel pair of the chunk)
  const size_t total = (size_t)nchunk * kk * rows * 8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    size_t r = i;
    const int cp = (int)(r % 8); r /= 8;            // channels 2cp, 2cp+1 of the chunk
    const int row = (int)(r % rows); r /= rows;
    const int tap = (int)(r % kk);
    const int chunk = (int)(r / kk);
    const int wrow = row_off + (chunk / cpb) * npad + row;
    float w[2], wl[2];
    uint16_t hb[2];
#pragma unroll
    for (int t = 0; t < 2; t++) {
      w[t] = dense[((size_t)wrow * cinpad + chunk * 16 + 2 * cp + t) * kk + tap];
      const __nv_bfloat16 h = __float2bfloat16_rn(w[t]);
      hb[t] = __bfloat16_as_ushort(h);
      wl[t] = w[t] - __bfloat162float(h);
    }
    const size_t unit = ((size_t)(chunk / 2) * (kk / tps) + tap / tps) * 2 * tps + (chunk % 2) * tps + tap % tps;
    uint8_t* base = out + ((size_t)nchunk * kk + unit) * unit_bytes;
    // bf16 unit: channel c = 2cp+t -> k8 = c / 8, element c % 8.  bf16(w) * (ws * 2^9): an exact power-of-two scaling
    // that puts the bf16 product on the scale of the fp8 correction product (one shared accumulator)
    const int c = 2 * cp;
#pragma unroll
    for (int t = 0; t < 2; t++)
      hb[t] = __bfloat16_as_ushort(__float2bfloat16_rn(__bfloat162float(__ushort_as_bfloat16(hb[t])) * ws * 512.f));
    *reinterpret_cast<uint32_t*>(base + ((size_t)(c / 8) * rows + row) * 16 + (c % 8) * 2) =
        (uint32_t)hb[0] | ((uint32_t)hb[1] << 16);
    // e4m3 unit: K half 0 = e4m3(w * ws), K half 1 = e4m3(w_lo * ws * 512), 16 channels per row
    uint8_t* p1 = out + unit * unit_bytes;
    *reinterpret_cast<uint16_t*>(p1 + ((size_t)0 * rows + row) * 16 + c) = pack_e4m3x2(w[0] * ws, w[1] * ws);
    *reinterpret_cast<uint16_t*>(p1 + ((size_t)1 * rows + row) * 16 + c) =
        pack_e4m3x2(wl[0] * ws * 512.f, wl[1] * ws * 512.f);
  }
}

// kFmtPair8 (the first layer): per output column (dense row) c, scale[c] = s_c = 2^floor(log2(224 / max|w_c|)) and
// scale[npad + c] = 2^-9 / s_c, what the epilogue multiplies column c with.  One block per column.
static __global__ void pair_scale_kernel(const float* __restrict__ dense, float* __restrict__ scale, int npad, int n) {
  __shared__ float smax[256];
  float m = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(dense[(size_t)blockIdx.x * n + i]));
  smax[threadIdx.x] = m;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) smax[threadIdx.x] = fmaxf(smax[threadIdx.x], smax[threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float s = exp2f(floorf(log2f(224.f / fmaxf(smax[0], 1e-30f))));
    scale[blockIdx.x] = s;
    scale[npad + blockIdx.x] = 1.f / (512.f * s);
  }
}
// The tap-pair weight image of a 16-channel layer (dense [npad][16][kk]): units of npad * 32 B,
//   units 0 .. (kk + 1) / 2 - 1   pair p:  [K half 0|1][rows][16 e4m3]  e4m3(w_lo s_c 2^9) of taps t0, t0 + 1
//                                 (t0 = min(2p, kk - 2); half 0 of the last pair is zero when kk is odd)
//   then one unit per tap t:      [k8 0|1][rows][8 bf16]               bf16(w) s_c 2^9 (exact: a power of two)
// One thread per (unit, row).
static __global__ void pack_stages_pair_kernel(const float* __restrict__ dense, uint8_t* __restrict__ out,
                                               const float* __restrict__ scale, int npad, int kk) {
  const int pairs = (kk + 1) / 2, units = pairs + kk;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < units * npad; i += gridDim.x * blockDim.x) {
    const int u = i / npad, row = i - u * npad;
    const float s = scale[row] * 512.f;
    uint8_t* unit = out + (size_t)u * npad * 32;
    const float* w = dense + (size_t)row * 16 * kk;
    if (u < pairs) {
      const int t0 = 2 * u < kk - 2 ? 2 * u : kk - 2;
      for (int h = 0; h < 2; h++) {
        const int tap = t0 + h;
        const bool zero = h == 0 && 2 * u >= kk - 1;
        uint32_t q[4];
        for (int j = 0; j < 4; j++) {
          float f[4];
          for (int e = 0; e < 4; e++) {
            const float x = w[(4 * j + e) * kk + tap];
            f[e] = zero ? 0.f : (x - __bfloat162float(__float2bfloat16_rn(x))) * s;
          }
          q[j] = pack_e4m3x4(f[0], f[1], f[2], f[3]);
        }
        *reinterpret_cast<uint4*>(unit + ((size_t)h * npad + row) * 16) = make_uint4(q[0], q[1], q[2], q[3]);
      }
    } else {
      const int tap = u - pairs;
      for (int c = 0; c < 16; c++) {
        const float hi = __bfloat162float(__float2bfloat16_rn(w[c * kk + tap])) * s;
        *reinterpret_cast<__nv_bfloat16*>(unit + ((size_t)(c / 8) * npad + row) * 16 + (c % 8) * 2) =
            __float2bfloat16_rn(hi);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Host helpers
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;

static int get_encoder() {
  if (g_encode) return WN_OK;
  cudaDriverEntryPointQueryResult q;
  void* fn = nullptr;
  WN_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  if (!fn || q != cudaDriverEntryPointSuccess) {
    set_error("cuTensorMapEncodeTiled is not available from this driver");
    return WN_E_UNSUPPORTED;
  }
  g_encode = (EncodeTiledFn)fn;
  return WN_OK;
}

static int make_tmap(CUtensorMap* tm, void* base, int planes_total, int N, int H, int W, int halo_w, int halo_h) {
  cuuint64_t dims[5] = {8, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)planes_total, (cuuint64_t)N};
  cuuint64_t strides[4] = {16, (cuuint64_t)W * 16, (cuuint64_t)H * W * 16, (cuuint64_t)planes_total * H * W * 16};
  cuuint32_t box[5] = {8, (cuuint32_t)halo_w, (cuuint32_t)halo_h, 2, 1};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = g_encode(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with %d (planes=%d N=%d H=%d W=%d box=%dx%d)", (int)r, planes_total, N, H,
              W, halo_w, halo_h);
    return WN_E_CUDA;
  }
  return WN_OK;
}

// Launch one convolution.  `slot` is the timing slot (common.cuh).  One persistent CTA per SM (shared-memory footprint).
template <int KS, int CIN_PAD, int NPAD, int EPI, int CONCAT = 0, int NBLK = 1, int TPS = 1, int FMT = 0,
          bool RAG = false, int MW = 1, int NG = 1, int WGS = 2>
static int launch_conv(wn_handle* h, int slot, const uint8_t* wpk, const float* bias, void* in_base, ConvArgs a,
                       cudaStream_t stream) {
  using C = UmmaCfg<KS, CIN_PAD, NPAD, CONCAT, NBLK, TPS, FMT, MW, NG, WGS>;
  int rc = get_encoder();
  if (rc) return rc;
  CUtensorMap tm;
  rc = make_tmap(&tm, in_base, (a.a_hi_only ? 1 : 2) * (CIN_PAD / 8), a.N, a.H, a.W, C::HALO_W, C::HALO_H);
  if (rc) return rc;
  a.wpk = wpk;
  a.bias = bias;
  a.in_planes_half = CIN_PAD / 8;
  a.tiles_x = (a.W + C::TILE_W - 1) / C::TILE_W;
  a.tiles_y = (a.H + C::TILE_H - 1) / C::TILE_H;
  const long long tiles = (long long)a.tiles_x * a.tiles_y * a.N * NG;
  a.num_tiles = (int)tiles;
  auto kern = conv_umma_kernel<KS, CIN_PAD, NPAD, EPI, CONCAT, NBLK, TPS, FMT, RAG, MW, NG, WGS>;
  WN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
  TimedScope ts(h, slot, stream);
  const int grid = (int)(tiles < h->sm_count ? tiles : h->sm_count);
  kern<<<grid, C::THREADS, C::SMEM_BYTES, stream>>>(tm, a);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

}  // namespace wn
