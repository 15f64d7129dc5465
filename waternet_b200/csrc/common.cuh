// Shared declarations for the waternet_b200 CUDA library (sm_90a).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <initializer_list>
#include <vector>

#include "../../include/waternet_b200.h"
#include "../../include/waternet_b200_metrics.h"
#include "../../include/waternet_b200_ssim.h"
#include "tiling.cuh"

namespace wn {

void set_error(const char* fmt, ...);

// workspace sub-buffers start at 256-byte boundaries
inline size_t align256(size_t v) { return (v + 255) / 256 * 256; }

#define WN_CUDA(call)                                                                   \
  do {                                                                                  \
    cudaError_t err__ = (call);                                                         \
    if (err__ != cudaSuccess) {                                                         \
      wn::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(err__)); \
      return WN_E_CUDA;                                                                 \
    }                                                                                   \
  } while (0)

// The device table of a ragged call: its parts in device order, each at a 256-byte boundary.  The parts are filled
// in one host staging buffer in that layout and copied with one cudaMemcpyAsync; bytes() is the workspace they take.
class HostTable {
 public:
  HostTable(std::initializer_list<size_t> part_bytes) {
    for (size_t b : part_bytes) {
      len_[parts_] = b;
      off_[parts_ + 1] = off_[parts_] + align256(b);
      parts_++;
    }
  }
  size_t bytes() const { return off_[parts_]; }
  // part k of the staging buffer (zero-filled at first use) and of the device table at `table`
  template <class T> T* part(int k) {
    if (host_.empty()) host_.resize(bytes());
    return reinterpret_cast<T*>(host_.data() + off_[k]);
  }
  template <class T> T* dev(void* table, int k) const { return reinterpret_cast<T*>((uint8_t*)table + off_[k]); }
  // parts [first, end) -> the device table, from the start of part `first` to the last byte of part end - 1.
  // Pageable source: the copy is staged before cudaMemcpyAsync returns, so the table may go out of scope.
  int upload(void* table, cudaStream_t stream, int first = 0, int end = -1) {
    if (end < 0) end = parts_;
    if (host_.empty()) host_.resize(bytes());
    WN_CUDA(cudaMemcpyAsync(dev<uint8_t>(table, first), host_.data() + off_[first],
                            off_[end - 1] + len_[end - 1] - off_[first], cudaMemcpyHostToDevice, stream));
    return WN_OK;
  }

 private:
  static constexpr int kMaxParts = 4;
  size_t off_[kMaxParts + 1] = {}, len_[kMaxParts] = {};
  int parts_ = 0;
  std::vector<uint8_t> host_;
};

// the heights and widths of a ragged array (wn_ragged_tensors, wn_ragged_image)
template <class Img>
void ragged_sizes(const Img* images, int n, std::vector<int>* hs, std::vector<int>* ws) {
  hs->resize(n);
  ws->resize(n);
  for (int i = 0; i < n; i++) {
    (*hs)[i] = images[i].height;
    (*ws)[i] = images[i].width;
  }
}

#define WN_LAUNCH_CHECK(h)   \
  do {                       \
    (h)->launches++;         \
    WN_CUDA(cudaGetLastError()); \
  } while (0)

// ---- constant tables (OpenCV 8-bit Lab, gamma 0.7, u/255) -------------------
struct Tables {
  uint16_t gtab[256];    // sRGB decode, scaled 255*8
  uint16_t ctab[3072];   // Lab f(t), scaled 1<<15
  int16_t ytab[256];     // L -> Y, scaled 1<<14
  int16_t fytab[256];    // L -> f(Y), scaled 1<<14
  uint8_t igtab[4096];   // linear -> sRGB 8 bit
  uint8_t gamma[256];    // data.py:61-65 as a LUT
  float div255[256];     // float(u)/255.f
};

void build_tables_host(Tables* t);

// ---- network description (net.py:12-42, 62-70) ------------------------------
struct LayerDesc {
  int cin, cout, ks;
};
static const LayerDesc kCmg[8] = {{12, 128, 7}, {128, 128, 5}, {128, 128, 3}, {128, 64, 1},
                                  {64, 64, 7},  {64, 64, 5},   {64, 64, 3},   {64, 3, 3}};
static const LayerDesc kRef[3] = {{6, 32, 7}, {32, 32, 5}, {32, 3, 3}};
constexpr int kNumConvs = 17;  // 8 + 3*3, in state-dict order

struct SimtLayer {
  int cin, cout, cout_pad, ks;
  float* w;     // [cin][ks*ks][cout_pad]
  float* bias;  // [cout_pad]
};

struct UmmaWeights;  // conv_umma.cu
struct UmmaBwd;      // conv_bwd.cu
struct VggWeights;   // vgg.cu

// Optional per-kernel timing with CUDA events on the launching stream (bench.py's roofline leg).
enum TimingSlot {
  kSlotConv0 = 0,  // 0..16: the 17 convolutions in state-dict order (fused kernels use their first layer)
  kSlotPack = 17,  // input concat / operand packing
  kSlotGate = 18,  // sigmoid-gated weighted sum
  kSlotStats = 19,
  kSlotLuts = 20,
  kSlotApply = 21,
  kSlotPost = 22,
  kNumSlots = 23
};
// which part of WaterNet.forward a forward call evaluates (the reference's sub-modules are callable: net.py:45-56, :75-80)
enum FwdStack { kStackAll = 0, kStackCmg = 1, kStackRefiners = 2 };
struct Timing {
  static constexpr int kMax = 8192;
  bool on;
  int used, created;
  cudaEvent_t a[kMax], b[kMax];
  int slot[kMax];
};

}  // namespace wn

struct wn_handle {
  int device;
  uint64_t launches;
  wn::Tables* d_tables;
  bool packed;
  wn::SimtLayer simt[wn::kNumConvs];
  wn::UmmaWeights* umma;
  int sm_count;
  wn::Timing* timing;
  wn::UmmaBwd* bwd;
  long long chunk_pixels;  // cap on pixels per pass of the tensor-core forward (0 = default, wn_set_chunk_pixels)
  wn::VggWeights* vgg;     // the perceptual loss's VGG19 stages (wn_vgg_pack_weights)
  bool train_bf16;         // wn_set_train_mode(WN_MODE_BF16): the training calls run single-pass bf16 (kFmtHi)
};

namespace wn {

// Scope guard: records an event pair around the launches issued while it is alive.
struct TimedScope {
  Timing* t;
  int idx;
  cudaStream_t stream;
  TimedScope(wn_handle* h, int slot, cudaStream_t s) : t(h->timing), idx(-1), stream(s) {
    if (!t || !t->on || t->used >= Timing::kMax) return;
    idx = t->used;
    if (idx >= t->created) {
      if (cudaEventCreate(&t->a[idx]) != cudaSuccess || cudaEventCreate(&t->b[idx]) != cudaSuccess) {
        idx = -1;
        return;
      }
      t->created = idx + 1;
    }
    t->used++;
    t->slot[idx] = slot;
    cudaEventRecord(t->a[idx], stream);
  }
  ~TimedScope() {
    if (idx >= 0) cudaEventRecord(t->b[idx], stream);
  }
};

// preprocess.cu
size_t preprocess_workspace_bytes(int n, int h, int w);
int preprocess_u8(wn_handle* h, const uint8_t* rgb, int n, int height, int width, float* x,
                  float* wb, float* he, float* gc, uint8_t* wb_u8, uint8_t* he_u8, uint8_t* gc_u8,
                  void* workspace, size_t workspace_bytes, cudaStream_t stream);
int postprocess_u8(wn_handle* h, const float* out_nchw, uint8_t* out_nhwc, int n, int height,
                   int width, cudaStream_t stream);
size_t white_balance_gray_workspace_bytes(int n, int h, int w);
int white_balance_gray_u8(wn_handle* h, const uint8_t* gray, uint8_t* out, int n, int height, int width,
                          void* workspace, size_t workspace_bytes, cudaStream_t stream);
int resize_u8(wn_handle* h, const uint8_t* const* src, const int* src_h, const int* src_w, int n, uint8_t* dst,
              int dst_h, int dst_w, int swap_rb, cudaStream_t stream);
// transform + cat[x, wb, he, gc] straight into the first layer's operand planes: planes[n][2][H*W] of 16 B
// (8 bf16 levels 0..255: plane 0 = x.rgb wb.rgb he.rg, plane 1 = he.b gc.rgb 0 0 0 0)
int preprocess_u8_planes(wn_handle* h, const uint8_t* rgb, int n, int height, int width, uint4* planes,
                         void* workspace, size_t workspace_bytes, cudaStream_t stream);
// the same split in two for the tiled forward: the statistics and LUTs of all n images once, then the operand planes
// of `count` windows (win0, win0 + 1, ...) of `tiles` per pass, read from the full images at image coordinates
// (workspace: that of preprocess_u8_luts, untouched in between)
int preprocess_u8_luts(wn_handle* h, const uint8_t* rgb, int n, int height, int width, void* workspace,
                       size_t workspace_bytes, cudaStream_t stream);
// ... and for a ragged batch, where every image has its own size: the preprocess geometry of one image (CLAHE tile,
// clip limit, LUT scale, histogram slabs), and the statistics and LUTs of all n images from their device table (one
// stats and one LUT launch).  Workspace: that of preprocess_workspace_bytes(n, ...), untouched in between.
struct RaggedImage {
  const uint8_t* rgb;
  int H, W;
  int th, tw, clip;          // CLAHE tile and clip limit (PreGeom)
  int rows_per_slab, slabs;  // stats grid: slabs of tile rows per CLAHE tile
  float lut_scale;
};
static_assert(sizeof(RaggedImage) == 40, "RaggedImage: engine.RAGGED_IMAGE_BYTES restates this size");
RaggedImage ragged_image(const uint8_t* rgb, int height, int width);
int preprocess_u8_ragged_luts(wn_handle* h, int n, const RaggedImage* imgs, int max_slabs, void* workspace,
                              cudaStream_t stream);
// The operand planes of `count` slots of geo (tiling.cuh; zeros beyond each valid extent) from the LUTs of the n
// images above.  The image data of a slot: one record for a grid geometry (image i at rgb + i * H * W * 3), the
// device table of n records for a table geometry.  Defined for (GridGeom, RaggedImage) and (TableGeom, const
// RaggedImage*).
template <class Geom, class Img>
int preprocess_u8_slot_planes(wn_handle* h, const Geom& geo, const Img& imgs, int n, int count, uint4* planes,
                              void* workspace, cudaStream_t stream);

// conv_simt.cu
int simt_pack_weights(wn_handle* h, const float* const* params, cudaStream_t stream);
void simt_free(wn_handle* h);
size_t simt_forward_workspace_bytes(int n, int h, int w);
// stack (FwdStack): kStackCmg -> out = the three confidence maps; kStackRefiners -> out = refiner `which`'s image
int simt_forward(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], float* out,
                 int n, int height, int width, void* workspace, size_t workspace_bytes,
                 cudaStream_t stream, int stack = 0, int which = 0);

int simt_debug_layer(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], int n,
                     int height, int width, int layer, float* dst, void* workspace,
                     size_t workspace_bytes, cudaStream_t stream);

// conv_umma.cu
struct FwdBuffers {
  uint4* act0;    // packed input, 16 channels (bf16 hi/lo planes of v*255)
  uint4* a[8];    // a[l] = output of cmg.conv<l>, l = 1..7 (planes)
  uint4* r[3];    // r[1], r[2] = refiner conv1 / conv2 outputs, three refiners side by side (96 channels)
  float* cm;      // sigmoid confidence maps, fp32 [n][3][H][W]
  float* refined; // optional: refined images after ReLU, fp32 [n][9][H][W]
  int* exact_flag;
};
// Peer copies of the uint8 output (multi-GPU all-gather fused into the kernel that produces the output: plain stores
// to addresses mapped from the other ranks' buffers, wn_enhance_u8_peers)
struct PeerOut {
  uint8_t* p[WN_MAX_PEERS];
  int n;
};
constexpr int kSchemeBf16 = 2;  // FwdOpts::scheme of the WN_MODE_BF16 training forward (UmmaCfg kFmtHi)
// the scheme of a training forward: the handle's training arithmetic (wn_set_train_mode)
inline int train_scheme(const wn_handle* h) { return h->train_bf16 ? kSchemeBf16 : 0; }
struct FwdOpts {
  int scheme = 0;              // 1 = fp8 correction passes (WN_MODE_BF16_FP8); kSchemeBf16 = one bf16 pass (training)
  int dbg_layer = -1;          // wn_debug_forward_layer: stop after this layer and decode it into dbg_dst
  float* dbg_dst = nullptr;
  bool packed = false;         // act0 already holds the 16-channel operand planes of this batch
  bool hi_only = false;        // ... as exact 8-bit levels, hi planes only (written by the preprocess kernel)
  const int* run_if = nullptr; // every launch is conditional on *run_if != 0 (ConvArgs::run_if)
  uint8_t* out_u8 = nullptr;   // the last launch also writes ten2arr(out) as uint8 NHWC
  PeerOut peers = {};          // ... and the same bytes to every peer address (offsets as out_u8)
  int stack = kStackAll;       // kStackCmg: stop after the confidence maps; kStackRefiners: refiners only
  bool refiner_l1 = false;     // kStackRefiners, bf16x3: the first layer is the refiners' conv1 alone (kRL1)
  const TileGeom* tiles = nullptr;  // tiled forward: image n of the batch is window win0 + n of these tiles, and the
  long long win0 = 0;               // last launch stores its kept rectangle into out / out_u8 at image coordinates
  const RaggedWindow* rwin = nullptr;  // ragged pass (device table): image n of the batch is window rwin[n] in its
                                       // slot; every layer masks it, the last launch stores into its own image
  const int* slot_levels = nullptr;    // ragged fp32 pass: slot n holds 8-bit levels only (ConvArgs::slot_levels)
  bool fuse_c4 = false;        // inference: cmg.conv4 runs in cmg.conv3's epilogue (kFmtFuse1x1); the outputs of
                               // cmg.conv4 to cmg.conv7 take the buffers a[3] .. a[6]
};
int umma_forward_layers(wn_handle* h, const float* const in[4], const int64_t st[4][4], float* out, int n,
                        int height, int width, const FwdBuffers& b, cudaStream_t stream,
                        const FwdOpts& opts = FwdOpts());
int umma_debug_layer(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], int n,
                     int height, int width, int layer, float* dst, void* workspace,
                     size_t workspace_bytes, cudaStream_t stream, int scheme = 0);
// bf16 hi + lo planes (planes_half 8-channel planes per half) of n images -> fp32 NCHW, hi + lo (test aid)
int decode_planes(wn_handle* h, const uint4* src, float* dst, int planes_half, int n, int hw, cudaStream_t stream);
int umma_pack_weights(wn_handle* h, const float* const* params, cudaStream_t stream);
void umma_free(wn_handle* h);
size_t umma_forward_workspace_bytes(int n, int h, int w);
int umma_chunk_images(const wn_handle* h, int n, int height, int width);
// stack = kStackCmg: out receives the three confidence maps; kStackRefiners: `refined` receives the three
// refined images as [n][9][H][W] and out is unused
int umma_forward(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], float* out,
                 int n, int height, int width, void* workspace, size_t workspace_bytes,
                 cudaStream_t stream, int scheme = 0, int stack = kStackAll, float* refined = nullptr);
// the tiled forward of fp32 tensors (arguments checked by the caller, api.cu).  stack as umma_forward; the
// sub-modules write `out` directly (kStackRefiners: refiner `which`) and need the `submodule` workspace
size_t umma_forward_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels,
                                          bool submodule);
int umma_forward_tiled(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], float* out, int n,
                       int height, int width, int tile_h, int tile_w, long long max_pass_pixels, void* workspace,
                       size_t workspace_bytes, cudaStream_t stream, int scheme, int stack = kStackAll, int which = 0);
size_t umma_enhance_workspace_bytes(int n, int h, int w);
int mirror_u8(wn_handle* h, const uint8_t* src, const PeerOut& peers, size_t bytes, const int* run_if, cudaStream_t stream);
int umma_enhance_u8(wn_handle* h, const uint8_t* rgb, uint8_t* out_u8, float* out_f32, int n, int height,
                    int width, void* workspace, size_t workspace_bytes, cudaStream_t stream, int scheme,
                    const PeerOut& peers = PeerOut());
// 0 when the arguments are out of range (tiles < 1, an image over the preprocess limit)
size_t umma_enhance_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels);
int umma_enhance_u8_tiled(wn_handle* h, const uint8_t* rgb, uint8_t* out_u8, float* out_f32, int n, int height,
                          int width, int tile_h, int tile_w, long long max_pass_pixels, void* workspace,
                          size_t workspace_bytes, cudaStream_t stream, int scheme);
// the arguments are checked by the caller (api.cu)
size_t umma_enhance_ragged_workspace_bytes(const int* hs, const int* ws, int n, int tile_h, int tile_w,
                                           long long max_pass_pixels);
int umma_enhance_u8_ragged(wn_handle* h, const wn_ragged_image* images, int n, int tile_h, int tile_w,
                           long long max_pass_pixels, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                           int scheme);
int umma_f8_overflowed(const wn_handle* h);

// conv_umma.cu: the operand packing of fp32 inputs, shared with the training forward and the windowed backward.  The
// four inputs of an image and their element strides; a grid geometry reads image n of one set at offset n * s[t][0].
struct PackInArgs {
  const float* p[4];
  long long s[4][4];
};
inline PackInArgs pack_args(const float* const in[4], const int64_t st[4][4]) {
  PackInArgs pa;
  for (int t = 0; t < 4; t++) {
    pa.p[t] = in[t];
    for (int k = 0; k < 4; k++) pa.s[t][k] = st[t][k];
  }
  return pa;
}
// `count` slots of geo, read at image coordinates: the slots' act0 planes when act0 is given (zeros beyond each valid
// extent), and the exact-levels flag when flag is given (cleared unless every input pixel of the valid extents is an
// 8-bit level).  The grid form reads one set of (N,3,H,W) tensors and sets the flag to 1 before it packs.  The table
// form reads one PackInArgs per image, a device table; its flag spans several launches, so the caller sets it to 1
// once, and with act0 given the table form leaves the flag alone.  hi: the act0 planes of the single-pass bf16
// training forward (kSchemeBf16), lo planes stored as 0.
int pack_inputs(wn_handle* h, const GridGeom& geo, const PackInArgs& in, int count, uint4* act0, int* flag,
                cudaStream_t stream, bool hi = false);
int pack_inputs(wn_handle* h, const TableGeom& geo, const PackInArgs* imgs, int count, uint4* act0, int* flag,
                cudaStream_t stream, bool hi = false, int* slot_flags = nullptr);
// wn_forward_ragged (arguments checked by the caller, api.cu): the windows and passes of ragged_plan
size_t umma_forward_ragged_workspace_bytes(const int* hs, const int* ws, int n, int tile_h, int tile_w,
                                           long long max_pass_pixels);
int umma_forward_ragged(wn_handle* h, const wn_ragged_tensors* images, int n, int tile_h, int tile_w,
                        long long max_pass_pixels, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                        int scheme);

// conv_bwd.cu
constexpr long long kTrainMaxPixels = 8ll << 20;  // pixels of one training pass (activations kept: ~5.6 KB each)
constexpr long long kTiledTrainPassPixels = 2ll << 20;  // wn_backward_tiled: window pixels per pass by default
int bwd_pack_weights(wn_handle* h, const float* const* params, cudaStream_t stream);
void bwd_free(wn_handle* h);
size_t train_workspace_bytes_padded(int n, int h, int w);
int forward_train(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], float* out, int n,
                  int height, int width, void* workspace, size_t workspace_bytes, cudaStream_t stream);
int backward(wn_handle* h, const float* grad_out, float* const* grads, float* const* input_grads, int n,
             int height, int width, void* workspace, size_t workspace_bytes, cudaStream_t stream);
// The sub-modules under autograd (wn_confidence_maps_train / _backward, wn_refine_train / _backward); arguments
// checked by the caller (api.cu).  stack: kStackCmg or kStackRefiners.  The workspace holds that stack's activations
// and gradient buffers only.
size_t submodule_train_workspace_bytes(int n, int height, int width, int stack);
int confidence_maps_train(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], float* out_maps,
                          int n, int height, int width, void* workspace, size_t workspace_bytes, cudaStream_t stream);
int confidence_maps_backward(wn_handle* h, const float* grad_maps, float* const* grads, float* const* input_grads,
                             int n, int height, int width, void* workspace, size_t workspace_bytes,
                             cudaStream_t stream);
int refine_train(wn_handle* h, int which, const float* const in[4], const int64_t in_strides[4][4], float* out, int n,
                 int height, int width, void* workspace, size_t workspace_bytes, cudaStream_t stream);
int refine_backward(wn_handle* h, int which, const float* grad_out, float* const* grads, float* const* input_grads,
                    int n, int height, int width, void* workspace, size_t workspace_bytes, cudaStream_t stream);
// wn_debug_backward_layer (test aid); stack: kStackAll, kStackCmg or kStackRefiners (refiner `which`); the buffer
// number, the pointers and the shape are checked by the caller (api.cu)
int debug_backward_layer(wn_handle* h, int stack, int which, int buffer, const float* grad_out, float* const* grads,
                         int n, int height, int width, float* dst, void* workspace, size_t workspace_bytes,
                         cudaStream_t stream);
// the windowed recompute backward; arguments checked by the caller (api.cu)
size_t backward_tiled_workspace_bytes(int n, int height, int width, int tile_h, int tile_w, long long max_pass_pixels);
int backward_tiled(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], const float* grad_out,
                   float* const* grads, float* const* input_grads, int n, int height, int width, int tile_h, int tile_w,
                   long long max_pass_pixels, void* workspace, size_t workspace_bytes, cudaStream_t stream);
// ... of one sub-module (stack kStackCmg, or kStackRefiners with refiner `which`); arguments checked by the caller.
// in: the stack's four packed inputs ({x, wb, he, gc}, or {x, xbar, xbar, xbar} for a refiner); grad: d(maps) or
// d(out); grads: the 34-entry layout, the stack's own entries written; input_grads: NULL or 4 / 2 entries, any NULL
size_t submodule_backward_tiled_workspace_bytes(int n, int height, int width, int tile_h, int tile_w,
                                                long long max_pass_pixels, int stack);
int submodule_backward_tiled(wn_handle* h, int stack, int which, const float* const in[4],
                             const int64_t in_strides[4][4], const float* grad, float* const* grads,
                             float* const* input_grads, int n, int height, int width, int tile_h, int tile_w,
                             long long max_pass_pixels, void* workspace, size_t workspace_bytes, cudaStream_t stream);
// the ragged training step (wn_forward_train_ragged / wn_backward_ragged): the n images of one call as one pass of
// slots of the per-axis maximum size; arguments checked by the caller (api.cu: n * slot pixels <= kTrainMaxPixels)
size_t train_ragged_workspace_bytes(const int* hs, const int* ws, int n);
int forward_train_ragged(wn_handle* h, const wn_ragged_tensors* images, int n, void* workspace, size_t workspace_bytes,
                         cudaStream_t stream);
int backward_ragged(wn_handle* h, const int* hs, const int* ws, const float* const* grad_out, float* const* grads,
                    float* const* input_grads, int n, void* workspace, size_t workspace_bytes, cudaStream_t stream);
// the windowed recompute backward of a ragged batch (wn_backward_ragged_tiled): the windows and passes of ragged_plan;
// arguments checked by the caller (api.cu: the limits of wn_backward_tiled for every image)
size_t backward_ragged_tiled_workspace_bytes(const int* hs, const int* ws, int n, int tile_h, int tile_w,
                                             long long max_pass_pixels);
int backward_ragged_tiled(wn_handle* h, const wn_ragged_tensors* images, const float* const* grad_out,
                          float* const* grads, float* const* input_grads, int n, int tile_h, int tile_w,
                          long long max_pass_pixels, void* workspace, size_t workspace_bytes, cudaStream_t stream);

// vgg.cu: the windowed VGG19 perceptual loss (wn_perceptual_loss).  The workspace function returns 0, and the calls
// fail with the reason set, for every argument set the loss rejects.
int vgg_pack_weights(wn_handle* h, const float* const* params, cudaStream_t stream);
void vgg_free(wn_handle* h);
size_t vgg_loss_workspace_bytes(int n, int height, int width, int tile_h, int tile_w, long long max_pass_pixels);
int vgg_perceptual_loss(wn_handle* h, const float* out, const int64_t out_strides[4], const float* ref,
                        const int64_t ref_strides[4], int n, int height, int width, int tile_h, int tile_w,
                        long long max_pass_pixels, float* loss, float* grad_out, void* workspace,
                        size_t workspace_bytes, cudaStream_t stream);
int vgg_debug_layer(wn_handle* h, const float* x, const int64_t strides[4], const float* ref,
                    const int64_t ref_strides[4], int n, int height, int width, int tile_h, int tile_w, int layer,
                    float* dst, void* workspace, size_t workspace_bytes, cudaStream_t stream);

// metrics.cu: SSIM / PSNR statistics (wn_quality).  quality_plan_check refuses sides below 6 and calls too large;
// quality runs on arguments the caller has checked (api.cu).  The workspace function returns 0 where the check fails.
int quality_plan_check(const int* hs, const int* ws, int n, const char* what);
size_t quality_workspace_bytes(const int* hs, const int* ws, int n);
int quality(wn_handle* h, const wn_quality_image* images, int n, double* stats, void* workspace,
            size_t workspace_bytes, cudaStream_t stream);
// ... and SSIM's gradient (wn_ssim_grad): the same checks, plus the gradient grid's size
int ssim_grad_plan_check(const int* hs, const int* ws, int n, const char* what);
size_t ssim_grad_workspace_bytes(const int* hs, const int* ws, int n);
int ssim_grad(wn_handle* h, const wn_ssim_grad_image* images, int n, double* stats, void* workspace,
              size_t workspace_bytes, cudaStream_t stream);

}  // namespace wn
