// C ABI of libwaternet_b200.so (see include/waternet_b200.h for the contract).
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace wn {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static int resolve_mode(int mode) {
  if (mode == WN_MODE_DEFAULT) return WN_MODE_BF16_FP8;
  return mode;
}

// the tensor-core scheme of a mode: 1 = fp8 corrections, 0 = bf16x3
static int scheme_of(int mode) { return resolve_mode(mode) == WN_MODE_BF16_FP8 ? 1 : 0; }

struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) ok = false;
    if (ok && prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// ---- the argument checks of the entry points, one helper per kind.  Each returns WN_OK or the error code with
// wn_last_error() set; `what` names the entry point in the message.
static bool all_set(std::initializer_list<const void*> ptrs) {
  for (const void* p : ptrs)
    if (!p) return false;
  return true;
}

static int invalid(const char* what, const char* msg) {
  set_error("%s: %s", what, msg);
  return WN_E_INVALID;
}

static int check_ptrs(const char* what, std::initializer_list<const void*> ptrs, const char* msg = "null argument") {
  return all_set(ptrs) ? WN_OK : invalid(what, msg);
}

// the calls that fold their pointers, their shape and `ok` into one "bad argument"
static int check_args(const char* what, std::initializer_list<const void*> ptrs, int n, int height, int width,
                      bool ok = true) {
  return all_set(ptrs) && n > 0 && height > 0 && width > 0 && ok ? WN_OK : invalid(what, "bad argument");
}

static int check_shape(const char* what, int n, int height, int width) {
  if (n > 0 && height > 0 && width > 0) return WN_OK;
  set_error("%s: bad shape n=%d h=%d w=%d", what, n, height, width);
  return WN_E_INVALID;
}

static int check_tiled_shape(const char* what, int n, int height, int width, int tile_h, int tile_w,
                             long long max_pass_pixels) {
  if (n > 0 && height > 0 && width > 0 && tile_h > 0 && tile_w > 0 && max_pass_pixels >= 0) return WN_OK;
  set_error("%s: bad shape n=%d h=%d w=%d tile=%dx%d max_pass_pixels=%lld", what, n, height, width, tile_h, tile_w,
            max_pass_pixels);
  return WN_E_INVALID;
}

// the image count and tiling of a ragged call
static int check_ragged_shape(const char* what, int n, int tile_h, int tile_w, long long max_pass_pixels) {
  if (n <= 0 || tile_h <= 0 || tile_w <= 0 || max_pass_pixels < 0) {
    set_error("%s: bad shape n=%d tile=%dx%d max_pass_pixels=%lld", what, n, tile_h, tile_w, max_pass_pixels);
    return WN_E_INVALID;
  }
  if (n > 65535) {
    set_error("%s: too many images: n=%d", what, n);
    return WN_E_UNSUPPORTED;
  }
  return WN_OK;
}

// one image per grid row of the per-pixel kernels
static int check_images_per_call(const char* what, int n) {
  if (n <= 65535) return WN_OK;
  set_error("%s: at most 65535 images per call, got n=%d", what, n);
  return WN_E_UNSUPPORTED;
}

static int check_ragged_count(const char* what, int n) {
  if (n > 0 && n <= 65535) return WN_OK;
  set_error("%s: 1..65535 images per call, got n=%d", what, n);
  return n <= 0 ? WN_E_INVALID : WN_E_UNSUPPORTED;
}

// the image-size limit: a plane's element index fits an int
static bool too_large(int height, int width) { return (size_t)height * width > (size_t)0x7fffffff / 3; }

static int check_size(int n, int height, int width) {
  if (!too_large(height, width) && n <= 65535) return WN_OK;
  set_error("image too large: n=%d h=%d w=%d", n, height, width);
  return WN_E_UNSUPPORTED;
}

// the size of image i of a ragged batch
static int check_ragged_size(const char* what, int i, int height, int width) {
  if (height <= 0 || width <= 0) {
    set_error("%s: bad size of image %d: h=%d w=%d", what, i, height, width);
    return WN_E_INVALID;
  }
  if (too_large(height, width)) {
    set_error("image too large: image %d h=%d w=%d", i, height, width);
    return WN_E_UNSUPPORTED;
  }
  return WN_OK;
}

static int check_packed(const char* what, const wn_handle* h) {
  if (h->packed) return WN_OK;
  set_error("%s: wn_pack_weights has not been called", what);
  return WN_E_STATE;
}

static int check_workspace(const char* what, size_t have, size_t need) {
  if (have >= need) return WN_OK;
  set_error("%s: workspace too small", what);
  return WN_E_WORKSPACE;
}

// The scheme of a mode (scheme_of), kSchemeSimt for WN_MODE_FP32_SIMT when `simt_refusal` is NULL, or the error:
// WN_E_UNSUPPORTED with "<what>: <simt_refusal>" for WN_MODE_FP32_SIMT, WN_E_INVALID for an unknown mode.
// Errors are negative.
constexpr int kSchemeSimt = 2;
static int check_mode(const char* what, int mode, const char* simt_refusal) {
  const int m = resolve_mode(mode);
  if (m == WN_MODE_FP32_SIMT) {
    if (!simt_refusal) return kSchemeSimt;
    set_error("%s: %s", what, simt_refusal);
    return WN_E_UNSUPPORTED;
  }
  if (m != WN_MODE_BF16X3 && m != WN_MODE_BF16_FP8) {
    set_error("%s: unknown mode %d", what, mode);
    return WN_E_INVALID;
  }
  return scheme_of(mode);
}
constexpr const char* kTiledRefusal = "the tiled forward runs in the tensor-core modes only, not WN_MODE_FP32_SIMT";
constexpr const char* kRaggedRefusal = "ragged batches run in the tensor-core modes only, not WN_MODE_FP32_SIMT";

// entries [first, first + count) of a host array of device pointers (params, grads, input_grads, grad_out_host)
template <class P>
static int check_entries(const char* what, const char* name, P const* a, int first, int count) {
  for (int i = first; i < first + count; i++)
    if (!a[i]) {
      set_error("%s: %s[%d] is NULL", what, name, i);
      return WN_E_INVALID;
    }
  return WN_OK;
}

// the backward calls: the parameter gradients [first, first + count) they write must be given
static int check_param_grads(const char* what, float* const* grads, int first, int count) {
  return check_entries(what, "grads", grads, first, count);
}

// the optional input gradients of the backward calls of WaterNet: all four or none
static int check_input_grads(const char* what, float* const* input_grads) {
  return input_grads ? check_entries(what, "input_grads", input_grads, 0, 4) : WN_OK;
}

// The images of a ragged table in order: `given(image, i)` says whether image i's device pointers are given; with
// `sizes` its size is checked after them.
template <class Image, class Given>
static int check_images(const char* what, const Image* images, int n, bool sizes, Given given) {
  for (int i = 0; i < n; i++) {
    if (!given(images[i], i)) {
      set_error("%s: null image pointer (image %d)", what, i);
      return WN_E_INVALID;
    }
    int rc = sizes ? check_ragged_size(what, i, images[i].height, images[i].width) : WN_OK;
    if (rc) return rc;
  }
  return WN_OK;
}
static bool inputs_given(const wn_ragged_tensors& t) { return t.x && t.wb && t.he && t.gc; }

static int check_which(const char* what, int which) {
  if (which >= 0 && which <= 2) return WN_OK;
  set_error("%s: which must be 0, 1 or 2, got %d", what, which);
  return WN_E_INVALID;
}
static bool submodule_stack(int stack) { return stack == 0 || stack == 1; }

// Refiner r sees cat[x, input r+1] (net.py:101-103): the refiner stack gets xbar in every slot after x, with the
// strides {x, xbar} of in_strides[2][4] spread to the [4][4] the stack takes.
struct RefinerInputs {
  const float* in[4];
  int64_t st[4][4];
  RefinerInputs(const float* x, const float* xbar, const int64_t in_strides[2][4]) : in{x, xbar, xbar, xbar} {
    for (int t = 0; t < 4; t++)
      for (int k = 0; k < 4; k++) st[t][k] = in_strides[t == 0 ? 0 : 1][k];
  }
};

}  // namespace wn

using namespace wn;

extern "C" {

int wn_abi_version(void) { return WN_ABI_VERSION; }

const char* wn_last_error(void) { return g_err; }

int wn_build_tables_host(uint16_t* gtab, uint16_t* ctab, int16_t* ytab, int16_t* fytab,
                         uint8_t* igtab, uint8_t* gamma, float* div255) {
  int rc = check_ptrs("wn_build_tables_host", {gtab, ctab, ytab, fytab, igtab, gamma, div255}, "null output");
  if (rc) return rc;
  Tables* t = (Tables*)malloc(sizeof(Tables));
  build_tables_host(t);
  memcpy(gtab, t->gtab, sizeof(t->gtab));
  memcpy(ctab, t->ctab, sizeof(t->ctab));
  memcpy(ytab, t->ytab, sizeof(t->ytab));
  memcpy(fytab, t->fytab, sizeof(t->fytab));
  memcpy(igtab, t->igtab, sizeof(t->igtab));
  memcpy(gamma, t->gamma, sizeof(t->gamma));
  memcpy(div255, t->div255, sizeof(t->div255));
  free(t);
  return WN_OK;
}

int wn_create(int device, wn_handle** out) {
  if (!out) {
    set_error("wn_create: out is NULL");
    return WN_E_INVALID;
  }
  *out = nullptr;
  int count = 0;
  WN_CUDA(cudaGetDeviceCount(&count));
  if (device < 0 || device >= count) {
    set_error("wn_create: device %d out of range (%d devices)", device, count);
    return WN_E_INVALID;
  }
  DeviceGuard guard(device);
  cudaDeviceProp prop;
  WN_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("wn_create: device %d is sm_%d%d; this library is built for sm_90a only", device,
              prop.major, prop.minor);
    return WN_E_UNSUPPORTED;
  }
  wn_handle* h = (wn_handle*)calloc(1, sizeof(wn_handle));
  h->device = device;
  h->sm_count = prop.multiProcessorCount;
  Tables* t = (Tables*)malloc(sizeof(Tables));
  build_tables_host(t);
  cudaError_t e = cudaMalloc(&h->d_tables, sizeof(Tables));
  if (e == cudaSuccess) e = cudaMemcpy(h->d_tables, t, sizeof(Tables), cudaMemcpyHostToDevice);
  free(t);
  if (e != cudaSuccess) {
    set_error("wn_create: %s", cudaGetErrorString(e));
    free(h);
    return WN_E_CUDA;
  }
  *out = h;
  return WN_OK;
}

void wn_destroy(wn_handle* h) {
  if (!h) return;
  DeviceGuard guard(h->device);
  simt_free(h);
  umma_free(h);
  bwd_free(h);
  vgg_free(h);
  if (h->d_tables) cudaFree(h->d_tables);
  if (h->timing) {
    for (int i = 0; i < h->timing->created; i++) {
      cudaEventDestroy(h->timing->a[i]);
      cudaEventDestroy(h->timing->b[i]);
    }
    free(h->timing);
  }
  free(h);
}

int wn_pack_weights(wn_handle* h, const float* const* params, void* stream) {
  const char* what = "wn_pack_weights";
  int rc = check_ptrs(what, {h, params});
  if (rc || (rc = check_entries(what, "params", params, 0, WN_NUM_PARAMS))) return rc;
  DeviceGuard guard(h->device);
  rc = simt_pack_weights(h, params, (cudaStream_t)stream);
  if (rc) return rc;
  rc = umma_pack_weights(h, params, (cudaStream_t)stream);
  if (rc) return rc;
  rc = bwd_pack_weights(h, params, (cudaStream_t)stream);
  if (rc) return rc;
  h->packed = true;
  return WN_OK;
}

size_t wn_forward_workspace_bytes(int n, int h, int w, int mode) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  switch (resolve_mode(mode)) {
    case WN_MODE_FP32_SIMT: return simt_forward_workspace_bytes(n, h, w);
    case WN_MODE_BF16X3:
    case WN_MODE_BF16_FP8: return umma_forward_workspace_bytes(n, h, w);
  }
  return 0;
}

int wn_forward(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
               const int64_t in_strides[4][4], float* out, int n, int height, int width, int mode,
               void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_forward";
  int rc = check_ptrs(what, {h, x, wb, he, gc, in_strides, out, workspace});
  if (rc || (rc = check_shape(what, n, height, width)) || (rc = check_packed(what, h))) return rc;
  DeviceGuard guard(h->device);
  const float* in[4] = {x, wb, he, gc};
  const int s = check_mode(what, mode, nullptr);
  if (s < 0) return s;
  if (s == kSchemeSimt)
    return simt_forward(h, in, in_strides, out, n, height, width, workspace, workspace_bytes, (cudaStream_t)stream);
  return umma_forward(h, in, in_strides, out, n, height, width, workspace, workspace_bytes, (cudaStream_t)stream, s);
}

size_t wn_preprocess_workspace_bytes(int n, int h, int w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  return preprocess_workspace_bytes(n, h, w);
}

int wn_preprocess_u8(wn_handle* h, const uint8_t* rgb, int n, int height, int width, float* x,
                     float* wb, float* he, float* gc, uint8_t* wb_u8, uint8_t* he_u8,
                     uint8_t* gc_u8, void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_preprocess_u8";
  int rc = check_ptrs(what, {h, rgb, workspace});
  if (rc || (rc = check_shape(what, n, height, width))) return rc;
  DeviceGuard guard(h->device);
  return preprocess_u8(h, rgb, n, height, width, x, wb, he, gc, wb_u8, he_u8, gc_u8, workspace,
                       workspace_bytes, (cudaStream_t)stream);
}

int wn_postprocess_u8(wn_handle* h, const float* out_nchw, uint8_t* out_nhwc, int n, int height,
                      int width, void* stream) {
  int rc = check_args("wn_postprocess_u8", {h, out_nchw, out_nhwc}, n, height, width);
  if (rc) return rc;
  DeviceGuard guard(h->device);
  return postprocess_u8(h, out_nchw, out_nhwc, n, height, width, (cudaStream_t)stream);
}

size_t wn_white_balance_gray_workspace_bytes(int n, int h, int w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  return white_balance_gray_workspace_bytes(n, h, w);
}

int wn_white_balance_gray_u8(wn_handle* h, const uint8_t* gray, uint8_t* out, int n, int height, int width,
                             void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_args("wn_white_balance_gray_u8", {h, gray, out, workspace}, n, height, width);
  if (rc || (rc = check_size(n, height, width))) return rc;
  DeviceGuard guard(h->device);
  return white_balance_gray_u8(h, gray, out, n, height, width, workspace, workspace_bytes, (cudaStream_t)stream);
}

int wn_resize_u8(wn_handle* h, const uint8_t* const* src_dev, const int* src_h, const int* src_w, int n,
                 uint8_t* dst_nhwc, int dst_h, int dst_w, int swap_rb, void* stream) {
  int rc = check_args("wn_resize_u8", {h, src_dev, src_h, src_w, dst_nhwc}, n, dst_h, dst_w);
  if (rc) return rc;
  DeviceGuard guard(h->device);
  return resize_u8(h, src_dev, src_h, src_w, n, dst_nhwc, dst_h, dst_w, swap_rb, (cudaStream_t)stream);
}


// fp32 CUDA-core mode: the API tensors are materialised (preprocess -> 4 fp32 tensors -> forward -> fp32 -> ten2arr)
static size_t enhance_simt_workspace_bytes(int n, int h, int w) {
  size_t tens = align256((size_t)n * 3 * h * w * sizeof(float));
  return 5 * tens + align256(preprocess_workspace_bytes(n, h, w)) +
         align256(simt_forward_workspace_bytes(n, h, w)) + 256;
}

size_t wn_enhance_workspace_bytes(int n, int h, int w, int mode) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  if (resolve_mode(mode) == WN_MODE_FP32_SIMT) return enhance_simt_workspace_bytes(n, h, w);
  return umma_enhance_workspace_bytes(n, h, w);
}

int wn_enhance_u8(wn_handle* h, const uint8_t* rgb, uint8_t* out_nhwc, float* out_f32_or_null,
                  int n, int height, int width, int mode, void* workspace, size_t workspace_bytes,
                  void* stream) {
  return wn_enhance_u8_peers(h, rgb, out_nhwc, out_f32_or_null, nullptr, 0, n, height, width, mode, workspace,
                             workspace_bytes, stream);
}

int wn_enhance_u8_peers(wn_handle* h, const uint8_t* rgb, uint8_t* out_nhwc, float* out_f32_or_null,
                        uint8_t* const* peer_out, int n_peers, int n, int height, int width, int mode,
                        void* workspace, size_t workspace_bytes, void* stream) {
  PeerOut peers = {};
  if (n_peers < 0 || n_peers > WN_MAX_PEERS || (n_peers > 0 && !peer_out)) {
    set_error("wn_enhance_u8_peers: 0..%d peer addresses", WN_MAX_PEERS);
    return WN_E_INVALID;
  }
  for (int k = 0; k < n_peers; k++) {
    if (!peer_out[k]) {
      set_error("wn_enhance_u8_peers: peer address %d is null", k);
      return WN_E_INVALID;
    }
    peers.p[k] = peer_out[k];
  }
  peers.n = n_peers;
  const char* what = "wn_enhance_u8";
  int rc = check_ptrs(what, {h, rgb, out_nhwc, workspace});
  if (rc || (rc = check_shape(what, n, height, width)) || (rc = check_packed(what, h)) ||
      (rc = check_workspace(what, workspace_bytes, wn_enhance_workspace_bytes(n, height, width, mode))) ||
      (rc = check_size(n, height, width)))
    return rc;
  DeviceGuard guard(h->device);
  if (resolve_mode(mode) != WN_MODE_FP32_SIMT)  // tensor-core modes: folded path, nothing fp32 is materialised
    return umma_enhance_u8(h, rgb, out_nhwc, out_f32_or_null, n, height, width, workspace, workspace_bytes,
                           (cudaStream_t)stream, scheme_of(mode), peers);
  uint8_t* ws = (uint8_t*)(((uintptr_t)workspace + 255) / 256 * 256);
  const size_t tens = align256((size_t)n * 3 * height * width * sizeof(float));
  float* t[5];
  for (int i = 0; i < 5; i++) {
    t[i] = (float*)ws;
    ws += tens;
  }
  void* pre_ws = ws;
  size_t pre_b = align256(preprocess_workspace_bytes(n, height, width));
  ws += pre_b;
  void* fwd_ws = ws;
  size_t fwd_b = align256(simt_forward_workspace_bytes(n, height, width));
  rc = wn_preprocess_u8(h, rgb, n, height, width, t[0], t[1], t[2], t[3], nullptr, nullptr,
                        nullptr, pre_ws, pre_b, stream);
  if (rc) return rc;
  const int64_t hw = (int64_t)height * width;
  const int64_t st[4][4] = {{3 * hw, hw, width, 1}, {3 * hw, hw, width, 1}, {3 * hw, hw, width, 1},
                            {3 * hw, hw, width, 1}};
  float* outf = out_f32_or_null ? out_f32_or_null : t[4];
  rc = wn_forward(h, t[0], t[1], t[2], t[3], st, outf, n, height, width, mode, fwd_ws, fwd_b, stream);
  if (rc) return rc;
  rc = wn_postprocess_u8(h, outf, out_nhwc, n, height, width, stream);
  if (rc) return rc;
  return mirror_u8(h, out_nhwc, peers, (size_t)n * height * width * 3, nullptr, (cudaStream_t)stream);
}

// ---- the tiled forward (wn_enhance_u8_tiled, and WaterNet.forward and its sub-modules in windows)
// the argument checks the tiled forward calls and the three tiled workspace functions share (pointers aside):
// the scheme, or the (negative) error
static int forward_tiled_check(const char* what, int n, int height, int width, int tile_h, int tile_w,
                               long long max_pass_pixels, int mode) {
  int rc = check_tiled_shape(what, n, height, width, tile_h, tile_w, max_pass_pixels);
  if (rc) return rc;
  const int s = check_mode(what, mode, kTiledRefusal);
  if (s < 0) return s;
  return (rc = check_size(n, height, width)) ? rc : s;
}

size_t wn_enhance_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels,
                                        int mode) {
  if (forward_tiled_check("wn_enhance_tiled_workspace_bytes", n, h, w, tile_h, tile_w, max_pass_pixels, mode) < 0)
    return 0;
  return umma_enhance_tiled_workspace_bytes(n, h, w, tile_h, tile_w, max_pass_pixels);
}

int wn_enhance_u8_tiled(wn_handle* h, const uint8_t* rgb, uint8_t* out_nhwc, float* out_f32_or_null, int n,
                        int height, int width, int tile_h, int tile_w, long long max_pass_pixels, int mode,
                        void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_enhance_u8_tiled";
  int rc = check_ptrs(what, {h, rgb, out_nhwc, workspace});
  if (rc || (rc = check_tiled_shape(what, n, height, width, tile_h, tile_w, max_pass_pixels))) return rc;
  const int s = check_mode(what, mode, kTiledRefusal);
  if (s < 0) return s;
  if ((rc = check_packed(what, h)) || (rc = check_size(n, height, width))) return rc;
  DeviceGuard guard(h->device);
  return umma_enhance_u8_tiled(h, rgb, out_nhwc, out_f32_or_null, n, height, width, tile_h, tile_w, max_pass_pixels,
                               workspace, workspace_bytes, (cudaStream_t)stream, s);
}

// ---- ragged batches (wn_enhance_u8_ragged, wn_forward_ragged)
// the argument checks the ragged calls and their workspace functions share (the images aside): the scheme, or the
// (negative) error
static int ragged_check(const char* what, int n, int tile_h, int tile_w, long long max_pass_pixels, int mode) {
  int rc = check_ragged_shape(what, n, tile_h, tile_w, max_pass_pixels);
  return rc ? rc : check_mode(what, mode, kRaggedRefusal);
}

// the checks of a ragged workspace function: those of its call, with the sizes for the images
static bool ragged_sizes_ok(const char* what, const int* hs, const int* ws, int n, int tile_h, int tile_w,
                            long long max_pass_pixels, int mode) {
  if (!hs || !ws || ragged_check(what, n, tile_h, tile_w, max_pass_pixels, mode) < 0) return false;
  for (int i = 0; i < n; i++)
    if (check_ragged_size(what, i, hs[i], ws[i])) return false;
  return true;
}

size_t wn_enhance_ragged_workspace_bytes(const int* heights_host, const int* widths_host, int n, int tile_h,
                                         int tile_w, long long max_pass_pixels, int mode) {
  if (!ragged_sizes_ok("wn_enhance_ragged_workspace_bytes", heights_host, widths_host, n, tile_h, tile_w,
                       max_pass_pixels, mode))
    return 0;
  return umma_enhance_ragged_workspace_bytes(heights_host, widths_host, n, tile_h, tile_w, max_pass_pixels);
}

int wn_enhance_u8_ragged(wn_handle* h, const wn_ragged_image* images_host, int n, int tile_h, int tile_w,
                         long long max_pass_pixels, int mode, void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_enhance_u8_ragged";
  int rc = check_ptrs(what, {h, images_host, workspace});
  if (rc) return rc;
  const int s = ragged_check(what, n, tile_h, tile_w, max_pass_pixels, mode);
  if (s < 0) return s;
  if ((rc = check_images(what, images_host, n, true,
                         [](const wn_ragged_image& im, int) { return im.rgb && im.out_u8; })) ||
      (rc = check_packed(what, h)))
    return rc;
  DeviceGuard guard(h->device);
  return umma_enhance_u8_ragged(h, images_host, n, tile_h, tile_w, max_pass_pixels, workspace, workspace_bytes,
                                (cudaStream_t)stream, s);
}

static_assert(sizeof(wn_ragged_tensors) == 176, "wn_ragged_tensors: _lib.RAGGED_TENSORS_BYTES restates this size");

size_t wn_forward_ragged_workspace_bytes(const int* heights_host, const int* widths_host, int n, int tile_h,
                                         int tile_w, long long max_pass_pixels, int mode) {
  if (!ragged_sizes_ok("wn_forward_ragged_workspace_bytes", heights_host, widths_host, n, tile_h, tile_w,
                       max_pass_pixels, mode))
    return 0;
  return umma_forward_ragged_workspace_bytes(heights_host, widths_host, n, tile_h, tile_w, max_pass_pixels);
}

int wn_forward_ragged(wn_handle* h, const wn_ragged_tensors* images_host, int n, int tile_h, int tile_w,
                      long long max_pass_pixels, int mode, void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_forward_ragged";
  int rc = check_ptrs(what, {h, images_host, workspace});
  if (rc) return rc;
  const int s = ragged_check(what, n, tile_h, tile_w, max_pass_pixels, mode);
  if (s < 0) return s;
  if ((rc = check_images(what, images_host, n, true,
                         [](const wn_ragged_tensors& t, int) { return inputs_given(t) && t.out; })) ||
      (rc = check_packed(what, h)))
    return rc;
  DeviceGuard guard(h->device);
  return umma_forward_ragged(h, images_host, n, tile_h, tile_w, max_pass_pixels, workspace, workspace_bytes,
                             (cudaStream_t)stream, s);
}

// ---- the reference's callable sub-modules (net.py:45-56 ConfidenceMapGenerator.forward, :75-80 Refiner.forward)
size_t wn_submodule_workspace_bytes(int n, int h, int w, int mode) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  if (resolve_mode(mode) == WN_MODE_FP32_SIMT) return simt_forward_workspace_bytes(n, h, w);
  // + the three refined images side by side (the refiners run as one block-diagonal stack)
  return align256(umma_forward_workspace_bytes(n, h, w)) + align256((size_t)n * 9 * h * w * sizeof(float)) + 256;
}

int wn_confidence_maps(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                       const int64_t in_strides[4][4], float* out_maps, int n, int height, int width, int mode,
                       void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_confidence_maps";
  int rc = check_args(what, {h, x, wb, he, gc, in_strides, out_maps, workspace}, n, height, width);
  if (rc || (rc = check_packed(what, h)) ||
      (rc = check_workspace(what, workspace_bytes, wn_submodule_workspace_bytes(n, height, width, mode))))
    return rc;
  DeviceGuard guard(h->device);
  const float* in[4] = {x, wb, he, gc};
  const int s = check_mode(what, mode, nullptr);
  if (s == kSchemeSimt)
    return simt_forward(h, in, in_strides, out_maps, n, height, width, workspace, workspace_bytes,
                        (cudaStream_t)stream, kStackCmg, 0);
  if (s < 0) return s;
  return umma_forward(h, in, in_strides, out_maps, n, height, width, workspace, workspace_bytes,
                      (cudaStream_t)stream, s, kStackCmg, nullptr);
}

int wn_refine(wn_handle* h, int which, const float* x, const float* xbar, const int64_t in_strides[2][4],
              float* out, int n, int height, int width, int mode, void* workspace, size_t workspace_bytes,
              void* stream) {
  const char* what = "wn_refine";
  int rc = check_args(what, {h, x, xbar, in_strides, out, workspace}, n, height, width, which >= 0 && which <= 2);
  if (rc || (rc = check_packed(what, h)) ||
      (rc = check_workspace(what, workspace_bytes, wn_submodule_workspace_bytes(n, height, width, mode))))
    return rc;
  DeviceGuard guard(h->device);
  const RefinerInputs r(x, xbar, in_strides);
  const int s = check_mode(what, mode, nullptr);
  if (s == kSchemeSimt)
    return simt_forward(h, r.in, r.st, out, n, height, width, workspace, workspace_bytes, (cudaStream_t)stream,
                        kStackRefiners, which);
  if (s < 0) return s;
  uint8_t* ws = (uint8_t*)(((uintptr_t)workspace + 255) / 256 * 256);
  const size_t fwd_b = align256(umma_forward_workspace_bytes(n, height, width));
  float* refined = (float*)(ws + fwd_b);
  rc = umma_forward(h, r.in, r.st, nullptr, n, height, width, ws, fwd_b, (cudaStream_t)stream, s, kStackRefiners,
                    refined);
  if (rc) return rc;
  const size_t img = (size_t)3 * height * width * sizeof(float);
  WN_CUDA(cudaMemcpy2DAsync(out, img, refined + (size_t)which * 3 * height * width, 3 * img, img, n,
                            cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return WN_OK;
}

// ---- the tiled forward of fp32 tensors (WaterNet.forward and its sub-modules, in windows)
size_t wn_forward_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels,
                                        int mode) {
  if (forward_tiled_check("wn_forward_tiled_workspace_bytes", n, h, w, tile_h, tile_w, max_pass_pixels, mode) < 0)
    return 0;
  return umma_forward_tiled_workspace_bytes(n, h, w, tile_h, tile_w, max_pass_pixels, false);
}

size_t wn_submodule_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels,
                                          int mode) {
  if (forward_tiled_check("wn_submodule_tiled_workspace_bytes", n, h, w, tile_h, tile_w, max_pass_pixels, mode) < 0)
    return 0;
  return umma_forward_tiled_workspace_bytes(n, h, w, tile_h, tile_w, max_pass_pixels, true);
}

// the checks and the call shared by the three fp32 entry points; `what` names the entry point
static int forward_tiled(const char* what, wn_handle* h, const float* const in[4], const int64_t st[4][4], float* out,
                         int n, int height, int width, int tile_h, int tile_w, long long max_pass_pixels, int mode,
                         void* workspace, size_t workspace_bytes, void* stream, int stack, int which) {
  const int s = forward_tiled_check(what, n, height, width, tile_h, tile_w, max_pass_pixels, mode);
  if (s < 0) return s;
  int rc = check_packed(what, h);
  if (rc) return rc;
  DeviceGuard guard(h->device);
  return umma_forward_tiled(h, in, st, out, n, height, width, tile_h, tile_w, max_pass_pixels, workspace,
                            workspace_bytes, (cudaStream_t)stream, s, stack, which);
}

int wn_forward_tiled(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                     const int64_t in_strides[4][4], float* out, int n, int height, int width, int tile_h, int tile_w,
                     long long max_pass_pixels, int mode, void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_forward_tiled";
  int rc = check_ptrs(what, {h, x, wb, he, gc, in_strides, out, workspace});
  if (rc) return rc;
  const float* in[4] = {x, wb, he, gc};
  return forward_tiled(what, h, in, in_strides, out, n, height, width, tile_h, tile_w, max_pass_pixels, mode,
                       workspace, workspace_bytes, stream, kStackAll, 0);
}

int wn_confidence_maps_tiled(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                             const int64_t in_strides[4][4], float* out_maps, int n, int height, int width, int tile_h,
                             int tile_w, long long max_pass_pixels, int mode, void* workspace, size_t workspace_bytes,
                             void* stream) {
  const char* what = "wn_confidence_maps_tiled";
  int rc = check_ptrs(what, {h, x, wb, he, gc, in_strides, out_maps, workspace});
  if (rc) return rc;
  const float* in[4] = {x, wb, he, gc};
  return forward_tiled(what, h, in, in_strides, out_maps, n, height, width, tile_h, tile_w, max_pass_pixels, mode,
                       workspace, workspace_bytes, stream, kStackCmg, 0);
}

int wn_refine_tiled(wn_handle* h, int which, const float* x, const float* xbar, const int64_t in_strides[2][4],
                    float* out, int n, int height, int width, int tile_h, int tile_w, long long max_pass_pixels,
                    int mode, void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_refine_tiled";
  int rc = check_ptrs(what, {h, x, xbar, in_strides, out, workspace});
  if (rc || (rc = check_which(what, which))) return rc;
  const RefinerInputs r(x, xbar, in_strides);
  return forward_tiled(what, h, r.in, r.st, out, n, height, width, tile_h, tile_w, max_pass_pixels, mode, workspace,
                       workspace_bytes, stream, kStackRefiners, which);
}

int wn_set_chunk_pixels(wn_handle* h, long long max_pixels) {
  if (!h || max_pixels < 0) {
    set_error("wn_set_chunk_pixels: bad argument");
    return WN_E_INVALID;
  }
  h->chunk_pixels = max_pixels;
  return WN_OK;
}

int wn_set_train_mode(wn_handle* h, int mode) {
  int rc = check_ptrs("wn_set_train_mode", {h}, "null handle");
  if (rc) return rc;
  if (mode != WN_MODE_BF16X3 && mode != WN_MODE_BF16) {
    set_error("wn_set_train_mode: mode %d is not a training mode (WN_MODE_BF16X3 = 1 or WN_MODE_BF16 = 3)", mode);
    return WN_E_INVALID;
  }
  h->train_bf16 = mode == WN_MODE_BF16;
  return WN_OK;
}

int wn_forward_chunk_images(const wn_handle* h, int n, int height, int width) {
  if (!h || n <= 0 || height <= 0 || width <= 0) return 0;
  return umma_chunk_images(h, n, height, width);
}

int wn_f8_overflowed(const wn_handle* h) { return h ? umma_f8_overflowed(h) : 0; }

uint64_t wn_launch_count(const wn_handle* h) { return h ? h->launches : 0; }

// ---- the training step (wn_forward_train / wn_backward)
size_t wn_train_workspace_bytes(int n, int h, int w) {
  if (n <= 0 || h <= 0 || w <= 0 || n > 65535) return 0;
  return train_workspace_bytes_padded(n, h, w);
}

int wn_forward_train(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                     const int64_t in_strides[4][4], float* out, int n, int height, int width,
                     void* train_workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_forward_train";
  int rc = check_args(what, {h, x, wb, he, gc, in_strides, out, train_workspace}, n, height, width);
  if (rc || (rc = check_packed(what, h)) || (rc = check_images_per_call(what, n))) return rc;
  DeviceGuard guard(h->device);
  const float* in[4] = {x, wb, he, gc};
  return forward_train(h, in, in_strides, out, n, height, width, train_workspace, workspace_bytes,
                       (cudaStream_t)stream);
}

int wn_backward(wn_handle* h, const float* grad_out, float* const* grads, float* const* input_grads, int n,
                int height, int width, void* train_workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_backward";
  int rc = check_args(what, {h, grad_out, grads, train_workspace}, n, height, width);
  if (rc || (rc = check_param_grads(what, grads, 0, WN_NUM_PARAMS)) || (rc = check_packed(what, h)) ||
      (rc = check_images_per_call(what, n)) || (rc = check_input_grads(what, input_grads)))
    return rc;
  DeviceGuard guard(h->device);
  return backward(h, grad_out, grads, input_grads, n, height, width, train_workspace, workspace_bytes,
                  (cudaStream_t)stream);
}

// ---- the ragged training step
// the shape checks the two calls and the workspace function share; 0 = accepted
static int train_ragged_check(const char* what, const int* hs, const int* ws, int n) {
  if (n <= 0) {
    set_error("%s: bad image count n=%d", what, n);
    return WN_E_INVALID;
  }
  int rc = check_images_per_call(what, n);
  if (rc) return rc;
  int sh = 0, sw = 0;
  for (int i = 0; i < n; i++) {
    if (hs[i] <= 0 || ws[i] <= 0) {
      set_error("%s: bad size of image %d: h=%d w=%d", what, i, hs[i], ws[i]);
      return WN_E_INVALID;
    }
    sh = hs[i] > sh ? hs[i] : sh;
    sw = ws[i] > sw ? ws[i] : sw;
  }
  if ((long long)n * sh * sw > kTrainMaxPixels) {
    set_error("%s: %d slots of %dx%d exceed the %lld pixels of one training pass", what, n, sh, sw, kTrainMaxPixels);
    return WN_E_UNSUPPORTED;
  }
  return WN_OK;
}

size_t wn_train_ragged_workspace_bytes(const int* heights_host, const int* widths_host, int n) {
  if (!heights_host || !widths_host ||
      train_ragged_check("wn_train_ragged_workspace_bytes", heights_host, widths_host, n))
    return 0;
  return train_ragged_workspace_bytes(heights_host, widths_host, n);
}

int wn_forward_train_ragged(wn_handle* h, const wn_ragged_tensors* images_host, int n, void* workspace,
                            size_t workspace_bytes, void* stream) {
  const char* what = "wn_forward_train_ragged";
  int rc = check_ptrs(what, {h, images_host, workspace});
  if (rc || (rc = check_ragged_count(what, n)) ||
      (rc = check_images(what, images_host, n, false,
                         [](const wn_ragged_tensors& t, int) { return inputs_given(t) && t.out; })))
    return rc;
  std::vector<int> hs, ws;
  ragged_sizes(images_host, n, &hs, &ws);
  if ((rc = train_ragged_check(what, hs.data(), ws.data(), n)) || (rc = check_packed(what, h))) return rc;
  DeviceGuard guard(h->device);
  return forward_train_ragged(h, images_host, n, workspace, workspace_bytes, (cudaStream_t)stream);
}

int wn_backward_ragged(wn_handle* h, const int* heights_host, const int* widths_host, const float* const* grad_out_host,
                       float* const* grads, float* const* input_grads_host, int n, void* workspace,
                       size_t workspace_bytes, void* stream) {
  const char* what = "wn_backward_ragged";
  int rc = check_ptrs(what, {h, heights_host, widths_host, grad_out_host, grads, workspace});
  if (rc || (rc = check_param_grads(what, grads, 0, WN_NUM_PARAMS)) ||
      (rc = train_ragged_check(what, heights_host, widths_host, n)) ||
      (rc = check_entries(what, "grad_out_host", grad_out_host, 0, n)) || (rc = check_packed(what, h)))
    return rc;
  DeviceGuard guard(h->device);
  return backward_ragged(h, heights_host, widths_host, grad_out_host, grads, input_grads_host, n, workspace,
                         workspace_bytes, (cudaStream_t)stream);
}

// ---- the sub-modules under autograd
// the shape checks the four calls and the workspace function share; 0 = accepted
static int submodule_train_check(const char* what, int n, int height, int width) {
  int rc = check_shape(what, n, height, width);
  if (rc) return rc;
  if (n > 65535 || (long long)n * height * width > kTrainMaxPixels) {
    set_error("%s: at most 65535 images and %lld pixels per call, got n=%d h=%d w=%d", what, kTrainMaxPixels, n,
              height, width);
    return WN_E_UNSUPPORTED;
  }
  return WN_OK;
}
// the backward calls: the sub-module's own parameter gradients [first, first + count) must be given
static int submodule_backward_check(const char* what, wn_handle* h, const float* grad, float* const* grads, int first,
                                    int count, int n, int height, int width, void* ws) {
  int rc = check_ptrs(what, {h, grad, grads, ws});
  if (rc || (rc = check_param_grads(what, grads, first, count)) ||
      (rc = submodule_train_check(what, n, height, width)))
    return rc;
  return check_packed(what, h);
}

size_t wn_submodule_train_workspace_bytes(int n, int h, int w, int stack) {
  if (!submodule_stack(stack) || submodule_train_check("wn_submodule_train_workspace_bytes", n, h, w)) return 0;
  return submodule_train_workspace_bytes(n, h, w, stack == 0 ? kStackCmg : kStackRefiners);
}

int wn_confidence_maps_train(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                             const int64_t in_strides[4][4], float* out_maps, int n, int height, int width, void* ws,
                             size_t ws_bytes, void* stream) {
  const char* what = "wn_confidence_maps_train";
  int rc = check_ptrs(what, {h, x, wb, he, gc, in_strides, out_maps, ws});
  if (rc || (rc = submodule_train_check(what, n, height, width)) || (rc = check_packed(what, h))) return rc;
  DeviceGuard guard(h->device);
  const float* in[4] = {x, wb, he, gc};
  return confidence_maps_train(h, in, in_strides, out_maps, n, height, width, ws, ws_bytes, (cudaStream_t)stream);
}

int wn_confidence_maps_backward(wn_handle* h, const float* grad_maps, float* const* grads, float* const* input_grads,
                                int n, int height, int width, void* ws, size_t ws_bytes, void* stream) {
  int rc = submodule_backward_check("wn_confidence_maps_backward", h, grad_maps, grads, 0, 16, n, height, width, ws);
  if (rc) return rc;
  DeviceGuard guard(h->device);
  return confidence_maps_backward(h, grad_maps, grads, input_grads, n, height, width, ws, ws_bytes,
                                  (cudaStream_t)stream);
}

int wn_refine_train(wn_handle* h, int which, const float* x, const float* xbar, const int64_t in_strides[2][4],
                    float* out, int n, int height, int width, void* ws, size_t ws_bytes, void* stream) {
  const char* what = "wn_refine_train";
  int rc = check_which(what, which);
  if (rc || (rc = check_ptrs(what, {h, x, xbar, in_strides, out, ws})) ||
      (rc = submodule_train_check(what, n, height, width)) || (rc = check_packed(what, h)))
    return rc;
  DeviceGuard guard(h->device);
  const RefinerInputs r(x, xbar, in_strides);
  return refine_train(h, which, r.in, r.st, out, n, height, width, ws, ws_bytes, (cudaStream_t)stream);
}

int wn_refine_backward(wn_handle* h, int which, const float* grad_out, float* const* grads, float* const* input_grads,
                       int n, int height, int width, void* ws, size_t ws_bytes, void* stream) {
  const char* what = "wn_refine_backward";
  int rc = check_which(what, which);
  if (rc || (rc = submodule_backward_check(what, h, grad_out, grads, 16 + 6 * which, 6, n, height, width, ws)))
    return rc;
  DeviceGuard guard(h->device);
  return refine_backward(h, which, grad_out, grads, input_grads, n, height, width, ws, ws_bytes, (cudaStream_t)stream);
}

// ---- the windowed recompute backward (wn_backward_tiled and the sub-modules' and ragged forms)
static int check_train_pass(const char* what, long long max_pass_pixels) {
  if (max_pass_pixels <= kTrainMaxPixels) return WN_OK;
  set_error("%s: max_pass_pixels=%lld exceeds the %lld pixels of one training pass", what, max_pass_pixels,
            kTrainMaxPixels);
  return WN_E_UNSUPPORTED;
}

// the argument checks wn_backward_tiled and its workspace function share (pointers aside)
static int backward_tiled_check(const char* what, int n, int height, int width, int tile_h, int tile_w,
                                long long max_pass_pixels) {
  int rc = check_tiled_shape(what, n, height, width, tile_h, tile_w, max_pass_pixels);
  if (rc || (rc = check_size(n, height, width)) || (rc = check_train_pass(what, max_pass_pixels))) return rc;
  const TileGeom g = tile_geom(height, width, tile_h, tile_w);
  if ((long long)g.win_h * g.win_w > kTrainMaxPixels) {
    set_error("%s: a %dx%d window exceeds the %lld pixels of one training pass; use a smaller tile", what, g.win_h,
              g.win_w, kTrainMaxPixels);
    return WN_E_UNSUPPORTED;
  }
  return WN_OK;
}

size_t wn_backward_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels) {
  if (backward_tiled_check("wn_backward_tiled_workspace_bytes", n, h, w, tile_h, tile_w, max_pass_pixels)) return 0;
  return backward_tiled_workspace_bytes(n, h, w, tile_h, tile_w, max_pass_pixels);
}

int wn_backward_tiled(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                      const int64_t in_strides[4][4], const float* grad_out, float* const* grads,
                      float* const* input_grads, int n, int height, int width, int tile_h, int tile_w,
                      long long max_pass_pixels, void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_backward_tiled";
  int rc = check_ptrs(what, {h, x, wb, he, gc, in_strides, grad_out, grads, workspace});
  if (rc || (rc = check_param_grads(what, grads, 0, WN_NUM_PARAMS)) || (rc = check_input_grads(what, input_grads)) ||
      (rc = backward_tiled_check(what, n, height, width, tile_h, tile_w, max_pass_pixels)) ||
      (rc = check_packed(what, h)))
    return rc;
  DeviceGuard guard(h->device);
  const float* in[4] = {x, wb, he, gc};
  return backward_tiled(h, in, in_strides, grad_out, grads, input_grads, n, height, width, tile_h, tile_w,
                        max_pass_pixels, workspace, workspace_bytes, (cudaStream_t)stream);
}

// ---- the windowed recompute backward of a ragged batch: the limits of wn_backward_tiled, for every image
static int backward_ragged_tiled_check(const char* what, const int* hs, const int* ws, int n, int tile_h, int tile_w,
                                       long long max_pass_pixels) {
  int rc = check_ragged_shape(what, n, tile_h, tile_w, max_pass_pixels);
  if (rc || (rc = check_train_pass(what, max_pass_pixels))) return rc;
  for (int i = 0; i < n; i++) {
    if ((rc = check_ragged_size(what, i, hs[i], ws[i]))) return rc;
    const TileGeom g = tile_geom(hs[i], ws[i], tile_h, tile_w);
    if ((long long)g.win_h * g.win_w > kTrainMaxPixels) {
      set_error("%s: a %dx%d window of image %d exceeds the %lld pixels of one training pass; use a smaller tile",
                what, g.win_h, g.win_w, i, kTrainMaxPixels);
      return WN_E_UNSUPPORTED;
    }
  }
  return WN_OK;
}

size_t wn_backward_ragged_tiled_workspace_bytes(const int* heights_host, const int* widths_host, int n, int tile_h,
                                                int tile_w, long long max_pass_pixels) {
  if (!heights_host || !widths_host ||
      backward_ragged_tiled_check("wn_backward_ragged_tiled_workspace_bytes", heights_host, widths_host, n, tile_h,
                                  tile_w, max_pass_pixels))
    return 0;
  return backward_ragged_tiled_workspace_bytes(heights_host, widths_host, n, tile_h, tile_w, max_pass_pixels);
}

int wn_backward_ragged_tiled(wn_handle* h, const wn_ragged_tensors* images_host, const float* const* grad_out_host,
                             float* const* grads, float* const* input_grads_host, int n, int tile_h, int tile_w,
                             long long max_pass_pixels, void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "wn_backward_ragged_tiled";
  int rc = check_ptrs(what, {h, images_host, grad_out_host, grads, workspace});
  if (rc || (rc = check_param_grads(what, grads, 0, WN_NUM_PARAMS)) || (rc = check_ragged_count(what, n)) ||
      (rc = check_images(what, images_host, n, false,
                         [&](const wn_ragged_tensors& t, int i) { return inputs_given(t) && grad_out_host[i]; })))
    return rc;
  std::vector<int> hs, ws;
  ragged_sizes(images_host, n, &hs, &ws);
  if ((rc = backward_ragged_tiled_check(what, hs.data(), ws.data(), n, tile_h, tile_w, max_pass_pixels)) ||
      (rc = check_packed(what, h)))
    return rc;
  DeviceGuard guard(h->device);
  return backward_ragged_tiled(h, images_host, grad_out_host, grads, input_grads_host, n, tile_h, tile_w,
                               max_pass_pixels, workspace, workspace_bytes, (cudaStream_t)stream);
}

// ---- the windowed recompute backward of one sub-module: the limits of wn_backward_tiled
size_t wn_submodule_backward_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w,
                                                   long long max_pass_pixels, int stack) {
  if (!submodule_stack(stack) ||
      backward_tiled_check("wn_submodule_backward_tiled_workspace_bytes", n, h, w, tile_h, tile_w, max_pass_pixels))
    return 0;
  return submodule_backward_tiled_workspace_bytes(n, h, w, tile_h, tile_w, max_pass_pixels,
                                                  stack == 0 ? kStackCmg : kStackRefiners);
}

int wn_confidence_maps_backward_tiled(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                                      const int64_t in_strides[4][4], const float* grad_maps, float* const* grads,
                                      float* const* input_grads, int n, int height, int width, int tile_h, int tile_w,
                                      long long max_pass_pixels, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  const char* what = "wn_confidence_maps_backward_tiled";
  int rc = check_ptrs(what, {h, x, wb, he, gc, in_strides, grad_maps, grads, workspace});
  if (rc || (rc = check_param_grads(what, grads, 0, 16)) ||
      (rc = backward_tiled_check(what, n, height, width, tile_h, tile_w, max_pass_pixels)) ||
      (rc = check_packed(what, h)))
    return rc;
  DeviceGuard guard(h->device);
  const float* in[4] = {x, wb, he, gc};
  return submodule_backward_tiled(h, kStackCmg, 0, in, in_strides, grad_maps, grads, input_grads, n, height, width,
                                  tile_h, tile_w, max_pass_pixels, workspace, workspace_bytes, (cudaStream_t)stream);
}

int wn_refine_backward_tiled(wn_handle* h, int which, const float* x, const float* xbar, const int64_t in_strides[2][4],
                             const float* grad_out, float* const* grads, float* const* input_grads, int n, int height,
                             int width, int tile_h, int tile_w, long long max_pass_pixels, void* workspace,
                             size_t workspace_bytes, void* stream) {
  const char* what = "wn_refine_backward_tiled";
  int rc = check_which(what, which);
  if (rc || (rc = check_ptrs(what, {h, x, xbar, in_strides, grad_out, grads, workspace})) ||
      (rc = check_param_grads(what, grads, 16 + 6 * which, 6)) ||
      (rc = backward_tiled_check(what, n, height, width, tile_h, tile_w, max_pass_pixels)) ||
      (rc = check_packed(what, h)))
    return rc;
  DeviceGuard guard(h->device);
  const RefinerInputs r(x, xbar, in_strides);
  return submodule_backward_tiled(h, kStackRefiners, which, r.in, r.st, grad_out, grads, input_grads, n, height, width,
                                  tile_h, tile_w, max_pass_pixels, workspace, workspace_bytes, (cudaStream_t)stream);
}

int wn_debug_forward_layer(wn_handle* h, const float* x, const float* wb, const float* he,
                           const float* gc, const int64_t in_strides[4][4], int n, int height,
                           int width, int mode, int layer, float* dst, void* workspace,
                           size_t workspace_bytes, void* stream) {
  const char* what = "wn_debug_forward_layer";
  if (layer < 0 || layer > 10) {
    set_error("%s: layer %d is not in 0..10", what, layer);
    return WN_E_INVALID;
  }
  int rc = check_ptrs(what, {h, x, wb, he, gc, in_strides, dst, workspace}, "bad argument");
  if (rc || (rc = check_packed(what, h))) return rc;
  DeviceGuard guard(h->device);
  const float* in[4] = {x, wb, he, gc};
  if (resolve_mode(mode) == WN_MODE_FP32_SIMT)
    return simt_debug_layer(h, in, in_strides, n, height, width, layer, dst, workspace, workspace_bytes,
                            (cudaStream_t)stream);
  return umma_debug_layer(h, in, in_strides, n, height, width, layer, dst, workspace, workspace_bytes,
                          (cudaStream_t)stream, scheme_of(mode));
}

int wn_debug_backward_layer(wn_handle* h, int stack, int which, int buffer, const float* grad_out,
                            float* const* grads, int n, int height, int width, float* dst, void* workspace,
                            size_t workspace_bytes, void* stream) {
  const char* what = "wn_debug_backward_layer";
  if (buffer < 0 || buffer >= WN_DEBUG_BACKWARD_BUFFERS) {
    set_error("%s: buffer %d is not in 0..%d", what, buffer, WN_DEBUG_BACKWARD_BUFFERS - 1);
    return WN_E_INVALID;
  }
  if (stack < -1 || stack > 1 || (stack == 1 && (which < 0 || which > 2))) {
    set_error("%s: stack must be -1, 0 or 1 (with which 0, 1 or 2), got stack %d which %d", what, stack, which);
    return WN_E_INVALID;
  }
  // grad_out from the seeds on, the parameter gradients from the first data-gradient launch on
  if (!all_set({h, dst, workspace}) || (buffer >= 12 && !grad_out) || (buffer >= 14 && !grads))
    return invalid(what, "null argument");
  int rc;
  // the parameter gradients the backward up to the launch writes: the stack's own entries
  const int first = stack == 1 ? 16 + 6 * which : 0, count = stack == -1 ? WN_NUM_PARAMS : stack == 0 ? 16 : 6;
  if ((buffer >= 14 && (rc = check_param_grads(what, grads, first, count))) ||
      (rc = submodule_train_check(what, n, height, width)) || (rc = check_packed(what, h)))
    return rc;
  DeviceGuard guard(h->device);
  return debug_backward_layer(h, stack == -1 ? kStackAll : stack == 0 ? kStackCmg : kStackRefiners, which, buffer,
                              grad_out, grads, n, height, width, dst, workspace, workspace_bytes,
                              (cudaStream_t)stream);
}

// ---- the VGG19 perceptual loss (vgg.cu)
int wn_vgg_pack_weights(wn_handle* h, const float* const* params, void* stream) {
  const char* what = "wn_vgg_pack_weights";
  int rc = check_ptrs(what, {h, params});
  if (rc || (rc = check_entries(what, "params", params, 0, WN_VGG_NUM_PARAMS))) return rc;
  DeviceGuard guard(h->device);
  return vgg_pack_weights(h, params, (cudaStream_t)stream);
}

size_t wn_perceptual_loss_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels) {
  return vgg_loss_workspace_bytes(n, h, w, tile_h, tile_w, max_pass_pixels);
}

int wn_perceptual_loss(wn_handle* h, const float* out, const int64_t out_strides[4], const float* ref,
                       const int64_t ref_strides[4], int n, int height, int width, int tile_h, int tile_w,
                       long long max_pass_pixels, float* loss_dev, float* grad_out, void* workspace,
                       size_t workspace_bytes, void* stream) {
  int rc = check_ptrs("wn_perceptual_loss", {h, out, out_strides, ref, ref_strides, loss_dev, workspace});
  if (rc) return rc;
  DeviceGuard guard(h->device);
  return vgg_perceptual_loss(h, out, out_strides, ref, ref_strides, n, height, width, tile_h, tile_w, max_pass_pixels,
                             loss_dev, grad_out, workspace, workspace_bytes, (cudaStream_t)stream);
}

int wn_debug_vgg_layer(wn_handle* h, const float* x, const int64_t strides[4], const float* ref,
                       const int64_t ref_strides[4], int n, int height, int width, int tile_h, int tile_w, int layer,
                       float* dst, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_ptrs("wn_debug_vgg_layer", {h, x, strides, dst, workspace});
  if (rc) return rc;
  DeviceGuard guard(h->device);
  return vgg_debug_layer(h, x, strides, ref, ref_strides, n, height, width, tile_h, tile_w, layer, dst, workspace,
                         workspace_bytes, (cudaStream_t)stream);
}

// ---- SSIM / PSNR statistics (metrics.cu)
static_assert(sizeof(wn_quality_image) == 32, "wn_quality_image: _lib.QualityImage restates this layout");

size_t wn_quality_workspace_bytes(const int* heights_host, const int* widths_host, int n) {
  const char* what = "wn_quality_workspace_bytes";
  if (check_ptrs(what, {heights_host, widths_host}) || check_ragged_count(what, n)) return 0;
  return quality_workspace_bytes(heights_host, widths_host, n);
}

int wn_quality(wn_handle* h, const wn_quality_image* images_host, int n, double* stats, void* workspace,
               size_t workspace_bytes, void* stream) {
  const char* what = "wn_quality";
  int rc = check_ptrs(what, {h, images_host, stats, workspace});
  if (rc || (rc = check_ragged_count(what, n)) ||
      (rc = check_images(what, images_host, n, true, [](const wn_quality_image& im, int) { return im.out && im.ref; })))
    return rc;
  for (int i = 0; i < n; i++)
    if (images_host[i].group < 0 || images_host[i].group >= n) {
      set_error("%s: image %d: group %d outside 0..%d", what, i, images_host[i].group, n - 1);
      return WN_E_INVALID;
    }
  if ((uintptr_t)stats % alignof(double)) return invalid(what, "stats is not 8-byte aligned");
  std::vector<int> hs, ws;
  ragged_sizes(images_host, n, &hs, &ws);
  if ((rc = quality_plan_check(hs.data(), ws.data(), n, what)) ||
      (rc = check_workspace(what, workspace_bytes, quality_workspace_bytes(hs.data(), ws.data(), n))))
    return rc;
  DeviceGuard guard(h->device);
  return quality(h, images_host, n, stats, workspace, workspace_bytes, (cudaStream_t)stream);
}

// ---- SSIM's gradient (metrics.cu)
static_assert(sizeof(wn_ssim_grad_image) == 48, "wn_ssim_grad_image: _lib.SSIMGradImage restates this layout");

size_t wn_ssim_grad_workspace_bytes(const int* heights_host, const int* widths_host, int n) {
  const char* what = "wn_ssim_grad_workspace_bytes";
  if (check_ptrs(what, {heights_host, widths_host}) || check_ragged_count(what, n)) return 0;
  return ssim_grad_workspace_bytes(heights_host, widths_host, n);
}

// no grad overlaps any out, ref or other grad: the intervals in order of their start, each writer checked against
// the furthest end of everything before it and each reader against the furthest end of the writers before it
static int check_grad_overlap(const char* what, const wn_ssim_grad_image* images, int n) {
  struct Span {
    uintptr_t begin, end;
    bool writes;
    int image;
  };
  std::vector<Span> spans;
  spans.reserve(3 * (size_t)n);
  for (int i = 0; i < n; i++) {
    const size_t bytes = (size_t)3 * images[i].height * images[i].width * sizeof(float);
    for (const void* p : {(const void*)images[i].out, (const void*)images[i].ref, (const void*)images[i].grad})
      spans.push_back({(uintptr_t)p, (uintptr_t)p + bytes, p == images[i].grad, i});
  }
  std::sort(spans.begin(), spans.end(), [](const Span& a, const Span& b) { return a.begin < b.begin; });
  uintptr_t reach = 0, reach_w = 0;
  for (const Span& s : spans) {
    if (s.begin < (s.writes ? reach : reach_w)) {
      set_error("%s: grad of image %d overlaps an out, ref or grad of the call", what, s.image);
      return WN_E_INVALID;
    }
    reach = std::max(reach, s.end);
    if (s.writes) reach_w = std::max(reach_w, s.end);
  }
  return WN_OK;
}

int wn_ssim_grad(wn_handle* h, const wn_ssim_grad_image* images_host, int n, double* stats, void* workspace,
                 size_t workspace_bytes, void* stream) {
  const char* what = "wn_ssim_grad";
  int rc = check_ptrs(what, {h, images_host, stats, workspace});
  if (rc || (rc = check_ragged_count(what, n)) ||
      (rc = check_images(what, images_host, n, true,
                         [](const wn_ssim_grad_image& im, int) { return im.out && im.ref && im.grad; })))
    return rc;
  for (int i = 0; i < n; i++) {
    if (images_host[i].group < 0 || images_host[i].group >= n) {
      set_error("%s: image %d: group %d outside 0..%d", what, i, images_host[i].group, n - 1);
      return WN_E_INVALID;
    }
    if (!std::isfinite(images_host[i].scale)) {
      set_error("%s: image %d: scale %g is not finite", what, i, images_host[i].scale);
      return WN_E_INVALID;
    }
  }
  if ((uintptr_t)stats % alignof(double)) return invalid(what, "stats is not 8-byte aligned");
  if ((rc = check_grad_overlap(what, images_host, n))) return rc;
  std::vector<int> hs, ws;
  ragged_sizes(images_host, n, &hs, &ws);
  if ((rc = ssim_grad_plan_check(hs.data(), ws.data(), n, what)) ||
      (rc = check_workspace(what, workspace_bytes, ssim_grad_workspace_bytes(hs.data(), ws.data(), n))))
    return rc;
  DeviceGuard guard(h->device);
  return ssim_grad(h, images_host, n, stats, workspace, workspace_bytes, (cudaStream_t)stream);
}

int wn_enable_timing(wn_handle* h, int on) {
  int rc = check_ptrs("wn_enable_timing", {h}, "null handle");
  if (rc) return rc;
  if (!h->timing) h->timing = (Timing*)calloc(1, sizeof(Timing));
  h->timing->on = on != 0;
  h->timing->used = 0;
  return WN_OK;
}

int wn_read_timings(wn_handle* h, float* ms, int* count) {
  int rc = check_ptrs("wn_read_timings", {h, ms, count});
  if (rc) return rc;
  if (!h->timing) return WN_OK;
  DeviceGuard guard(h->device);
  Timing* t = h->timing;
  for (int i = 0; i < t->used; i++) {
    float e = 0.f;
    WN_CUDA(cudaEventElapsedTime(&e, t->a[i], t->b[i]));
    ms[t->slot[i]] += e;
    count[t->slot[i]] += 1;
  }
  t->used = 0;
  return WN_OK;
}

}  // extern "C"
