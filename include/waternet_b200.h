/*
 * waternet_b200 -- C ABI of the H100-native (sm_90a) WaterNet hot path.
 *
 * The reference (tnwei/waternet @ 2091896) is pure Python; it has no FFI.  The
 * boundary it exposes for this path is its Python API, and every entry point
 * below is what a binding for one of those calls would bind (file:line are
 * relative to the reference checkout):
 *
 *   wn_preprocess_u8      waternet/data.py:81-90   transform(rgb) -> wb, gc, he
 *                         + hubconf.py:8-21        arr2ten_noeinops (x/255, HWC->1CHW)
 *                         + hubconf.py:85-91       preprocess(rgb) -> rgb, wb, he, gc tensors
 *   wn_pack_weights       waternet/net.py:12-42,62-70,94-97  the 34-tensor state dict
 *                         (hubconf.py:83 / inference.py:111-120 load_state_dict)
 *   wn_forward            waternet/net.py:99-108   WaterNet.forward(x, wb, ce, gc)
 *   wn_confidence_maps    waternet/net.py:45-56    ConfidenceMapGenerator.forward(x, wb, ce, gc)
 *   wn_refine             waternet/net.py:75-80    Refiner.forward(x, xbar)
 *   wn_forward_tiled,     the same three, computed in overlapping windows: bounded workspace for images of any size
 *   wn_confidence_maps_tiled, wn_refine_tiled
 *   wn_resize_u8          waternet/training_utils.py:94-107  cv2.resize + BGR2RGB of the dataset items
 *   wn_postprocess_u8     hubconf.py:24-34         ten2arr_noeinops (clip, *255, truncate, NCHW->NHWC)
 *   wn_enhance_u8         hubconf.py:85-94 + net.py:99-108: preprocess -> model -> postprocess
 *                         (the per-frame body of inference.py:261-323)
 *   wn_enhance_u8_tiled   the same, computed in overlapping windows: bounded workspace for images of any size
 *   wn_enhance_u8_ragged  the same for n images of n sizes in one call (inference.py --source <directory>)
 *   wn_forward_ragged     wn_forward for n images of n sizes in one call
 *   wn_forward_train /    train.py:108 `out = model(...)` and train.py:130-131 `loss.backward()`
 *   wn_backward           (autograd through net.py:99-108)
 *   wn_forward_train_ragged / wn_backward_ragged
 *                         the same for n images of n sizes in one call (a dataset without a fixed size)
 *   wn_backward_tiled     the same gradients from the inputs alone, recomputed in overlapping windows
 *   wn_backward_ragged_tiled
 *                         ... for n images of n sizes in one call
 *   wn_confidence_maps_train / _backward, wn_refine_train / _backward
 *                         the sub-modules under autograd (net.py:45-56, :75-80 with parameters that require grad)
 *   wn_confidence_maps_backward_tiled, wn_refine_backward_tiled
 *                         their gradients from the inputs alone, recomputed in overlapping windows
 *
 * Conventions: every data pointer is a DEVICE pointer on the handle's device
 * unless its name ends in _host; the caller owns every buffer (the handle only
 * owns its packed weights and constant tables); every call is asynchronous on
 * `stream` (a cudaStream_t passed as void*); return 0 on success, a negative
 * WN_E_* code otherwise with a message available from wn_last_error() (thread
 * local).  A handle may be used from one thread at a time.
 */
#ifndef WATERNET_B200_H_
#define WATERNET_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WN_ABI_VERSION 11

#define WN_OK 0
#define WN_E_INVALID (-1)   /* bad argument (NULL pointer, non-positive size, unknown mode) */
#define WN_E_CUDA (-2)      /* a CUDA call failed; wn_last_error() has cudaGetErrorString */
#define WN_E_STATE (-3)     /* call order: forward before wn_pack_weights, etc. */
#define WN_E_WORKSPACE (-4) /* workspace smaller than wn_*_workspace_bytes() */
#define WN_E_UNSUPPORTED (-5)

/* Arithmetic used for the 17 convolutions of wn_forward. */
#define WN_MODE_FP32_SIMT 0 /* fp32 FMA on CUDA cores (bit-for-bit independent of tensor cores) */
#define WN_MODE_BF16X3 1    /* wgmma tensor cores, 3-term bf16 split operands, fp32 accumulate */
#define WN_MODE_BF16_FP8 2  /* same, the two correction terms of the tensor-bound layers as one fp8 MMA */
#define WN_MODE_DEFAULT (-1) /* the library's fastest mode that meets the 1e-3 parity bar: WN_MODE_BF16_FP8 */
/* Not a forward mode: the training arithmetic of wn_set_train_mode (3), one bf16 wgmma per product, fp32 accumulate */
#define WN_MODE_BF16 (WN_MODE_BF16_FP8 + 1)

#define WN_NUM_PARAMS 34

typedef struct wn_handle wn_handle;

int wn_abi_version(void);
const char* wn_last_error(void);

/* One handle per device.  Builds the constant tables (sRGB / Lab / gamma). */
int wn_create(int device, wn_handle** out);
void wn_destroy(wn_handle* h);

/*
 * Host-only: fill the constant tables the preprocess kernels use, so that they
 * can be checked on a machine without a GPU.  Sizes: gtab[256], ctab[3072],
 * ytab[256], fytab[256], igtab[4096], gamma[256], div255[256].
 */
int wn_build_tables_host(uint16_t* gtab, uint16_t* ctab, int16_t* ytab, int16_t* fytab,
                         uint8_t* igtab, uint8_t* gamma, float* div255);

/*
 * params: WN_NUM_PARAMS device pointers to contiguous fp32 tensors in the order of
 * WaterNet().state_dict(): cmg.conv1.weight, cmg.conv1.bias, ... cmg.conv8.bias,
 * wb_refiner.conv1.weight ... gc_refiner.conv3.bias; weights are OIHW.
 * Re-packs them into the kernels' layouts (device side, asynchronous).
 */
int wn_pack_weights(wn_handle* h, const float* const* params, void* stream);

/*
 * WaterNet.forward.  x/wb/he/gc: fp32 (N,3,H,W) with arbitrary element strides
 * in_strides[i] = {sN, sC, sH, sW} (contiguous NCHW and the channels_last strides
 * arr2ten produces are both accepted).  out: fp32 contiguous NCHW (N,3,H,W).
 */
size_t wn_forward_workspace_bytes(int n, int h, int w, int mode);
int wn_forward(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
               const int64_t in_strides[4][4], float* out, int n, int height, int width, int mode,
               void* workspace, size_t workspace_bytes, void* stream);

/*
 * transform + arr2ten.  rgb: uint8 NHWC (N,H,W,3).  Any output pointer may be
 * NULL.  fp32 outputs are contiguous NCHW (N,3,H,W) in [0,1] (u/255, true
 * division); *_u8 outputs are NHWC like the reference's numpy arrays.
 * Statistics (white balance quantiles, CLAHE tiles) are per image.
 */
size_t wn_preprocess_workspace_bytes(int n, int h, int w);
int wn_preprocess_u8(wn_handle* h, const uint8_t* rgb, int n, int height, int width, float* x,
                     float* wb, float* he, float* gc, uint8_t* wb_u8, uint8_t* he_u8,
                     uint8_t* gc_u8, void* workspace, size_t workspace_bytes, void* stream);

/*
 * The grayscale branch of white_balance_transform (waternet/data.py:30-36: saturation levels 0.001 / 0.005):
 * gray / out are uint8 (N,H,W).  No caller in the reference uses it; provided for completeness of data.py.
 */
size_t wn_white_balance_gray_workspace_bytes(int n, int h, int w);
int wn_white_balance_gray_u8(wn_handle* h, const uint8_t* gray, uint8_t* out, int n, int height, int width,
                             void* workspace, size_t workspace_bytes, void* stream);

/*
 * Batched cv2.resize(img, (dst_w, dst_h)) of 8-bit 3-channel images, default INTER_LINEAR, as the training
 * dataset applies it per item (waternet/training_utils.py:94-103) -- bit-exact OpenCV arithmetic.  src_dev,
 * src_h, src_w are HOST arrays of n entries: device pointers to HWC uint8 images and their sizes.  dst_nhwc:
 * (n, dst_h, dst_w, 3).  swap_rb != 0 also applies the BGR<->RGB swap that follows the resize
 * (training_utils.py:106-107).
 */
int wn_resize_u8(wn_handle* h, const uint8_t* const* src_dev, const int* src_h, const int* src_w, int n,
                 uint8_t* dst_nhwc, int dst_h, int dst_w, int swap_rb, void* stream);

/* ten2arr: fp32 NCHW (N,3,H,W) -> uint8 NHWC, clip to [0,1], *255, truncate. */
int wn_postprocess_u8(wn_handle* h, const float* out_nchw, uint8_t* out_nhwc, int n, int height,
                      int width, void* stream);

/*
 * The reference's callable sub-modules, evaluated with the weights of the packed state dict.
 * wn_confidence_maps: the three sigmoid maps as one fp32 contiguous (N,3,H,W) tensor (channel r = the map
 * net.py:55 returns as out<r+1>).  wn_refine: refiner `which` (0 = wb_refiner, 1 = ce_refiner, 2 = gc_refiner)
 * applied to cat[x, xbar]; in_strides[0] / [1] are the element strides of x / xbar; out fp32 contiguous
 * (N,3,H,W).  Both take the workspace of wn_submodule_workspace_bytes.
 */
size_t wn_submodule_workspace_bytes(int n, int h, int w, int mode);
int wn_confidence_maps(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                       const int64_t in_strides[4][4], float* out_maps, int n, int height, int width, int mode,
                       void* workspace, size_t workspace_bytes, void* stream);
int wn_refine(wn_handle* h, int which, const float* x, const float* xbar, const int64_t in_strides[2][4],
              float* out, int n, int height, int width, int mode, void* workspace, size_t workspace_bytes,
              void* stream);

/*
 * wn_forward, wn_confidence_maps and wn_refine with a workspace that does not grow with the image: the same bits,
 * computed in windows.  The untiled calls run whole images per pass (~1.9 KB of workspace per pixel, so one 45 MP
 * photo needs more than an 80 GB card).  Each image is cut into the windows of wn_enhance_u8_tiled (balanced output
 * tiles of at most tile_h x tile_w, each computed from a window up to 13 pixels larger per side, clamped into the
 * image); a pass runs as many windows as fit in max_pass_pixels (0 = 8 Mi pixels; at least one window).  The first
 * layer drops its a_lo pass when every input value of the call is an 8-bit level (u/255), as wn_forward does for a
 * batch it runs in one pass; the results then equal those of the untiled calls bit for bit.  Inputs and strides as
 * wn_forward / wn_refine; the outputs are fp32 contiguous NCHW (N,3,H,W).
 * Workspace: wn_forward_tiled_workspace_bytes for wn_forward_tiled, wn_submodule_tiled_workspace_bytes for the two
 * sub-modules (one pass of windows, ~1.9 KB per window pixel, plus 36 B per window pixel for the sub-modules),
 * whatever the image size.  Tensor-core modes only (WN_MODE_FP32_SIMT: WN_E_UNSUPPORTED); the size limits of
 * wn_enhance_u8_tiled.  max_pass_pixels is this call's own argument (wn_set_chunk_pixels does not apply).  Nothing
 * is copied from the host, so a call can be captured in a CUDA graph.  The workspace functions return 0 for
 * arguments the calls reject.
 */
size_t wn_forward_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels,
                                        int mode);
int wn_forward_tiled(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                     const int64_t in_strides[4][4], float* out, int n, int height, int width, int tile_h, int tile_w,
                     long long max_pass_pixels, int mode, void* workspace, size_t workspace_bytes, void* stream);
size_t wn_submodule_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels,
                                          int mode);
int wn_confidence_maps_tiled(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                             const int64_t in_strides[4][4], float* out_maps, int n, int height, int width, int tile_h,
                             int tile_w, long long max_pass_pixels, int mode, void* workspace, size_t workspace_bytes,
                             void* stream);
int wn_refine_tiled(wn_handle* h, int which, const float* x, const float* xbar, const int64_t in_strides[2][4],
                    float* out, int n, int height, int width, int tile_h, int tile_w, long long max_pass_pixels,
                    int mode, void* workspace, size_t workspace_bytes, void* stream);

/*
 * preprocess -> forward -> postprocess without leaving the device.  In the tensor-core modes nothing fp32 is
 * materialised: the per-pixel preprocess kernel writes the first layer's operand planes (8-bit levels, the /255
 * of arr2ten is folded into the first layer's weights) and the last launch's epilogue writes the uint8 image
 * (and the fp32 output too when out_f32_or_null is given).
 */
size_t wn_enhance_workspace_bytes(int n, int h, int w, int mode);
int wn_enhance_u8(wn_handle* h, const uint8_t* rgb, uint8_t* out_nhwc, float* out_f32_or_null,
                  int n, int height, int width, int mode, void* workspace, size_t workspace_bytes,
                  void* stream);

/*
 * wn_enhance_u8 with a workspace that does not grow with the image: the same bits, computed in windows.
 * wn_enhance_u8 runs whole images per pass (~1.9 KB of workspace per pixel, so one 45 MP photo needs more than
 * an 80 GB card).  Every output pixel depends on the input within 13 pixels, so each image is cut into balanced
 * output tiles of at most tile_h x tile_w, each computed from a window that extends it by up to 13 pixels per side
 * (clamped into the image; all windows of a call have one size).  The statistics of the preprocess (white balance,
 * CLAHE) are taken over the full images.  A pass runs as many windows as fit in max_pass_pixels (0 = 8 Mi pixels;
 * at least one window); the workspace is that pass plus ~84 KB per image of LUTs, whatever the image size.  With
 * tile 998 x 998 a window is at most 1024 x 1024.  The result equals wn_enhance_u8's bit for bit.
 * Tensor-core modes only (WN_MODE_FP32_SIMT: WN_E_UNSUPPORTED); no peer outputs.  max_pass_pixels is this call's
 * own argument (wn_set_chunk_pixels does not apply), so that the workspace function and the call agree.
 * The workspace function returns 0 for arguments the call rejects.
 */
size_t wn_enhance_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels,
                                        int mode);
int wn_enhance_u8_tiled(wn_handle* h, const uint8_t* rgb, uint8_t* out_nhwc, float* out_f32_or_null,
                        int n, int height, int width, int tile_h, int tile_w, long long max_pass_pixels,
                        int mode, void* workspace, size_t workspace_bytes, void* stream);

/*
 * A ragged batch: n images, each of its own size, enhanced in one call (a directory of photos).  Image i is cut into
 * exactly the windows wn_enhance_u8_tiled would use for it alone (tile_h x tile_w; a small image is one window).
 * The windows of all images are sorted by shape and packed into passes of equally sized slots, each window at its
 * slot's top-left, with the slot pixels outside it held at zero; a pass holds at most max_pass_pixels slot pixels
 * (0 = 8 Mi; at least one window), at most 65535 windows, and -- when it holds more than one -- at most 25 % of
 * zero padding.  The outputs of image i equal, bit for bit, what wn_enhance_u8 returns for image i alone, in both
 * tensor-core modes, provided the e4m3 range guard stays down: the guard's flag is sticky, so once a pass raises it,
 * that pass and every later one are recomputed with the bf16x3 kernels, including images that did not raise it.
 * Workspace: the largest pass (~1.9 KB per slot pixel) plus ~84 KB of LUTs per image plus the window table; it does
 * not grow with any image's size.  images_host is a HOST array of n entries with device pointers; out_f32 may be
 * NULL per image.  Tensor-core modes only (WN_MODE_FP32_SIMT: WN_E_UNSUPPORTED); no peer outputs.  The call copies
 * its plan to the device from pageable host memory once, so it cannot be captured in a CUDA graph.
 * The workspace function returns 0 for arguments the call rejects.
 */
typedef struct {
  const uint8_t* rgb;  /* device, HWC uint8 (height, width, 3), contiguous */
  uint8_t* out_u8;     /* device, HWC uint8, same size */
  float* out_f32;      /* device, fp32 NCHW (1, 3, height, width), or NULL */
  int height, width;
} wn_ragged_image;
size_t wn_enhance_ragged_workspace_bytes(const int* heights_host, const int* widths_host, int n, int tile_h,
                                         int tile_w, long long max_pass_pixels, int mode);
int wn_enhance_u8_ragged(wn_handle* h, const wn_ragged_image* images_host, int n, int tile_h, int tile_w,
                         long long max_pass_pixels, int mode, void* workspace, size_t workspace_bytes, void* stream);

/*
 * WaterNet.forward of a ragged batch of fp32 tensors: n images, each of its own size, in one call.  The windows,
 * passes, limits and workspace bound of wn_enhance_u8_ragged (tile_h x tile_w windows, max_pass_pixels slot pixels
 * per pass, 0 = 8 Mi, 25 % padding, 65535 windows per pass).  images_host is a HOST array of n descriptors with device
 * pointers: the four inputs with their element strides (as in_strides of wn_forward; sN is not used) and the fp32
 * contiguous (1,3,height,width) output.  Whether the first layer drops its a_lo pass is decided once over every input
 * pixel of the n images, as wn_forward_tiled decides it.  The output of image i equals, bit for bit, what wn_forward
 * returns for image i alone, in both tensor-core modes, while the e4m3 range guard stays down (the guard's flag is
 * sticky, as in wn_enhance_u8_ragged).  Tensor-core modes only (WN_MODE_FP32_SIMT: WN_E_UNSUPPORTED).  The call copies
 * its plan to the device from pageable host memory once, so it cannot be captured in a CUDA graph.  The workspace
 * function returns 0 for arguments the call rejects.
 */
typedef struct {
  const float* x;  /* device, fp32 (1,3,height,width) with the strides below */
  const float* wb;
  const float* he;
  const float* gc;
  int64_t in_strides[4][4]; /* {sN, sC, sH, sW} of x, wb, he, gc */
  float* out;               /* device, fp32 contiguous (1,3,height,width) */
  int height, width;
} wn_ragged_tensors;
size_t wn_forward_ragged_workspace_bytes(const int* heights_host, const int* widths_host, int n, int tile_h,
                                         int tile_w, long long max_pass_pixels, int mode);
int wn_forward_ragged(wn_handle* h, const wn_ragged_tensors* images_host, int n, int tile_h, int tile_w,
                      long long max_pass_pixels, int mode, void* workspace, size_t workspace_bytes, void* stream);

/*
 * wn_enhance_u8 with the all-gather of the output fused into the kernel that produces it (SURVEY 8e: the one
 * exchange of the sharded path): the launch that writes out_nhwc stores the same bytes to peer_out[0..n_peers) --
 * addresses inside the other ranks' buffers, mapped with wn_peer_open (NVLink stores), each the start of where THIS
 * batch belongs there.  Any alignment works; 4-byte aligned rows leave as whole 96-byte segments (16-byte aligned
 * buffers as 16-byte copies in the copy-kernel forms), anything else byte by byte.  In the default mode that launch is
 * the HBM-bound gather/gate kernel at the end of every pass, so the exchange of a pass rides on a kernel that
 * leaves the tensor cores and most of the power budget idle; the other modes (and the range guard's re-run)
 * finish with a copy kernel.  Completion at the peers is the caller's business (wn_stream_write_value32 +
 * wn_memcpy_async of the flag word + wn_stream_wait_value32, see below).
 */
#define WN_MAX_PEERS 15
int wn_enhance_u8_peers(wn_handle* h, const uint8_t* rgb, uint8_t* out_nhwc, float* out_f32_or_null,
                        uint8_t* const* peer_out, int n_peers, int n, int height, int width, int mode,
                        void* workspace, size_t workspace_bytes, void* stream);

/*
 * Training step (reference train.py:100-133: out = model(...); loss.backward()).
 * wn_forward_train is wn_forward (tensor-core mode) that additionally keeps every activation in
 * `train_workspace`; wn_backward consumes that workspace and d(loss)/d(out) (fp32 contiguous NCHW)
 * and OVERWRITES the 34 gradient tensors `grads` (device pointers, same order, shapes and layout as
 * `params` of wn_pack_weights).  input_grads is NULL or four device pointers to fp32 contiguous
 * (N,3,H,W) tensors that receive d(loss)/d(x), d/d(wb), d/d(he), d/d(gc).
 * The workspace must stay untouched between the two calls; n*h*w <= 8 Mi pixels and n <= 65535 images per call
 * (wn_train_workspace_bytes returns 0 beyond that).
 */
size_t wn_train_workspace_bytes(int n, int h, int w);

/*
 * The arithmetic of the training calls of this handle: WN_MODE_BF16X3 (the default of a new handle: three bf16
 * products per product, ~1e-5 of fp32) or WN_MODE_BF16 (one bf16 product, a_hi x w_hi, with fp32 accumulation: the
 * operands rounded to bf16 once, as autocast trains convolutions).  Any other mode returns WN_E_INVALID.  A host-side
 * setting: no device pointer, no launch.  It is read by wn_forward_train / wn_backward, wn_forward_train_ragged /
 * wn_backward_ragged, wn_backward_tiled, wn_backward_ragged_tiled, wn_confidence_maps_train / _backward / _backward_tiled,
 * wn_refine_train / _backward / _backward_tiled and wn_debug_backward_layer: their training forward, seeds, data
 * gradients and weight gradients all run in it.  wn_perceptual_loss and wn_debug_vgg_layer read it too: their VGG
 * convolutions, data gradients, packed image and seed run in it (DESIGN.md 4.14).  In WN_MODE_BF16 every stored
 * activation and gradient plane holds bf16(v) with lo = 0; the workspace sizes do not change.  A backward must run under the mode of the forward that
 * filled its workspace.  The inference calls ignore the setting (and reject WN_MODE_BF16 as their `mode`).
 * WN_ABI_VERSION stays 11: an addition, no existing signature or structure changed (as with wn_backward_ragged_tiled).
 */
int wn_set_train_mode(wn_handle* h, int mode);
int wn_forward_train(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                     const int64_t in_strides[4][4], float* out, int n, int height, int width,
                     void* train_workspace, size_t workspace_bytes, void* stream);
int wn_backward(wn_handle* h, const float* grad_out, float* const* grads, float* const* input_grads, int n,
                int height, int width, void* train_workspace, size_t workspace_bytes, void* stream);

/*
 * The training step of a ragged batch: n images of their own sizes as ONE pass of n equally sized slots (the
 * per-axis maximum of the sizes), each image at its slot's top-left; n * slot pixels <= 8 Mi and n <= 65535
 * (wn_train_ragged_workspace_bytes returns 0 for every argument set the calls reject).
 *   - wn_forward_train_ragged: wn_forward_train of every image (the WN_MODE_BF16X3 arithmetic; the exact-levels
 *     decision over every input pixel of the n images), keeping the activations in `workspace`.  Descriptors as
 *     wn_forward_ragged.  Slot pixels beyond an image are stored as zeros by every ReLU layer.
 *   - wn_backward_ragged: consumes that workspace (untouched in between) and d(loss)/d(out) of every image.
 *     heights_host / widths_host: the sizes of the forward call, in its order.  They fix where the call finds the
 *     activations; the forward records its image count and slot in the workspace, and a backward whose sizes give
 *     another count or slot stops with a device-side assertion (the CUDA context is then unusable).  grad_out_host: HOST array of n device
 *     pointers to fp32 contiguous (1,3,H_i,W_i).  grads: as wn_backward, OVERWRITTEN with the gradients of the sum
 *     of the n images' losses.  input_grads_host: NULL or a HOST array of 4n device pointers, image i's d/d(x),
 *     d/d(wb), d/d(he), d/d(gc) at 4i .. 4i+3, fp32 contiguous (1,3,H_i,W_i); any entry may be NULL.
 * Image i's output and input gradients equal those of wn_forward_train / wn_backward on image i alone bit for bit;
 * the parameter gradients equal the sum of the per-image ones up to the order of the fp32 sums.  Both calls copy a
 * small table from pageable host memory, so they cannot be captured in a CUDA graph.
 */
size_t wn_train_ragged_workspace_bytes(const int* heights_host, const int* widths_host, int n);
int wn_forward_train_ragged(wn_handle* h, const wn_ragged_tensors* images_host, int n, void* workspace,
                            size_t workspace_bytes, void* stream);
int wn_backward_ragged(wn_handle* h, const int* heights_host, const int* widths_host, const float* const* grad_out_host,
                       float* const* grads, float* const* input_grads_host, int n, void* workspace,
                       size_t workspace_bytes, void* stream);

/*
 * The sub-modules under autograd (a ConfidenceMapGenerator or a Refiner trained on its own): the training step of
 * wn_forward_train / wn_backward for one stack.
 *   - The forward calls compute what wn_confidence_maps / wn_refine compute, in the WN_MODE_BF16X3 arithmetic of
 *     wn_forward_train (the first layer drops its a_lo pass when every input value is an 8-bit level), and keep the
 *     stack's activations in `ws`.  out_maps: the (N,3,H,W) maps; out: the refined image of refiner `which`
 *     (0 = wb_refiner, 1 = ce_refiner, 2 = gc_refiner).  Inputs and strides as wn_confidence_maps / wn_refine.
 *     A refiner's first layer is the refiners' conv1 alone: it does not pay for cmg.conv1.
 *   - The backward calls consume that workspace and d(loss)/d(maps) or d(loss)/d(out) (fp32 contiguous NCHW).
 *     grads has the WN_NUM_PARAMS layout of wn_backward; only the sub-module's own entries are written (overwritten):
 *     0..15 for the cmg, 16 + 6 which .. 21 + 6 which for refiner `which`.  The other entries are ignored and may be
 *     NULL.  input_grads is NULL or 4 pointers (cmg: x, wb, he, gc) or 2 (refiner: x, xbar) to fp32 contiguous
 *     (N,3,H,W) tensors; any entry may be NULL.
 *   - stack: 0 = confidence maps, 1 = refiner.  The workspace holds that stack's activations and gradients only
 *     (~3.9 KB per pixel for the cmg, ~1.8 KB for a refiner, plus ~52 MB).  n*h*w <= 8 Mi pixels and n <= 65535
 *     per call; wn_submodule_train_workspace_bytes returns 0 for arguments the calls reject.  The workspace must stay
 *     untouched between the forward and the backward call of the same stack and `which`.
 */
size_t wn_submodule_train_workspace_bytes(int n, int h, int w, int stack);
int wn_confidence_maps_train(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                             const int64_t in_strides[4][4], float* out_maps, int n, int height, int width, void* ws,
                             size_t ws_bytes, void* stream);
int wn_confidence_maps_backward(wn_handle* h, const float* grad_maps, float* const* grads, float* const* input_grads,
                                int n, int height, int width, void* ws, size_t ws_bytes, void* stream);
int wn_refine_train(wn_handle* h, int which, const float* x, const float* xbar, const int64_t in_strides[2][4],
                    float* out, int n, int height, int width, void* ws, size_t ws_bytes, void* stream);
int wn_refine_backward(wn_handle* h, int which, const float* grad_out, float* const* grads, float* const* input_grads,
                       int n, int height, int width, void* ws, size_t ws_bytes, void* stream);

/*
 * The windowed recompute backward: the gradients wn_backward gives, from the four inputs alone, in memory that does
 * not grow with the image size.  The images are cut into the windows of wn_forward_tiled (tile_h x tile_w output
 * tiles, 13 pixels of context per side).  For each pass of windows the call recomputes the training forward (the
 * WN_MODE_BF16X3 arithmetic, the first layer's exact-levels decision taken over all input pixels, as
 * wn_forward_tiled takes it) and runs the backward pass with d(loss)/d(out) taken inside each window's kept
 * rectangle and 0 elsewhere.  The result equals the untiled gradients up to the order of the fp32 sums.
 *   - x, wb, he, gc, in_strides: as wn_forward_tiled.  grad_out: fp32 contiguous (N,3,H,W) of the full images.
 *   - grads, input_grads: as wn_backward, overwritten.
 *   - max_pass_pixels: window pixels per pass, 0 = 2 Mi (~11.8 GB of workspace); at most 8 Mi, and a single window
 *     may not exceed 8 Mi pixels either.  n <= 65535 and h * w <= 715,827,882 as the tiled forward.
 *   - Deterministic, no atomics.  Input gradients are added window by window in window order, so they do not depend
 *     on max_pass_pixels; the parameter gradients do (through the pixel split of the weight-gradient GEMMs).
 *   - Nothing is copied from the host: a call can be captured in a CUDA graph.
 * wn_backward_tiled_workspace_bytes returns 0 for every argument set the call rejects.
 */
size_t wn_backward_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w, long long max_pass_pixels);
int wn_backward_tiled(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                      const int64_t in_strides[4][4], const float* grad_out, float* const* grads,
                      float* const* input_grads, int n, int height, int width, int tile_h, int tile_w,
                      long long max_pass_pixels, void* workspace, size_t workspace_bytes, void* stream);

/*
 * The windowed recompute backward of a ragged batch: wn_backward_tiled for n images of their own sizes in one call.
 * Every image is cut into the windows wn_backward_tiled cuts it into; the windows of all images are sorted by shape
 * and packed into passes of equally sized slots, as wn_forward_ragged packs them.  For each pass the call recomputes
 * the training forward (the WN_MODE_BF16X3 arithmetic; the exact-levels decision over every input pixel of the n
 * images, as wn_forward_ragged takes it) and runs the backward pass with d(loss)/d(out) taken inside each window's kept
 * rectangle and 0 elsewhere.
 *   - images_host: HOST array of n wn_ragged_tensors (the inputs of the forward; `out` is not used and may be NULL).
 *   - grad_out_host: HOST array of n device pointers to fp32 contiguous (1,3,H_i,W_i).  grads: as wn_backward,
 *     OVERWRITTEN with the gradients of the sum of the n images' losses.  input_grads_host: NULL or a HOST array of
 *     4n device pointers, image i's d/d(x), d/d(wb), d/d(he), d/d(gc) at 4i .. 4i+3, fp32 contiguous (1,3,H_i,W_i);
 *     any entry may be NULL.
 *   - max_pass_pixels: slot pixels per pass, 0 = 2 Mi; at most 8 Mi.  A pass of one window may exceed it, but no
 *     window may exceed 8 Mi pixels.  At most 65535 windows per pass; n <= 65535.
 *   - Image i's input gradients equal those of wn_backward_tiled on image i alone at the same tile, bit for bit, and
 *     do not depend on max_pass_pixels or on the other images.  The parameter gradients equal the sum of the
 *     per-image ones up to the order of the fp32 sums; for n images of one size they equal wn_backward_tiled of the
 *     batch bit for bit.  Deterministic, no atomics.
 *   - The call copies its plan to the device from pageable host memory once, so it cannot be captured in a CUDA
 *     graph.  The workspace is one pass of training buffers, the scratch parameter gradients and the plan.
 * wn_backward_ragged_tiled_workspace_bytes returns 0 for every argument set the call rejects.
 */
size_t wn_backward_ragged_tiled_workspace_bytes(const int* heights_host, const int* widths_host, int n, int tile_h,
                                                int tile_w, long long max_pass_pixels);
int wn_backward_ragged_tiled(wn_handle* h, const wn_ragged_tensors* images_host, const float* const* grad_out_host,
                             float* const* grads, float* const* input_grads_host, int n, int tile_h, int tile_w,
                             long long max_pass_pixels, void* workspace, size_t workspace_bytes, void* stream);

/*
 * The windowed recompute backward of one sub-module: the gradients wn_confidence_maps_backward / wn_refine_backward
 * give, from the sub-module's inputs alone, in memory that does not grow with the image size.  The windows, the
 * recomputed WN_MODE_BF16X3 training forward (of that stack alone, as wn_confidence_maps_train / wn_refine_train run
 * it) and the exactness argument are those of wn_backward_tiled; a refiner's receptive-field radius (6) is within
 * the windows' 13 pixels of context.
 *   - x, wb, he, gc / x, xbar, in_strides: as wn_confidence_maps_tiled / wn_refine_tiled.  grad_maps / grad_out:
 *     fp32 contiguous (N,3,H,W) of the full images.
 *   - grads, input_grads: as wn_confidence_maps_backward / wn_refine_backward (only the stack's own entries of grads
 *     are overwritten, the others may be NULL; input_grads NULL or 4 / 2 pointers, any of them NULL).
 *   - max_pass_pixels and the size limits: as wn_backward_tiled.  stack: 0 = confidence maps, 1 = refiner.  At the
 *     default pass of 2 Mi window pixels the workspace is at most ~8.1 GB for the cmg and ~3.9 GB for a refiner.
 *   - Deterministic, no atomics; input gradients are folded in window order and do not depend on max_pass_pixels.
 *   - Nothing is copied from the host: a call can be captured in a CUDA graph.
 * wn_submodule_backward_tiled_workspace_bytes returns 0 for every argument set the calls reject.
 */
size_t wn_submodule_backward_tiled_workspace_bytes(int n, int h, int w, int tile_h, int tile_w,
                                                   long long max_pass_pixels, int stack);
int wn_confidence_maps_backward_tiled(wn_handle* h, const float* x, const float* wb, const float* he, const float* gc,
                                      const int64_t in_strides[4][4], const float* grad_maps, float* const* grads,
                                      float* const* input_grads, int n, int height, int width, int tile_h, int tile_w,
                                      long long max_pass_pixels, void* workspace, size_t workspace_bytes, void* stream);
int wn_refine_backward_tiled(wn_handle* h, int which, const float* x, const float* xbar, const int64_t in_strides[2][4],
                             const float* grad_out, float* const* grads, float* const* input_grads, int n, int height,
                             int width, int tile_h, int tile_w, long long max_pass_pixels, void* workspace,
                             size_t workspace_bytes, void* stream);

/*
 * Per-kernel device timing (measurement aid for bench.py, off by default).  When on, every
 * kernel group is bracketed by a cudaEvent pair on the launching stream.  wn_read_timings
 * must be called after the stream has been synchronised; it adds the elapsed milliseconds and
 * the number of bracketed launches per slot into ms[] / count[] (WN_NUM_TIMING_SLOTS entries:
 * 0..16 the convolutions in state-dict order, 17 operand packing, 18 gated sum, 19 preprocess
 * statistics, 20 LUT build, 21 per-pixel apply, 22 postprocess) and clears the record.
 */
#define WN_NUM_TIMING_SLOTS 23
int wn_enable_timing(wn_handle* h, int on);
int wn_read_timings(wn_handle* h, float* ms, int* count);

/*
 * Test aid: run wn_forward's layer chain in `mode` up to an intermediate activation and return it
 * as contiguous fp32 NCHW.  layer: 0..6 = output of cmg.conv1..conv7 (after ReLU), 7 = the three
 * sigmoid confidence maps, 8 = the three refiners' conv1 outputs concatenated (96 channels),
 * 9 = their conv2 outputs (96 channels), 10 = the three refined images (conv3 after ReLU, before the
 * gate; 9 channels, 3r..3r+2 for refiner r).  dst must hold n*C*h*w floats.  Workspace as wn_forward.
 */
int wn_debug_forward_layer(wn_handle* h, const float* x, const float* wb, const float* he,
                           const float* gc, const int64_t in_strides[4][4], int n, int height,
                           int width, int mode, int layer, float* dst, void* workspace,
                           size_t workspace_bytes, void* stream);

/*
 * Test aid: one buffer of the training backward, decoded to contiguous fp32 NCHW (bf16 hi + lo planes as hi + lo in
 * fp32).  `workspace` is a training workspace that the forward call of the same stack has just filled and nothing has
 * touched since: stack -1 = the whole network (wn_forward_train), 0 = the confidence maps
 * (wn_confidence_maps_train), 1 = refiner `which` (wn_refine_train of that `which`; ignored for the others).  The
 * buffers, by number, with their channel counts:
 *    0  act0      16  the packed input planes: the snapped v * 255 operands of x, wb, he, gc (12 real channels)
 *    1..7 a1..a7  128, 128, 128, 64, 64, 64, 64  the saved cmg.conv1..conv7 activations (after ReLU)
 *    8  cm         3  the confidence maps
 *    9  r1        96  the refiners' conv1 activations, three refiners side by side
 *   10  r2        96  their conv2 activations
 *   11  refined    9  the three refined images
 *   12  g8        16  the seed of cmg.conv8 (3 real channels): the gate's (stack -1) or the maps' (0)
 *   13  gr3       16  the seed of the refiners' conv3 (9 real): the gate's (-1) or refiner `which`'s (1)
 *   14 + k        the output of data-gradient launch k, the gradient with respect to that convolution's input (after
 *                 the ReLU' mask of the saved activation, where there is one): k = 0..6 cmg.conv8 .. cmg.conv2
 *                 (64, 64, 64, 64, 128, 128, 128), 7 and 8 the refiners' conv3 and conv2 (96, 96), 9 cmg.conv1
 *                 and 10 the refiners' conv1 (32 each: the packed input's channels, 12 real)
 * Buffers 0..11 only read the workspace.  12 and 13 run the seed from grad_out (d(loss)/d(out), d(maps) or refiner
 * `which`'s d(out), fp32 contiguous (N,3,H,W)).  14 + k run the seed and the backward up to launch k, then stop; the
 * parameter gradients of the layers before it are written into grads (the layout of wn_backward; the stack's own
 * entries must be given).  A stack has only its own buffers (0 belongs to all).  The buffer number is checked before
 * any other argument.  dst must hold n*C*h*w floats.  An addition: no existing call changed, WN_ABI_VERSION stays.
 */
#define WN_DEBUG_BACKWARD_BUFFERS 25
int wn_debug_backward_layer(wn_handle* h, int stack, int which, int buffer, const float* grad_out,
                            float* const* grads, int n, int height, int width, float* dst, void* workspace,
                            size_t workspace_bytes, void* stream);

/* Number of kernels the library has launched on this handle since creation. */
uint64_t wn_launch_count(const wn_handle* h);

/*
 * The tensor-core forward processes a batch in passes of at most 8 Mi pixels (workspace ~1.9 KB per pixel);
 * wn_forward_chunk_images returns the number of images per pass for a batch of n (callers that pipeline
 * host<->device copies or a collective against the passes split their batch at this granularity).
 * wn_set_chunk_pixels lowers the cap (0 restores the default); it never raises the workspace need.
 */
int wn_forward_chunk_images(const wn_handle* h, int n, int height, int width);
int wn_set_chunk_pixels(wn_handle* h, long long max_pixels);

/*
 * WN_MODE_BF16_FP8 keeps the correction terms of an activation in e4m3 (|v| <= 448).  A forward pass that
 * produces a larger activation -- far outside what the reference's [0,1] images and trained weights give --
 * raises a sticky device flag, and the batch that raised it is recomputed by the WN_MODE_BF16X3 kernels
 * WITHIN THE SAME CALL (the re-run is enqueued behind every pass, its launches return at once while the flag
 * is down).  The flag reaches the host with the completion of that call; from then on the handle goes
 * straight to the WN_MODE_BF16X3 kernels until wn_pack_weights is called again.  Returns the host-side value
 * of the flag (0/1).
 */
int wn_f8_overflowed(const wn_handle* h);

/*
 * Multi-GPU exchange without a kernel and without touching the peer device's contexts (SURVEY 8e; the all-gather
 * of the output batch, waternet_b200/dist.py PeerGather).  Two things a collective library does cost this path
 * time, measured at N=2 (tools/probe_gather.py): (1) the convolution kernels are persistent and own every SM's shared
 * memory, so a collective's kernel beside them takes an SM at a kernel boundary and stalls that SM's CTA pair while
 * it waits for the peer; (2) work submitted to a context this process holds ON THE PEER GPU -- which is what a
 * framework-level cross-device copy does to order itself against the destination's streams -- makes the peer GPU
 * time-slice away from its owner process, ~0.4 ms per switch with these kernels resident.  Hence this plumbing;
 * every call acts on the calling thread's current device, none launches a kernel:
 *
 *   wn_peer_alloc   cudaMalloc + zero fill + cudaIpcGetMemHandle: a buffer other ranks may map; handle_out
 *                   receives WN_PEER_HANDLE_BYTES bytes to send to them (any transport).
 *   wn_peer_open    cudaIpcOpenMemHandle in the CURRENT device's context (peer access enabled lazily): the
 *                   returned pointer is valid for copies issued on this device's streams.  wn_peer_close unmaps.
 *   wn_memcpy_async cudaMemcpyAsync(cudaMemcpyDefault): with a wn_peer_open'ed destination it is a copy-engine
 *                   push over NVLink, ordered on `stream`, issued entirely from this device.
 *   wn_stream_write_value32 / wn_stream_wait_value32
 *                   the driver's stream memory operations (cuStreamWriteValue32 / cuStreamWaitValue32, executed by
 *                   the stream's front end): store `value` to the 4-byte aligned device address when the stream
 *                   reaches it / hold the stream until (int32)(*addr - value) >= 0.  A peer's copy engine may be
 *                   the writer of a waited-on address.
 */
#define WN_PEER_HANDLE_BYTES 64
int wn_peer_alloc(size_t bytes, void** ptr, unsigned char* handle_out);
int wn_peer_open(const unsigned char* handle, void** ptr);
int wn_peer_close(void* ptr);
int wn_peer_free(void* ptr);
int wn_memcpy_async(void* dst, const void* src, size_t bytes, void* stream);
int wn_stream_write_value32(void* stream, void* addr, uint32_t value);
int wn_stream_wait_value32(void* stream, void* addr, uint32_t value);

/*
 * The VGG19 perceptual loss of training, and its gradient, in overlapping windows (DESIGN.md 4.12):
 *
 *   L = mean over (n, c < 512, i < floor(H/16), j < floor(W/16)) of (255 * (F(out) - F(ref)))^2
 *
 * F = VGG19 features[:-1] (conv5_4 + ReLU) of (v - mean) / std with the ImageNet mean and std.  Every convolution
 * and data gradient runs in the handle's training mode (wn_set_train_mode) with fp32 accumulation: WN_MODE_BF16X3,
 * the default of a new handle, three bf16 products per product; WN_MODE_BF16 one, a_hi x w_hi, with the packed image,
 * every activation and gradient plane and the seed stored as bf16 with lo = 0 (DESIGN.md 4.14).  The loss partials
 * are float64 sums of the decoded features in both modes.  A max-pool takes the first maximum in row-major order.
 * No VGG weight gradient is computed.
 *
 * wn_vgg_pack_weights: params = weight and bias of the 16 convolutions in `features` order (fp32, contiguous OIHW
 *   and O), device pointers.  Packs the forward and the data-gradient stages; call again after the weights change.
 * wn_perceptual_loss: out and ref are (n, 3, H, W) fp32 with element strides (sN, sC, sH, sW).  *loss_dev (device
 *   fp32) receives L.  grad_out, when not NULL, receives dL/d(out) as a contiguous (n, 3, H, W) fp32 tensor; ref
 *   is a constant.  A window owns a rectangle of features (tile_h x tile_w input pixels, rounded up to multiples of
 *   16) and reads 128 pixels of context per side, clamped to the image; tile_h = tile_w = 0 makes one window per
 *   image.  Windows of one extent run in passes of at most max_pass_pixels window pixels (0 = 2 Mi, at most 8 Mi,
 *   at least one window per pass); memory is bounded by one pass, about 1.9 KB per window pixel.  Limits: n in
 *   1..65535, H and W at least 16, no window over 8 Mi pixels.  The result is deterministic and independent of the
 *   workspace contents and of max_pass_pixels.  The call copies nothing from the host.
 * wn_perceptual_loss_workspace_bytes: the workspace of that call; 0 for every argument set it rejects.
 * wn_debug_vgg_layer (test aid): layer 0..19 = the output of launch `layer` of the forward (the 16 convolutions and
 *   4 pools in features order) of x, whole images, tile 0 x 0, all n in one pass, as fp32 (n, C, H >> level,
 *   W >> level); layer 20 = the conv5_4 features of the windowed call with that tile, as (n, 512, H/16, W/16).
 *   The backward of the loss of (out = x, ref), whole images, tile 0 x 0: layer 21 = the seed (the gradient with
 *   respect to conv5_4 before its ReLU, (n, 512, H >> 4, W >> 4)); layer 22 + k = the output of the backward launch
 *   of forward launch k, the gradient with respect to that launch's input (k = 0: the 16 normalised channels, 3
 *   real).  ref and ref_strides may be NULL for layers 0..20.  The workspace is that of
 *   wn_perceptual_loss_workspace_bytes(n, H, W, tile_h, tile_w, 0).  Every layer runs in the handle's training mode.
 *
 * WN_ABI_VERSION stays 11: these four entry points are additions and no existing signature or structure changed,
 * so a library built before them still serves every client that does not call them (as with wn_backward_ragged_tiled).
 */
#define WN_VGG_NUM_PARAMS 32
int wn_vgg_pack_weights(wn_handle* h, const float* const* params, void* stream);
size_t wn_perceptual_loss_workspace_bytes(int n, int height, int width, int tile_h, int tile_w,
                                          long long max_pass_pixels);
int wn_perceptual_loss(wn_handle* h, const float* out, const int64_t out_strides[4], const float* ref,
                       const int64_t ref_strides[4], int n, int height, int width, int tile_h, int tile_w,
                       long long max_pass_pixels, float* loss_dev, float* grad_out, void* workspace,
                       size_t workspace_bytes, void* stream);
int wn_debug_vgg_layer(wn_handle* h, const float* x, const int64_t strides[4], const float* ref,
                       const int64_t ref_strides[4], int n, int height, int width, int tile_h, int tile_w, int layer,
                       float* dst, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* WATERNET_B200_H_ */
