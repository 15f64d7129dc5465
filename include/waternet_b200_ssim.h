/*
 * waternet_b200 SSIM loss: SSIM and its gradient with respect to the enhanced image on the library's kernels
 * (DESIGN.md 4.17).
 *
 * An optional part of the C ABI of libwaternet_b200.so, kept out of include/waternet_b200.h and
 * include/waternet_b200_metrics.h: nothing of the enhancement and training path uses it.  The handle, the error
 * codes and wn_last_error() are those of waternet_b200.h, the statistics those of wn_quality.  These entry points
 * were added without changing any existing signature or structure, so WN_ABI_VERSION stays 11.
 */
#ifndef WATERNET_B200_SSIM_H_
#define WATERNET_B200_SSIM_H_

#include "waternet_b200_metrics.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * The wn_quality statistics of n image pairs and, per image i, grad_i = d/d(out_i) of sum_j scale_j SSIM_j, where
 * SSIM_j is image j's SSIM: the mean over its counted pixels of the three planes (wn_quality's [0] / [1]).
 *
 * images_host is a HOST array of n entries: out, ref and grad of one image, device fp32 contiguous (3, height,
 * width), its group and its scale.  Groups, sizes, SSIM's window, padding and crop, the limits and stats are those
 * of wn_quality (waternet_b200_metrics.h); the stats are the same bits as wn_quality's on the same images.  The
 * gradient includes the data-range term: c1 and c2 depend on the group's range max(max out - min out, max ref -
 * min ref), whose gradient goes to the elements of out equal to the group's max or min, split evenly over ties, all
 * of it when out's range is the larger, half when the two are equal, none when ref's is larger.  ref is a constant.
 *
 * grad must not overlap any out, ref or other grad; scale must be finite.  Every element of every grad is written.
 * Four launches; no floating-point atomics: image i's statistics and gradient depend on its own pixels and its
 * group only (bit for bit), whatever else the call holds and whatever the workspace held.  A constant pair gives
 * NaN.  wn_ssim_grad_workspace_bytes returns 0 for sizes the call rejects; the workspace holds the table and about
 * 140 bytes per 1024 pixels of partial sums, nothing per pixel.
 */
typedef struct {
  const float* out; /* device, fp32 contiguous (3, height, width) */
  const float* ref; /* device, same size */
  float* grad;      /* device, same size: receives d/d(out) */
  int height, width;
  int group;        /* 0 .. n-1 */
  double scale;     /* the weight of this image's SSIM in the differentiated sum */
} wn_ssim_grad_image;
size_t wn_ssim_grad_workspace_bytes(const int* heights_host, const int* widths_host, int n);
int wn_ssim_grad(wn_handle* h, const wn_ssim_grad_image* images_host, int n, double* stats, void* workspace,
                 size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* WATERNET_B200_SSIM_H_ */
