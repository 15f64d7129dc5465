/*
 * waternet_b200 metrics: SSIM and PSNR statistics on the library's kernels (DESIGN.md 4.16).
 *
 * An optional part of the C ABI of libwaternet_b200.so, kept out of include/waternet_b200.h: nothing of the
 * enhancement and training path uses it, and a client of that path needs none of it.  The handle, the error codes
 * and wn_last_error() are those of waternet_b200.h.  These entry points were added without changing any existing
 * signature or structure, so WN_ABI_VERSION stays 11.
 */
#ifndef WATERNET_B200_METRICS_H_
#define WATERNET_B200_METRICS_H_

#include "waternet_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * SSIM and PSNR statistics of n image pairs of their own sizes in one call (DESIGN.md 4.16): the quantities
 * waternet_b200/metrics.py (ssim, psnr) and training.batch_quality are made of, per image.
 *
 * images_host is a HOST array of n entries: out and ref of one image, device fp32 contiguous (3, height, width), and
 * its group.  The images of one group share SSIM's data range, max(max out - min out, max ref - min ref) over all
 * of the group's images, hence c1 = (0.01 range)^2 and c2 = (0.03 range)^2: a tensor batch is one group, each image
 * of a list its own.  SSIM: an 11 x 11 Gaussian window (sigma 1.5) over reflect-padded planes (padding 5), the
 * border of 5 pixels left out when both sides exceed 10.  Both sides must be at least 6 (reflect padding of 5).
 *
 * stats (device, 8-byte aligned) receives WN_QUALITY_STATS float64 values per image i at stats[i * 7]:
 *   [0] the sum of the SSIM of every counted pixel of the three planes, [1] their count, [2] the sum of the squared
 *   differences over all 3 H W elements, [3] min out, [4] max out, [5] min ref, [6] max ref.
 * Two launches; no floating-point atomics: the statistics of image i depend on its own pixels and its group's data
 * range only (bit for bit), whatever else the call holds and whatever the workspace held.  A constant pair (range 0)
 * gives an SSIM sum of NaN.  Limits: n in 1..65535, groups in 0..n-1, each image at most 0x7fffffff / 3 pixels per
 * plane.  The call copies its table to the device from pageable host memory once, so it cannot be captured in a
 * CUDA graph.  wn_quality_workspace_bytes returns 0 for sizes the call rejects; the workspace holds the table and
 * about 40 bytes per 1024 pixels of partial sums.
 */
typedef struct {
  const float* out; /* device, fp32 contiguous (3, height, width) */
  const float* ref; /* device, same size */
  int height, width;
  int group;        /* 0 .. n-1 */
} wn_quality_image;
#define WN_QUALITY_STATS 7
size_t wn_quality_workspace_bytes(const int* heights_host, const int* widths_host, int n);
int wn_quality(wn_handle* h, const wn_quality_image* images_host, int n, double* stats, void* workspace,
               size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* WATERNET_B200_METRICS_H_ */
