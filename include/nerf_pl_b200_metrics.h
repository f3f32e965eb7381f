/* nerf_pl_b200 — image metrics of the reference's eval and validation loop, on the device.
 *
 * Companion of nerf_pl_b200.h: the same library, return codes, nerfb200_last_error() and conventions (DEVICE
 * pointers unless the name ends in `_host`, `stream` a cudaStream_t as void*, no allocation).  Definitions and their
 * provenance: DESIGN.md "Image metrics".
 */
#ifndef NERF_PL_B200_METRICS_H_
#define NERF_PL_B200_METRICS_H_

#include "nerf_pl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- SSIM -----------------------------------------------------------------------------------
 * Replaces: metrics.py:15-20 ssim(image_pred, image_gt, reduction) = 1 - 2 * kornia.losses.ssim(pred, gt, 3,
 * reduction), kornia 0.2.0's published definition: a 3 x 3 window (outer product of the normalised size-3 Gaussian,
 * sigma 1.5), zero padding 1, per channel; mu, sigma^2 and sigma12 as filter(x*y) - mu_x*mu_y; C1 = 0.01^2,
 * C2 = 0.03^2; loss = clamp(1 - ssim_map, 0, 1) / 2.  Every pixel's moments and ssim_map are computed in double.
 *
 * pred, gt: (b, c, h, w) fp32 with element strides pred_strides_host / gt_strides_host (4 HOST int64 each, >= 0),
 * b, c, h, w >= 1.  reduction:
 *   NERFB200_SSIM_MEAN / NERFB200_SSIM_SUM: out is ONE device float, 1 - 2 * (mean / sum of the loss); the sum is
 *     taken in double in a fixed order, so the result does not depend on the grid.  Needs the workspace; does not
 *     synchronise.
 *   NERFB200_SSIM_NONE: out is the contiguous (b, c, h, w) map 1 - 2 * loss; ws may be NULL. */
#define NERFB200_SSIM_MEAN 0
#define NERFB200_SSIM_SUM 1
#define NERFB200_SSIM_NONE 2
size_t nerfb200_ssim_workspace_bytes(int64_t b, int64_t c, int64_t h, int64_t w);
int nerfb200_ssim(const float* pred, const int64_t pred_strides_host[4], const float* gt,
                  const int64_t gt_strides_host[4], int64_t b, int64_t c, int64_t h, int64_t w, int32_t reduction,
                  void* ws, size_t bytes, float* out, void* stream);

/* ---- depth visualisation ----------------------------------------------------------------------
 * Replaces: utils/visualization.py:6-18 visualize_depth(depth) with the default cmap=cv2.COLORMAP_JET, bit for
 * bit: nan_to_num (NaN -> 0, +-inf -> +-FLT_MAX), y = (x - min) / (max - min + 1e-8f) in fp32, uint8(255 * y) by
 * truncation, OpenCV's JET table (csrc/jet_lut.h), u8 / 255.  depth: (h, w) fp32 with element strides stride_h,
 * stride_w (>= 0); out: contiguous (3, h, w) fp32 in cv2's channel order (channel 0 = blue), as the reference
 * returns it.  A map holding both +inf and -inf is outside the contract.  Two launches, no synchronisation. */
size_t nerfb200_visualize_depth_workspace_bytes(int64_t h, int64_t w);
int nerfb200_visualize_depth(const float* depth, int64_t h, int64_t w, int64_t stride_h, int64_t stride_w, void* ws,
                             size_t bytes, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_METRICS_H_ */
