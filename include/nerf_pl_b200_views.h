/* nerf_pl_b200 — training batches generated on the device from the dataset's views.
 *
 * Companion of nerf_pl_b200.h: the same library, return codes, nerfb200_last_error() and conventions (DEVICE
 * pointers unless the name ends in `_host`, `stream` a cudaStream_t as void*, no allocation).  Definitions and their
 * exactness argument: DESIGN.md "Training batches from the views".
 */
#ifndef NERF_PL_B200_VIEWS_H_
#define NERF_PL_B200_VIEWS_H_

#include "nerf_pl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- one training batch from the views --------------------------------------------------------
 * Replaces: the all_rays / all_rgbs buffers of datasets/blender.py:47-69 and datasets/llff.py:221-253 and the
 * DataLoader's gather from them.  Row k of the batch is pixel ids[k] of the reference's concatenation order
 * (view-major, pixels row-major): p = (v * H + j) * W + i, 0 <= p < V * H * W (an id outside gives a NaN row).
 *   images: (V, H, W, C) uint8, C = 3 (RGB) or 4 (RGBA);  c2w: (V, 3, 4) fp32 poses, 16-byte aligned.
 *   rays:   (n, 8) fp32 [o(3) d(3) near far], 16-byte aligned: nerfb200_generate_rays' row of pixel (j, i) of view v
 *           (ndc != 0: the forward-facing NDC warp of llff.py:236-241, near/far columns 0/1).
 *   rgbs:   (n, 3) fp32: u8 / 255 (T.ToTensor()); with C = 4, rgb * a + (1 - a) (blender.py:58).
 * V, H, W >= 1, focal > 0, n >= 0.  One launch; reads nothing on the host, so it can be captured in a graph. */
int nerfb200_view_batch(const uint8_t* images, int64_t V, int32_t H, int32_t W, int32_t C, const float* c2w,
                        float focal, float near, float far, int32_t ndc, const int64_t* ids, int64_t n, float* rays,
                        float* rgbs, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_VIEWS_H_ */
