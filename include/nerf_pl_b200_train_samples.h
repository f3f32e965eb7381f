/* nerf_pl_b200 — the training step with empty samples skipped.
 *
 * Companion of nerf_pl_b200.h: the same library, return codes, nerfb200_last_error() and conventions (DEVICE
 * pointers unless the name ends in `_host`, `stream` a cudaStream_t as void*, no allocation).  Definition and
 * guarantees: DESIGN.md "Training with empty samples skipped".
 */
#ifndef NERF_PL_B200_TRAIN_SAMPLES_H_
#define NERF_PL_B200_TRAIN_SAMPLES_H_

#include "nerf_pl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One training step's render + loss over n_rays rays in which a sample is evaluated only when its point lies in an
 * occupied cell of the occupancy grid (bits, N, ranges: as nerfb200_render_samples).  The coarse depths are the
 * render kernel's stratified depths with the perturb jitter; perturb_rand / u_rand (or rng_in_kernel and rng_seed,
 * with the meaning they have in nerfb200_render_args) and noise_coarse / noise_fine are the render kernel's random
 * inputs.  An evaluated sample gets the network's sigma + noise * noise_std, a skipped one sigma = 0 (no noise), so
 * its weight is 0 and it gets no gradient.  A ray with a non-finite value or far <= near, and a pass whose interval
 * lengths delta |d| are not all finite, is evaluated at every sample.  Compositing, white_back, the inverse-CDF
 * resampling with the render kernel's sorted random u (linspace with perturb = 0) and the merge run on those weights.
 *   rays (n_rays, 8) fp32 and target (n_rays, 3), 16-byte aligned.  Results: the six outputs of nerfb200_render_args
 * (the fine ones with n_importance > 0), loss_out[4] as its fused loss epilogue (mse_coarse, mse_fine, their sum,
 * psnr of the finest pass), reduced in an order that does not depend on the launch.  Optional (null = not written):
 * z_coarse (n, S_c), z_fine (n, S_f), weights_coarse / weights_fine, samples_coarse / samples_fine (n, S, 4: raw
 * network rgb and sigma, 0 where skipped; 16-byte aligned), mask_coarse / mask_fine (n, 6) uint32 (bit b of word w:
 * sample 32 w + b evaluated).  The backward fills, when given: dsigma_coarse / dsigma_fine (rows) and dprergb_coarse /
 * dprergb_fine (rows, 3), the per-row d loss / d sigma and d loss / d (rgb before the sigmoid) of the evaluated
 * samples, rows in ray-major, depth-index order (live_samples_host rows per pass). */
typedef struct nerfb200_train_samples_args {
  const float* rays;
  int64_t n_rays;
  const void* packed_coarse;
  const void* packed_fine;
  int32_t n_samples;
  int32_t n_importance;
  int32_t use_disp;
  int32_t white_back;
  float perturb;
  float noise_std;
  const float* perturb_rand;
  const float* noise_coarse;
  const float* u_rand;
  const float* noise_fine;
  uint64_t rng_seed;
  int32_t rng_in_kernel;
  const uint32_t* bits;
  int64_t N;
  double ranges[6];
  const float* target;
  float* rgb_coarse;
  float* depth_coarse;
  float* opacity_coarse;
  float* rgb_fine;
  float* depth_fine;
  float* opacity_fine;
  float* loss_out;
  float* z_coarse;
  float* z_fine;
  float* weights_coarse;
  float* weights_fine;
  float* samples_coarse;
  float* samples_fine;
  uint32_t* mask_coarse;
  uint32_t* mask_fine;
  float* dsigma_coarse;
  float* dsigma_fine;
  float* dprergb_coarse;
  float* dprergb_fine;
} nerfb200_train_samples_args;

/* Workspace bytes for n_rays rays: sized for every sample evaluated, so one workspace serves every step of a batch
 * shape (0 for an unsupported shape).  Zero it once before its first use; it is never re-zeroed. */
size_t nerfb200_train_samples_workspace_bytes(int64_t n_rays, int32_t n_samples, int32_t n_importance);

/* The forward.  n_samples in {32, 64, 128}, n_importance a multiple of 32, their sum <= 192, 1 <= n_rays <= 2^22.
 * ws: 1024-byte aligned, held until the backward.  live_samples_host[2] receives the evaluated coarse and fine
 * sample counts.  Synchronises the stream once, to read them back when the last pass's count is known; no launch is
 * sized from them. */
int nerfb200_train_samples_forward(const nerfb200_train_samples_args* args, void* ws, size_t bytes,
                                   int64_t* live_samples_host, void* stream);

/* The same forward without the read-back: live_samples_dev[2] (device) receives the counts.  No launch is sized from
 * a count on the host, and nothing is synchronised or read from host memory, so a CUDA graph can capture it. */
int nerfb200_train_samples_forward_dev(const nerfb200_train_samples_args* args, void* ws, size_t bytes,
                                       int64_t* live_samples_dev, void* stream);

/* The backward of the forward that used `args`, `ws` and returned live_samples_host: the gradients of the 24
 * parameters of each network (the tables of nerfb200_backward_args) for the seed loss_grad (a device scalar dL/dloss
 * of loss_out[2], or null for 1).  A network with no evaluated sample launches nothing and its gradients are not
 * written (they are 0).  Non-finite per-sample gradients are reported as device status 103. */
int nerfb200_train_samples_backward(const nerfb200_train_samples_args* args, void* ws, size_t bytes,
                                    const int64_t* live_samples_host, const float* loss_grad,
                                    const float* const params_coarse[24], const float* const params_fine[24],
                                    float* const grads_coarse[24], float* const grads_fine[24], void* stream);

/* The backward of either forward with the counts the workspace holds (no host counts): capturable as the forward_dev
 * entry.  Every network's gradients are written, exact zeros for one with no evaluated sample, so both tables must be
 * complete.  The optional per-row outputs receive the first live_samples rows of each pass. */
int nerfb200_train_samples_backward_dev(const nerfb200_train_samples_args* args, void* ws, size_t bytes,
                                        const float* loss_grad, const float* const params_coarse[24],
                                        const float* const params_fine[24], float* const grads_coarse[24],
                                        float* const grads_fine[24], void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_TRAIN_SAMPLES_H_ */
