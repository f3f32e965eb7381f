/* nerf_pl_b200 — rendering with empty samples skipped (inference).
 *
 * Companion of nerf_pl_b200.h: the same library, return codes, nerfb200_last_error() and conventions (DEVICE
 * pointers unless the name ends in `_host`, `stream` a cudaStream_t as void*, no allocation).  Definition and
 * guarantees: DESIGN.md "Skipping empty samples".
 */
#ifndef NERF_PL_B200_SAMPLES_H_
#define NERF_PL_B200_SAMPLES_H_

#include "nerf_pl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One render of n_rays rays with perturb = noise_std = 0 in which a sample is evaluated only when its point
 * o + d z (rounded as the render kernel rounds it) lies in the closed box of an occupied cell of the occupancy grid
 * (bits, N, ranges_host: as nerfb200_cull_count).  A skipped sample has sigma = 0.  A ray with a non-finite value or
 * far <= near, and a pass whose interval lengths delta |d| are not all finite, is evaluated at every sample.
 * Compositing, the inverse-CDF resampling (u = linspace(0, 1, N_importance)) and the merge are the render kernel's.
 *   rays: (n_rays, 8) fp32, 16-byte aligned.  live_flag: nullable (n_rays) uint8; a ray whose flag is 0 has every
 *   sample skipped.  Results: as nerfb200_render_args (rgb / depth_coarse only with test_time = 0, the fine ones
 *   with n_importance > 0); z_fine (n, S_f), weights_coarse (n, S_c), weights_fine (n, S_f) optional.
 *   samples_coarse (n, S_c, 4) / samples_fine (n, S_f, 4), optional, 16-byte aligned: rgb and sigma of every sample,
 *   0 where skipped (rgb 0 in the coarse pass with test_time).  mask_coarse / mask_fine, optional (n, 6) uint32:
 *   bit b of word w set iff sample 32 w + b is evaluated.  live_samples_host[2] receives the evaluated coarse and
 *   fine sample counts.
 * n_samples in {32, 64, 128}, n_importance a multiple of 32, their sum <= 192, 0 <= n_rays <= 2^22.  Synchronises
 * the stream twice (each sample count sizes the launches after it); no MLP launch for a pass without an evaluated
 * sample. */
typedef struct nerfb200_samples_args {
  const float* rays;
  int64_t n_rays;
  const uint8_t* live_flag;
  const void* packed_coarse;
  const void* packed_fine;
  int32_t n_samples;
  int32_t n_importance;
  int32_t use_disp;
  int32_t white_back;
  int32_t test_time;
  const uint32_t* bits;
  int64_t N;
  double ranges[6];
  float* rgb_coarse;
  float* depth_coarse;
  float* opacity_coarse;
  float* rgb_fine;
  float* depth_fine;
  float* opacity_fine;
  float* z_fine;
  float* weights_coarse;
  float* weights_fine;
  float* samples_coarse;
  float* samples_fine;
  uint32_t* mask_coarse;
  uint32_t* mask_fine;
} nerfb200_samples_args;

/* Workspace bytes of nerfb200_render_samples for n_rays rays (0 for an unsupported shape). */
size_t nerfb200_samples_workspace_bytes(int64_t n_rays, int32_t n_samples, int32_t n_importance);

int nerfb200_render_samples(const nerfb200_samples_args* args, void* ws, size_t bytes, int64_t* live_samples_host,
                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_SAMPLES_H_ */
