/* nerf_pl_b200 — C ABI of the H100-native volumetric-rendering hot path of kwea123/nerf_pl.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch types.  Every entry point
 * cites the reference interface it replaces (paths relative to the reference repository).
 * All pointers are DEVICE pointers unless the name ends in `_host`.  `stream` is a
 * cudaStream_t passed as void* (NULL = legacy default stream).  Functions never allocate or
 * free caller-visible memory and never throw.
 *
 * Return value: 0 = ok; negative = invalid argument (NERFB200_E*); positive = cudaError_t.
 * nerfb200_last_error() returns a thread-local, human-readable description of the last
 * non-zero return on this thread.
 */
#ifndef NERF_PL_B200_H_
#define NERF_PL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Version 3 has grown in place: nerfb200_samples_args and nerfb200_train_samples_args gained fields at their ends.
 * Zero in every new field keeps the earlier behaviour, but a caller compiled against the shorter structs is not
 * supported: build against this header. */
#define NERFB200_ABI_VERSION 3

#define NERFB200_EINVAL (-1)      /* bad argument value / null pointer            */
#define NERFB200_EUNSUPPORTED (-2) /* shape outside what the fused kernel supports */
#define NERFB200_EDEVICE (-3)     /* device is not sm_90 / kernel image missing    */

int nerfb200_abi_version(void);
const char* nerfb200_last_error(void);

/* ---- weights --------------------------------------------------------------------------
 * Replaces: the implicit use of the 12 nn.Linear parameter tensors by NeRF.forward
 * (models/nerf.py:61-81, 83-124).  `params` are the 24 fp32 device tensors of one NeRF in
 * state_dict order: xyz_encoding_{1..8}.0.{weight,bias}, xyz_encoding_final.{weight,bias},
 * dir_encoding.0.{weight,bias}, sigma.{weight,bias}, rgb.0.{weight,bias}; weights are
 * (out,in) row-major as torch stores them.  Produces the fp16/fp32 image the kernels stream
 * (nerfb200_packed_bytes() bytes, 1024-byte aligned): the forward slices, the fp32 constants and
 * the transposed 16-bit slices of the backward chain kernel. */
size_t nerfb200_packed_bytes(void);
int nerfb200_pack_weights(const float* const params[24], void* packed, void* stream);
/* Both networks of a render (coarse, fine) in ONE launch: what a training step does after every optimiser update. */
int nerfb200_pack_weights_pair(const float* const params_a[24], void* packed_a, const float* const params_b[24],
                               void* packed_b, void* stream);

/* ---- render_rays -----------------------------------------------------------------------
 * Replaces: models/rendering.py:58-244 render_rays(models, embeddings, rays, N_samples,
 * use_disp, perturb, noise_std, N_importance, chunk, white_back, test_time) including the
 * inner inference() closure (:91-172), sample_pdf (:14-55), the torchsearchsorted call
 * (:42) and the torch.sort merge (:229).  `chunk` has no equivalent (nothing is chunked).
 *
 * rays: (n_rays, 8) fp32 rows [o(3) d(3) near far], row stride `ray_stride` floats.
 * Random inputs are supplied by the caller so a seeded torch stream can be reproduced:
 *   perturb_rand (n_rays,N_samples) U[0,1)  — required iff perturb > 0     (:203)
 *   noise_coarse (n_rays,N_samples) N(0,1)  — required iff noise_std > 0   (:152)
 *   u_rand       (n_rays,N_importance) U[0,1) — required iff perturb > 0 and N_importance > 0 (:39)
 *   noise_fine   (n_rays,N_samples+N_importance) N(0,1) — iff noise_std > 0 and N_importance > 0
 * Outputs (result-dict keys, :209-221, :240-242); fp32:
 *   rgb_coarse (n,3), depth_coarse (n) — written unless test_time; may be NULL if test_time
 *   opacity_coarse (n); rgb_fine (n,3), depth_fine (n), opacity_fine (n) iff N_importance > 0
 * Optional outputs (NULL to skip): z_fine (n, N_samples+N_importance) merged sorted depths,
 *   weights_coarse (n,N_samples), weights_fine (n,N_samples+N_importance).
 * Supported shapes: N_samples in {32, 64, 128}; N_importance a multiple of 32 (0 = coarse only);
 * N_samples + N_importance <= 192 (the reference defaults 64 + 128 and the README recipes 64 + 64 included).
 * `status` is a device int32 the kernel sets non-zero on a device-side fault.  It may be NULL:
 * then a per-device internal word (mapped pinned host memory) is used; the library reads it
 * without synchronising at the START of every later call on that device and returns
 * NERFB200_EDEVICE once if an earlier kernel reported a fault (nerfb200_check_status() does the
 * same check on demand, e.g. after a stream synchronise).  The *_host entry always checks the
 * word of its own launch before returning. */
typedef struct nerfb200_render_args {
  const float* rays;
  int64_t n_rays;
  int64_t ray_stride;
  const void* packed_coarse;
  const void* packed_fine; /* NULL iff n_importance == 0 */
  int32_t n_samples;
  int32_t n_importance;
  int32_t use_disp;
  float perturb;
  float noise_std;
  int32_t white_back;
  int32_t test_time;
  const float* perturb_rand;
  const float* noise_coarse;
  const float* u_rand;
  const float* noise_fine;
  float* rgb_coarse;
  float* depth_coarse;
  float* opacity_coarse;
  float* rgb_fine;
  float* depth_fine;
  float* opacity_fine;
  float* z_fine;
  float* weights_coarse;
  float* weights_fine;
  int32_t* status;
  int32_t max_ctas; /* 0 = one CTA per SM */
  /* Optional: the (stratified) coarse depths (n, N_samples) (models/rendering.py:189-204). */
  float* z_coarse;
  /* Training mode (NULL = inference; requires test_time == 0): a device workspace of
   * nerfb200_train_workspace_bytes() bytes, initialised once with nerfb200_train_workspace_init().
   * The same fused launch then also stores, per sample, what nerfb200_render_backward needs: the
   * encoded input and the outputs of xyz_encoding_1..8 (fp16), the ReLU sign bits, the output of
   * dir_encoding, raw sigma, rgb and the depths of both passes. */
  void* train_workspace;
  /* Fused loss epilogue (replaces losses.py:9-14 MSELoss.forward and metrics.py:4-13 psnr on the
   * rendered batch; all NULL = off): target (n,3) -> loss_out[4] (device) = {mse(rgb_coarse),
   * mse(rgb_fine) or 0, their sum (= MSELoss), psnr of the finest pass}.  Needs train_workspace
   * (it holds the per-CTA partial sums; the reduction order is fixed, so the result is
   * deterministic). */
  const float* target;
  float* loss_out;
  /* Uniform random inputs drawn INSIDE the kernel (rng_in_kernel != 0): perturb_rand / u_rand may then be NULL and
   * are ignored; element (ray r, index i) of stream s (0 = perturb_rand, 1 = u_rand) is word i & 3 of
   * Philox4x32-10(counter = {r, i >> 2, s, 0}, key = {rng_seed lo, hi}) mapped to [0,1) as (x >> 8) * 2^-24 -
   * counter-based, so the numbers do not depend on the launch shape and a host replica reproduces them
   * (tests/philox.py).  The reference draws these with torch.rand from the global generator
   * (models/rendering.py:203, :39); the tensor inputs remain the way to replay a seeded torch stream.  The Gaussian
   * noise inputs (noise_std > 0) are always tensors.
   * rng_in_kernel == 2: the key is read from DEVICE memory, *rng_seed_dev (same Philox stream for the same value), so
   * that a captured CUDA graph can advance it between replays; rng_seed_dev shares the storage of rng_seed, which
   * keeps this struct's layout (ABI version 3) unchanged for existing callers. */
  union {
    uint64_t rng_seed;
    const uint64_t* rng_seed_dev;
  };
  int32_t rng_in_kernel;
} nerfb200_render_args;

int nerfb200_render_rays(const nerfb200_render_args* args, void* stream);

/* ---- training step: backward of render_rays -------------------------------------------------
 * Replaces: loss.backward() of train.py:103-117 through models/rendering.py:143-170 (quadrature)
 * and models/nerf.py:100-124 (both MLPs); no gradient flows through the fine-depth sampling
 * (models/rendering.py:225-227 .detach()) nor into the rays.
 *
 * Protocol: (1) nerfb200_render_rays(args with train_workspace set, test_time = 0);
 * (2) nerfb200_render_backward with the SAME render args (rays, random inputs, flags, packed
 * images, outputs) and either the upstream gradients of the result tensors (g_*, any may be
 * NULL = zero) or `target` (the fused MSE seed dL/drgb = 2 (rgb - target) / (3 n) * *loss_grad for
 * both passes, added to g_rgb_* if those are given).  Writes the gradients of the 24 parameter
 * tensors of each network (state_dict order and shapes, fp32; `params_*` are the live fp32
 * parameters).  grads_fine / params_fine are ignored when n_importance == 0.
 * All kernels are hand-written sm_90a code on `stream`: compositing backward, rgb head,
 * wgmma dgrad chain, wgmma split-K wgrad, partial reduction, unfolding of the packed
 * final.dir layer. */
size_t nerfb200_train_workspace_bytes(int64_t n_rays, int32_t n_samples, int32_t n_importance);
/* One-time set-up of a workspace for (n_rays, n_samples, n_importance): zeroes the padding rows,
 * counters and uploads the wgrad job table.  Synchronous with respect to `stream`. */
int nerfb200_train_workspace_init(void* workspace, size_t bytes, int64_t n_rays, int32_t n_samples,
                                  int32_t n_importance, void* stream);
typedef struct nerfb200_backward_args {
  const nerfb200_render_args* render;   /* as passed to the forward call */
  const float* const* params_coarse;    /* 24 device pointers */
  const float* const* params_fine;
  const float* g_rgb_coarse;            /* (n,3) */
  const float* g_depth_coarse;          /* (n)   */
  const float* g_opacity_coarse;        /* (n)   */
  const float* g_rgb_fine;
  const float* g_depth_fine;
  const float* g_opacity_fine;
  const float* target;                  /* (n,3) or NULL */
  const float* loss_grad;               /* device scalar or NULL (= 1) */
  float* const* grads_coarse;           /* 24 device pointers, shapes of params_coarse */
  float* const* grads_fine;
} nerfb200_backward_args;
int nerfb200_render_backward(const nerfb200_backward_args* args, void* stream);

/* ---- optimiser step ("next" row: the caller of the backward) ---------------------------------
 * Replaces: torch.optim.Adam.step() as the reference configures it (utils/__init__.py:16-18:
 * Adam(lr, eps, weight_decay), betas (0.9, 0.999), no amsgrad; train.py:77-82) for up to 64 fp32
 * tensors in one launch.  `step` is the 1-based count of this update (bias correction).  The pointers of a
 * tensor with numel 0 may be NULL (torch gives empty tensors no storage). */
int nerfb200_adam_step(int32_t n_tensors, float* const* params, const float* const* grads, float* const* exp_avg,
                       float* const* exp_avg_sq, const int64_t* numel, float lr, float beta1, float beta2, float eps,
                       float weight_decay, int64_t step, void* stream);
/* The same update with no per-step host values, so that a CUDA graph can replay it (torch.optim.Adam(capturable=True)):
 * `lr_dev` is a device fp32 scalar; `steps` holds one device pointer per tensor to its fp32 step count BEFORE this
 * update (torch's 0-dim state["step"]; the caller increments it afterwards).  Tensors at different step counts go in
 * the same launch.  The bias corrections are formed on the device in double, as nerfb200_adam_step forms them on the
 * host; the device pow is not correctly rounded, so they can differ by one fp32 ulp from the host's (m and v never
 * differ: they do not depend on the step). */
int nerfb200_adam_step_dev(int32_t n_tensors, float* const* params, const float* const* grads, float* const* exp_avg,
                           float* const* exp_avg_sq, const int64_t* numel, const float* lr_dev,
                           const float* const* steps, float beta1, float beta2, float eps, float weight_decay,
                           void* stream);

/* Same call with HOST buffers; returns with the requested outputs readable on the host (synchronises `stream`).
 * The packed weight images stay device-resident.  This is the end-to-end entry the reference's eval.py loop
 * (eval.py:117-123 `.cuda()` ... `.cpu()`) maps to.
 *   - every buffer page-locked and mapped (cudaHostAlloc / cudaHostRegister, torch pin_memory()): the kernel reads
 *     the rays and writes the results over PCIe itself; the call is launch + synchronise, no staging copies;
 *   - otherwise (pageable memory): rays and the random inputs that are non-NULL and not already device memory are
 *     staged with cudaMemcpyAsync, results are copied back the same way.
 * Random inputs may be device pointers in both cases (drawn on the device by the caller). */
int nerfb200_render_rays_host(const nerfb200_render_args* host_args, void* stream);

/* ---- NeRF.forward ------------------------------------------------------------------------
 * Replaces: models/nerf.py:83-124 NeRF.forward(x, sigma_only).  x: (n, x_stride) fp32 rows of
 * embedded xyz (63) followed, unless sigma_only, by the embedded direction (27).
 * out: (n,4) [r,g,b,sigma] or (n,1) sigma. */
int nerfb200_nerf_forward(const float* x, int64_t n, int64_t x_stride, const void* packed,
                          int32_t sigma_only, float* out, void* stream);

/* ---- training a direct NeRF.forward call -------------------------------------------------
 * Replaces: loss.backward() through models/nerf.py:83-124 NeRF.forward(x) (sigma_only = False, the
 * default architecture) when the caller renders with its own code.  No gradient with respect to x.
 * Workspace: nerfb200_nerf_train_workspace_bytes(n) bytes (0 for n <= 0), 1024-byte aligned,
 * initialised once per n with nerfb200_nerf_train_workspace_init (zeroes it and uploads the wgrad job
 * table; synchronous with respect to `stream`; a workspace smaller than the bytes for n is
 * NERFB200_EINVAL).  The forward and the backward of a call use a workspace initialised for the same
 * n; one workspace holds one call between its forward and its backward. */
size_t nerfb200_nerf_train_workspace_bytes(int64_t n);
int nerfb200_nerf_train_workspace_init(void* ws, size_t bytes, int64_t n, void* stream);
/* Replaces: models/nerf.py:83-124 NeRF.forward(x) in training.  x as for nerfb200_nerf_forward
 * (x_stride >= 90); out (n,4) [r,g,b,sigma] equals nerfb200_nerf_forward's bit for bit.  Also stores in
 * `ws`, per sample, what the backward reads: the fp16 encoded-input and direction rows the tensor core
 * consumed, the 8 hidden activations and their ReLU sign bits, the direction-layer output, sigma, rgb. */
int nerfb200_nerf_forward_train(const float* x, int64_t n, int64_t x_stride, const void* packed, void* ws, float* out,
                                void* stream);
/* Replaces: the backward of models/nerf.py:83-124 for one nerfb200_nerf_forward_train call.
 * g_out: (n,4) upstream gradient [rgb, sigma], 16-byte aligned; packed / ws: those of the forward;
 * params: the live 24 fp32 parameters (state_dict order); writes the 24 gradient tensors `grads`
 * (overwritten, not accumulated).  All kernels are sm_90a code on `stream`: gradient seed, rgb head,
 * wgmma dgrad chain, wgmma split-K wgrad (with the direction slice of dir_encoding), reduction,
 * unfolding.  A per-sample gradient outside its layer's fp16 range (status 102) or not finite (status 103)
 * is reported like the render backward's (nerfb200_check_status / the next call). */
int nerfb200_nerf_backward(const float* g_out, int64_t n, const void* packed, const float* const params[24], void* ws,
                           float* const grads[24], void* stream);

/* ---- dense sigma query ("next" row: mesh extraction) -------------------------------------
 * Replaces: extract_color_mesh.py:127-140 (embedding_xyz + embedding_dir + cat + nerf(...)[:, -1]
 * per chunk): raw positions xyz (n, xyz_stride >= 3) -> raw sigma (n); the positional encoding is
 * computed in the kernel, the direction does not enter sigma (models/nerf.py:112). */
int nerfb200_query_sigma(const float* xyz, int64_t n, int64_t xyz_stride, const void* packed, float* sigma,
                         void* stream);

/* ---- loss / metric epilogue ("next" row) -------------------------------------------------
 * Replaces: losses.py:9-14 MSELoss.forward and metrics.py:4-13 psnr on the rendered batch.
 * rgb_coarse / rgb_fine: (n_rays,3), either may be NULL; target (n_rays,3).
 * out4 (device): [mse_coarse, mse_fine, mse_coarse + mse_fine, psnr of the finest pass]. */
int nerfb200_mse_psnr(const float* rgb_coarse, const float* rgb_fine, const float* target, int64_t n_rays,
                      float* out4, void* stream);

/* ---- Embedding.forward -------------------------------------------------------------------
 * Replaces: models/nerf.py:21-38.  x: (n,3) -> out: (n, 3 + 6*n_freqs). */
int nerfb200_embed(const float* x, int64_t n, int32_t n_freqs, float* out, void* stream);

/* ---- searchsorted ------------------------------------------------------------------------
 * Replaces: torchsearchsorted/src/torchsearchsorted/searchsorted.py:20-53 and
 * src/cuda/searchsorted_cuda_kernel.cu:83-142.  a: (nrow_a, ncol_a) sorted rows,
 * v: (nrow_v, ncol_v); nrow_a == nrow_v or one of them is 1 (broadcast).
 * out: (max(nrow_a,nrow_v), ncol_v) int64.  side_right: 0 = 'left', 1 = 'right'. */
int nerfb200_searchsorted(const float* a, const float* v, int64_t* out, int64_t nrow_a,
                          int64_t nrow_v, int32_t ncol_a, int32_t ncol_v, int32_t side_right,
                          void* stream);

/* ---- sample_pdf --------------------------------------------------------------------------
 * Replaces: models/rendering.py:14-55 with the random/deterministic u supplied by the caller.
 * bins (n_rays, n_weights+1), weights (n_rays, n_weights), u (n_rays, n_u) -> out (n_rays, n_u).
 * 1 <= n_weights <= 4096. */
int nerfb200_sample_pdf(const float* bins, const float* weights, const float* u, int64_t n_rays,
                        int32_t n_weights, int32_t n_u, float* out, void* stream);

/* ---- volume rendering quadrature ---------------------------------------------------------
 * Replaces: models/rendering.py:143-170 (inside inference()).  sigmas (n,S), rgbs (n,S,3) or
 * NULL (weights_only), z_vals (n,S), dirs (n,3), noise (n,S) or NULL.  S % 32 == 0, S <= 192.
 * weights (n,S) may be NULL; rgb (n,3) / depth (n) ignored when rgbs is NULL; opacity (n). */
int nerfb200_composite(const float* sigmas, const float* rgbs, const float* z_vals,
                       const float* dirs, const float* noise, float noise_std, int32_t white_back,
                       int64_t n_rays, int32_t n_samples, float* weights, float* rgb, float* depth,
                       float* opacity, void* stream);

/* ---- ray generation ("next" row: the caller side of the path) ----------------------------
 * Replaces: datasets/ray_utils.py:5-94 get_ray_directions + get_rays (+ get_ndc_rays as
 * datasets/llff.py:236-241 applies it when ndc != 0: near plane 1.0, near/far columns 0/1) and
 * the torch.cat of datasets/blender.py:97-102.  c2w_host: 12 HOST floats, row-major (3,4).
 * rays: (H*W, 8) device rows [o(3) d(3) near far], pixel order row-major (j, i). */
int nerfb200_generate_rays(int32_t H, int32_t W, float focal, const float c2w_host[12], float near, float far,
                           int32_t ndc, float* rays, void* stream);

/* Replaces: eval.py:126-128 (clip(img,0,1)*255).astype(uint8) on the rendered image, on device. */
int nerfb200_to_uint8(const float* src, int64_t n, uint8_t* dst, void* stream);

/* ---- coloured mesh extraction ------------------------------------------------------------
 * Replaces: extract_color_mesh.py:113-284 (the dense grid, mcubes.marching_cubes, the index->world
 * transform, open3d's largest-cluster filter and the default colour-averaging loop).  Sizes that
 * depend on the data come back from a *_count call (it synchronises `stream`); the caller allocates
 * and runs the matching *_emit call with the SAME workspace.  Conventions: DESIGN.md. */

/* extract_color_mesh.py:113-140.  ranges_host: 6 HOST doubles {xmin, xmax, ymin, ymax, zmin, zmax}.
 * Positions of the flattened points [start, start + count) of np.stack(np.meshgrid(x, y, z), -1)
 * .reshape(-1, 3) with x = np.linspace(xmin, xmax, N) etc., cast to float32: point (i*N + j)*N + k is
 * (x_j, y_i, z_k). */
int nerfb200_grid_positions(int64_t N, const double ranges_host[6], int64_t start, int64_t count, float* xyz,
                            void* stream);
/* The whole grid, `chunk` points at a time (positions -> nerfb200_query_sigma -> max(sigma, 0)):
 * sigma (N, N, N), sigma[i, j, k] = max(sigma(x_j, y_i, z_k), 0).  Workspace: the positions of one chunk. */
size_t nerfb200_sigma_grid_workspace_bytes(int64_t chunk);
int nerfb200_sigma_grid(const void* packed, int64_t N, const double ranges_host[6], int64_t chunk, void* ws,
                        size_t bytes, float* sigma, void* stream);

/* extract_mesh.ipynb "Search for tight bounds": nerf_fine(cat(embedding_xyz(xyz), embedding_dir(0))) at raw
 * positions xyz (n rows of xyz_stride >= 3 floats, encoded in-kernel) with the direction (0, 0, 0):
 * rgbsigma (n, 4) [sigmoid rgb, raw sigma], 16-byte aligned.  Bit for bit NeRF.forward on the same fp16 xyz
 * encoding followed by the embedded zero direction. */
int nerfb200_query_rgb_sigma(const float* xyz, int64_t n, int64_t xyz_stride, const void* packed, float* rgbsigma,
                             void* stream);
/* The whole grid of nerfb200_grid_positions, `chunk` points at a time: rgbsigma (N, N, N, 4), raw sigma
 * (no max(sigma, 0)).  Workspace: nerfb200_sigma_grid_workspace_bytes(chunk).  2 <= N <= 1625. */
int nerfb200_rgb_sigma_grid(const void* packed, int64_t N, const double ranges_host[6], int64_t chunk, void* ws,
                            size_t bytes, float* rgbsigma, void* stream);

/* extract_mesh.ipynb "Generate .vol file for volume rendering in Unity" on a (N^3, 4) rgbsigma grid (16-byte
 * aligned, raw sigma, point (i*N + j)*N + k): a = 1 - exp(float32(-(xmax - xmin)/N) * max(sigma, 0)) in float32
 * (exp correctly rounded); the points with a > 0 in increasing order as (M, 2) uint32 pairs
 * [i, r << 24 + g << 16 + b << 8 + trunc(a * 255)], r = trunc(rgb * 255).  2 <= N <= 1625 (uint32 indices).
 * count_host = M; the emit call takes the same workspace. */
size_t nerfb200_volume_workspace_bytes(int64_t N);
int nerfb200_volume_count(const float* rgbsigma, int64_t N, double xmin, double xmax, void* ws, size_t bytes,
                          int64_t* count_host, void* stream);
int nerfb200_volume_emit(const float* rgbsigma, int64_t N, double xmin, double xmax, void* ws, size_t bytes,
                         uint32_t* packed_out, void* stream);

/* extract_color_mesh.py:144 mcubes.marching_cubes(sigma, threshold) on a C-order (n0, n1, n2) fp32 grid.
 * Inside: sigma > threshold.  counts_host[2] = {vertices, triangles}.  vertices (V, 3) fp64 in index
 * space, ordered by the lower endpoint's linear index then edge axis; triangles (T, 3) int32 ordered by
 * cell then case-table order; normals (right-hand rule) point from inside to outside.  Either output of
 * the emit call may be NULL.  At most 4e8 grid points. */
size_t nerfb200_mc_workspace_bytes(int64_t n0, int64_t n1, int64_t n2);
int nerfb200_mc_count(const float* sigma, int64_t n0, int64_t n1, int64_t n2, double threshold, void* ws, size_t bytes,
                      int64_t counts_host[2], void* stream);
int nerfb200_mc_emit(const float* sigma, int64_t n0, int64_t n1, int64_t n2, double threshold, void* ws, size_t bytes,
                     double* vertices, int32_t* triangles, void* stream);

/* extract_color_mesh.py:148-154: out (n, 3) fp32 = the reference's world vertices, with its quirks
 * (divides by N, not N - 1; column 0 takes y_range, column 1 x_range). */
int nerfb200_mesh_to_world(const double* vertices, int64_t n, int64_t N, const double ranges_host[6], float* out,
                           void* stream);

/* extract_color_mesh.py:163-171: keep the edge-connected component with the most triangles (ties: the
 * one holding the lowest-indexed triangle), drop unreferenced vertices; both lists keep their order.
 * counts_host[2] = {kept vertices, kept triangles}.  vertices (n_verts, 3) fp32. */
size_t nerfb200_mesh_cluster_workspace_bytes(int64_t n_vertices, int64_t n_triangles);
int nerfb200_mesh_cluster_count(const int32_t* triangles, int64_t n_tris, int64_t n_verts, void* ws, size_t bytes,
                                int64_t counts_host[2], void* stream);
int nerfb200_mesh_cluster_emit(const float* vertices, const int32_t* triangles, int64_t n_tris, int64_t n_verts, void* ws,
                               size_t bytes, float* vertices_out, int32_t* triangles_out, void* stream);

/* extract_color_mesh.py:240-243 cv2.remap(image, x, y, INTER_LINEAR) (constant 0 border) of a (H, W, 3)
 * uint8 image at n points xy (n, 2) fp32 -> out (n, 3) uint8. */
int nerfb200_remap_bilinear(const uint8_t* image, int32_t H, int32_t W, const float* xy, int64_t n, uint8_t* out,
                            void* stream);
/* extract_color_mesh.py:220-262 for one view: w2c_host = np.linalg.inv(c2w4)[:3] (12 HOST doubles),
 * origin_host = float32(c2w[:, 3]).  Writes the sampled colours (n, 3) uint8, depth (n) fp64 and the
 * occlusion rays (n, 8) [o, (v - o)/|v - o|, near, float32(depth)] for nerfb200_render_rays. */
int nerfb200_color_project(const float* vertices, int64_t n, const double w2c_host[12], const float origin_host[3],
                           float focal, int32_t W, int32_t H, const uint8_t* image, float near, uint8_t* colors,
                           double* depth, float* rays, void* stream);
/* extract_color_mesh.py:269-277: sum4 (n, 4) fp64 [colour sums, weight sum] += the view's weighted
 * colour, w = 0.1/depth + (nan_to_num(opacity) < occ_threshold).  Zero sum4 before the first view. */
int nerfb200_color_accumulate(const uint8_t* colors, const double* depth, const float* opacity, int64_t n,
                              float occ_threshold, double* sum4, void* stream);
/* extract_color_mesh.py:283-284: colors (n, 3) = uint8(sum / wsum), truncated. */
int nerfb200_color_finalize(const double* sum4, int64_t n, uint8_t* colors, void* stream);

/* The vertex-normal colouring method.  Replaces: extract_color_mesh.py:187-203 and 280-284
 * (--use_vertex_normal): open3d's mesh.compute_vertex_normals(), the rays built from the normals, and the uint8
 * colours.  The render itself is nerfb200_render_rays (both networks, test_time = 1, perturb 0, noise 0) on these
 * rays, and the colours are nerfb200_to_uint8 of its rgb_fine, which equals (rgb * 255.0).astype(uint8) for every
 * rgb in [0, 1].  Definitions and provenance: DESIGN.md section 9, "Vertex-normal colours". */

/* :189 mesh.compute_vertex_normals() (open3d TriangleMesh::ComputeVertexNormals, normalized, on a mesh
 * without normals): normals (n_verts, 3) fp64 of fp32 vertices (n_verts, 3) and int32 triangles
 * (n_tris, 3).  Triangle normal (v1 - v0) x (v2 - v0) in fp64; each vertex sums the normals of its
 * triangles in increasing triangle index; then s = (x^2 + y^2) + z^2, each component divided by sqrt(s)
 * when s > 0, and (0, 0, 1) when x is NaN.  Bit for bit, whatever the launch shape.  The workspace is
 * the caller's (0 bytes: unsupported size).  Synchronises `stream`: an index outside [0, n_verts)
 * returns NERFB200_EINVAL, and the normals are then undefined. */
size_t nerfb200_vertex_normals_workspace_bytes(int64_t n_verts, int64_t n_tris);
int nerfb200_vertex_normals(const float* vertices, int64_t n_verts, const int32_t* triangles, int64_t n_tris, void* ws,
                            size_t bytes, double* normals, void* stream);

/* :190-193 and the torch.cat of :200: rays (n, 8) fp32 [v - (d * near) * near_t, d, near, far] with
 * d = float32(normal), each operation in fp32 as torch does it on the CPU; near, far and near_t are the
 * fp32 roundings of the host values (dataset.bounds.min(), .max(), args.near_t). */
int nerfb200_normal_rays(const float* vertices, const double* normals, int64_t n, float near, float far, float near_t,
                         float* rays, void* stream);

/* ---- empty-space skipping ----------------------------------------------------------------
 * An occupancy bit field is built once from a dense sigma grid of the trained network; before a render the rays
 * are classified against it and the live ones compacted (in order) into an ordinary (n_live, 8) ray tensor for
 * nerfb200_render_rays; afterwards the compacted results are scattered back over the value a ray through vacuum
 * renders.  The render kernel itself is untouched.  The reference has no counterpart.
 * What culling guarantees and what it does not: DESIGN.md section 10, "Empty-space skipping".
 *
 * AXIS ORDER.  The sigma grid is nerfb200_sigma_grid's, sigma[i, j, k] = sigma(x_j, y_i, z_k) (the first index is
 * y).  The occupancy grid undoes that: cell (cx, cy, cz), each in [0, N - 1), spans
 * [x_cx, x_cx+1] x [y_cy, y_cy+1] x [z_cz, z_cz+1] with x_j = linspace(x_range, N)[j] etc.  Its flat index is
 * c = (cz * (N-1) + cy) * (N-1) + cx (x fastest) and it is bit c % 32 of word c / 32; ceil((N-1)^3 / 32) words,
 * the bits past the last cell 0. */

/* sigma (N, N, N) fp32 -> bits.  A cell is occupied iff the largest sigma of its 8 corner points is
 * > sigma_threshold (a NaN corner is not above); the occupied set is then dilated by `dilate` cells in Chebyshev
 * distance (dilate >= 0) and packed.  2 <= N <= 1625.  The workspace (two bytes per cell) is the
 * caller's; 0 bytes: unsupported N. */
size_t nerfb200_occupancy_workspace_bytes(int64_t N);
int nerfb200_occupancy_pack(const float* sigma, int64_t N, double sigma_threshold, int32_t dilate, void* ws,
                            size_t bytes, uint32_t* bits, void* stream);
/* *count (one DEVICE int64) = the number of occupied cells of an N-point grid's bit field. */
int nerfb200_occupancy_popcount(const uint32_t* bits, int64_t N, int64_t* count, void* stream);

/* Ray classification.  rays (n_rays, 8) fp32 [o, d, near, far], contiguous and 16-byte aligned; ranges_host =
 * {xmin, xmax, ymin, ymax, zmin, zmax} of the grid (6 HOST doubles, min != max).  flag[i] = 1 iff the segment
 * o + t d, t in [near, far], crosses an occupied cell: the segment is clipped to the grid's box and its cells
 * are walked by an exact 3-D DDA in double.  Space outside the box is empty.  A ray with a non-finite value or
 * far <= near is live.  cull_count writes flag (n_rays) and the number of live rays to *n_live_host, and
 * synchronises `stream`; cull_emit, called next with the same workspace, writes live_idx (n_live) int64,
 * strictly increasing, and live_rays (n_live, 8) = rays[live_idx].  Either may be called with n_rays = 0. */
size_t nerfb200_cull_workspace_bytes(int64_t n_rays);
int nerfb200_cull_count(const float* rays, int64_t n_rays, const uint32_t* bits, int64_t N,
                        const double ranges_host[6], void* ws, size_t bytes, uint8_t* flag, int64_t* n_live_host,
                        void* stream);
int nerfb200_cull_emit(const float* rays, int64_t n_rays, const uint8_t* flag, void* ws, size_t bytes,
                       int64_t* live_idx, float* live_rays, void* stream);

/* One launch writes the full-size results of a culled render.  src_host / dst_host: 6 HOST entries, the device
 * pointers of rgb_coarse (., 3), depth_coarse, opacity_coarse, rgb_fine (., 3), depth_fine, opacity_fine: src of
 * n_live rows, dst of n_rays rows; an entry is NULL in both or in neither.  dst[live_idx[r]] = src[r]; every
 * other ray gets what a ray through vacuum renders: opacity 0, depth 0, rgb 1 if white_back else 0.  live_idx
 * must be strictly increasing and inside [0, n_rays). */
int nerfb200_scatter_results(const float* const src_host[6], float* const dst_host[6], const int64_t* live_idx,
                             int64_t n_live, int64_t n_rays, int32_t white_back, void* stream);

/* ---- diagnostics -------------------------------------------------------------------------
 * Number of kernels this library has launched on the calling process so far (all entry
 * points).  bench.py reports the delta as `gpu_launches`. */
int64_t nerfb200_launch_count(void);
/* Returns NERFB200_EDEVICE (and clears the flag) if a kernel launched by an earlier call on the
 * current device reported a device-side fault through the internal status word; 0 otherwise.
 * Does not synchronise: call it after synchronising the stream to cover the latest launch. */
int nerfb200_check_status(void);
/* Device properties the launcher uses: SM count of the current device (0 if none). */
int nerfb200_sm_count(void);


/* ==== image metrics of the reference's eval and validation loop, on the device ====================
 * Definitions and their provenance: DESIGN.md "Image metrics". */

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

/* ==== training batches generated on the device from the dataset's views ===========================
 * Definitions and their exactness argument: DESIGN.md "Training batches from the views". */

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

/* ==== rendering with empty samples skipped (inference) ============================================
 * Definition and guarantees: DESIGN.md "Skipping empty samples". */

/* One render of n_rays rays in which a sample is evaluated only when its point
 * o + d z (rounded as the render kernel rounds it) lies in the closed box of an occupied cell of the occupancy grid
 * (bits, N, ranges_host: as nerfb200_cull_count).  A skipped sample has sigma = 0.  A ray with a non-finite value or
 * far <= near, and a pass whose interval lengths delta |d| are not all finite, is evaluated at every sample.
 * Compositing, the inverse-CDF resampling (u = linspace(0, 1, N_importance), or the sorted random u with
 * perturb > 0) and the merge are the render kernel's; the random inputs (fields at the end) are optional.
 *   rays: (n_rays, 8) fp32, 16-byte aligned.  live_flag: nullable (n_rays) uint8; a ray whose flag is 0 has every
 *   sample skipped.  Results: as nerfb200_render_args (rgb / depth_coarse only with test_time = 0, the fine ones
 *   with n_importance > 0); z_fine (n, S_f), weights_coarse (n, S_c), weights_fine (n, S_f) optional.
 *   samples_coarse (n, S_c, 4) / samples_fine (n, S_f, 4), optional, 16-byte aligned: rgb and sigma of every sample,
 *   0 where skipped (rgb 0 in the coarse pass with test_time).  mask_coarse / mask_fine, optional (n, 6) uint32:
 *   bit b of word w set iff sample 32 w + b is evaluated.  live_samples_host[2] receives the evaluated coarse and
 *   fine sample counts.
 *   Appended under version 3 (perturb .. rng_ray_offset; zero-filled, the render is as before): the random inputs of
 * nerfb200_train_samples_args, checked by the same rules, so that a render perturbs the depths and adds noise as the
 * training step does.  perturb_rand / noise_coarse / u_rand / noise_fine are rows of this call's rays.  With
 * rng_in_kernel, ray r of the call draws as ray rng_ray_offset + r, so a render in chunks draws what one call over
 * all rays draws; 0 <= rng_ray_offset and rng_ray_offset + n_rays <= 2^32.
 *   Appended under version 3 (early_stop, cut_coarse; zero-filled, the render is as before): early ray termination
 * of a coarse-only render (DESIGN.md §10f).  With early_stop = eps > 0 the coarse samples are evaluated in rounds of
 * one mask word; a ray is cut after the first word k whose float64 transmittance T_k falls below eps, and the
 * samples of its later words are treated as empty (cleared in mask_coarse, not counted in live_samples_host).
 * Every weight up to the end of the cut word, and every output of a ray never cut, is bit for bit the render's
 * without termination.  cut_coarse, optional (n_rays) int32: the word each ray was cut after, or -1.  Needs
 * n_importance = 0 (NERFB200_EUNSUPPORTED) and perturb = noise_std = 0; eps in [0, 1].  With n_samples = 32 there
 * is one word, nothing can be dropped, and the render takes the path without termination (cut_coarse is then -1).
 * The workspace is nerfb200_samples_workspace_bytes(n_rays, n_samples, 0); the stream is synchronised once per word.
 *   Appended under version 3 (levels; zero-filled, one level as before): the occupancy grid's number of cascade
 * levels, 1..8 (see "cascaded occupancy grids" below); bits then holds levels bit fields.
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
  float perturb;
  float noise_std;
  const float* perturb_rand;
  const float* noise_coarse;
  const float* u_rand;
  const float* noise_fine;
  uint64_t rng_seed;
  int32_t rng_in_kernel;
  int64_t rng_ray_offset;
  float early_stop;
  int32_t* cut_coarse;
  int32_t levels;
} nerfb200_samples_args;

/* Workspace bytes of nerfb200_render_samples for n_rays rays (0 for an unsupported shape). */
size_t nerfb200_samples_workspace_bytes(int64_t n_rays, int32_t n_samples, int32_t n_importance);

int nerfb200_render_samples(const nerfb200_samples_args* args, void* ws, size_t bytes, int64_t* live_samples_host,
                            void* stream);

/* ==== the training step with empty samples skipped ===============================================
 * Definition and guarantees: DESIGN.md "Training with empty samples skipped". */

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
 * samples, rows in ray-major, depth-index order (live_samples_host rows per pass).
 *   target and loss_out are both given (the fused loss) or both null: the forward then has no loss epilogue and the
 * backward no MSE seed (loss_grad is ignored).
 *   Appended under version 3 (g_rgb_coarse .. g_opacity_fine; zero-filled, the step is as before): the upstream
 * gradients of the six results, each nullable, read by both backward entries.  Per pass the seed is
 * composite_bwd_kernel's: g = g_rgb + [target] 2 (rgb - target) / (3 n_rays) * loss_grad, g_depth, and
 * g_opacity - [white_back] sum g.  A pass with none of them (and no target) gets exact zero gradients.
 *   Appended under version 3 (levels; zero-filled, one level as before): as nerfb200_samples_args. */
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
  const float* g_rgb_coarse;
  const float* g_depth_coarse;
  const float* g_opacity_coarse;
  const float* g_rgb_fine;
  const float* g_depth_fine;
  const float* g_opacity_fine;
  int32_t levels;
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

/* ==== the density grid: an occupancy grid kept current during training ============================
 * Definition and guarantees: DESIGN.md "Keeping the grid current during training".
 *
 * The grid has the occupancy grid's conventions (nerfb200_occupancy_pack): N points per axis over ranges_host
 * {xmin, xmax, ymin, ymax, zmin, zmax} (each finite with min != max; a reversed range is allowed), M = N - 1 cells
 * per axis, cell c = (cz * M + cy) * M + cx, bit c % 32 of word c / 32, the bits past the last cell 0.  Its state is
 * density (M^3 float32, in cell order), bits (ceil(M^3 / 32) uint32 words) and key (one int64 in device memory).
 * An update from the packed network f with key s:
 *   1. u_a = the render kernel's in-kernel uniform (rng_in_kernel) of key s, ray c, element a, stream 2; a = 0, 1, 2;
 *   2. p_a = float32(lo_a + (double(cell_a) + double(u_a)) * ((hi_a - lo_a) / M)), every double operation rounded
 *      on its own;
 *   3. sigma_c = nerfb200_query_sigma(f, p);
 *   4. density_c = fmaxf(float32(decay * density_c), sigma_c > 0 ? sigma_c : 0) (a NaN sigma counts as 0);
 *   5. cell c is occupied iff double(density_c) > sigma_threshold; the set is dilated by `dilate` cells (Chebyshev)
 *      and packed into bits;
 *   6. key = key + 1, so that update k of a grid seeded with s uses s + k. */

/* Workspace bytes of an update of an N-point grid, `chunk` cells at a time (0 for N outside [2, 1625] or
 * chunk < 1).  A chunk larger than the grid is taken as the grid. */
size_t nerfb200_density_workspace_bytes(int64_t N, int64_t chunk);

/* Steps 1-2 for cells [start, start + count) with the key *key_dev: xyz (count, 3) fp32. */
int nerfb200_density_points(int64_t N, const double ranges_host[6], const int64_t* key_dev, int64_t start,
                            int64_t count, float* xyz, void* stream);

/* One whole update (steps 1-6) from the packed image of nerfb200_pack_weights, `chunk` cells at a time.
 * sigma_threshold must not be NaN, decay must be in [0, 1], dilate >= 0; ws: nerfb200_density_workspace_bytes(N,
 * chunk) bytes.  Every launch has a size fixed by (N, chunk): nothing is synchronised, allocated or read back, so a
 * CUDA graph can capture the call; a replay reads the key where the previous one left it. */
int nerfb200_density_update(const void* packed, int64_t N, const double ranges_host[6], double sigma_threshold,
                            float decay, int32_t dilate, int64_t chunk, int64_t* key_dev, float* density,
                            uint32_t* bits, void* ws, size_t bytes, void* stream);

/* ==== mesh and Unity-volume grids through an occupancy grid =======================================
 * Definition and guarantees: DESIGN.md "Grids through an occupancy grid".
 *
 * The mesh grid is nerfb200_sigma_grid's: N points per axis over ranges_host, flat point p = (i * N + j) * N + k at
 * the fp32 position (x_j, y_i, z_k) of nerfb200_grid_positions.  The occupancy grid is nerfb200_cull_count's: bits
 * (one bit per cell, cell (cz * M + cy) * M + cx, M = occ_N - 1) over occ_ranges_host (each finite with
 * min != max; a reversed range is allowed).  The two grids' N and ranges are independent.  A lattice point is
 * *evaluated* iff its position lies in the closed box of an occupied cell (the rule of nerfb200_render_samples: a
 * point on a shared face, edge or corner checks every cell that touches it; outside the box or NaN it is empty).
 *
 * Per chunk of `chunk` lattice points: classify, scan, compact the evaluated positions, query them with
 * nerfb200_query_sigma / nerfb200_query_rgb_sigma, scatter.  Each chunk reads its evaluated count back once, so the
 * calls synchronise.  *evaluated_host receives the number of evaluated points. */

/* Workspace bytes of either entry at `chunk` points per chunk (0 for chunk < 1). */
size_t nerfb200_masked_grid_workspace_bytes(int64_t chunk);

/* sigma_out (N^3) fp32: an evaluated point gets nerfb200_sigma_grid's value bit for bit, max(sigma, 0); every
 * other point gets +0.0.  N >= 2, occ_N in [2, 1625], chunk >= 1; ws: nerfb200_masked_grid_workspace_bytes(chunk). */
int nerfb200_sigma_grid_masked(const void* packed, int64_t N, const double ranges_host[6], const uint32_t* bits,
                               int64_t occ_N, const double occ_ranges_host[6], int64_t chunk, void* ws, size_t bytes,
                               float* sigma_out, int64_t* evaluated_host, void* stream);

/* rgbsigma_out (N^3, 4) fp32, 16-byte aligned: an evaluated point gets nerfb200_rgb_sigma_grid's four channels bit
 * for bit; every other point gets (0, 0, 0, 0).  N in [2, 1625]; otherwise as nerfb200_sigma_grid_masked. */
int nerfb200_rgb_sigma_grid_masked(const void* packed, int64_t N, const double ranges_host[6], const uint32_t* bits,
                                   int64_t occ_N, const double occ_ranges_host[6], int64_t chunk, void* ws,
                                   size_t bytes, float* rgbsigma_out, int64_t* evaluated_host, void* stream);

/* ==== cascaded occupancy grids ======================================================================
 * Definition and guarantees: DESIGN.md §10h.
 *
 * An occupancy grid of `levels` = L levels (1 <= L <= 8) over ranges_host.  Level 0's box is ranges_host as given;
 * for k >= 1, with c_a = 0.5 (lo_a + hi_a) and h_a = 0.5 (hi_a - lo_a) in double, level k's range on axis a is
 * c_a -+ 2^k h_a.  Every level has N points and M = N - 1 cells per axis with the one-level cell order, and level
 * k's ceil(M^3 / 32) words follow level k - 1's in bits (density: M^3 floats per level, the same way).  A point
 * belongs to the smallest level whose closed box holds it, compared in that level's grid coordinates
 * (x - lo) * M / (hi - lo); inside it the one-level rule applies; outside the last level's box, or NaN, it is empty.
 * A cell of level k >= 1 with every index a in [ceil(M / 4), floor(3 M / 4)) lies inside level k - 1's box: it is
 * *inner*, never reached by that rule, never evaluated, and always density 0 and bit 0.
 *
 * The entries above that take an occupancy or density grid's size as an int64_t (N of nerfb200_occupancy_workspace_bytes,
 * _pack, _popcount, nerfb200_cull_count and the density grid entries, occ_N of the masked grids) read a cascade from
 * it: NERFB200_GRID_N(N, L) keeps N in the low 32 bits and L - 1 above them, so every one-level value means what it
 * meant.  The argument structs take `levels` instead (their N is the point count).  Then:
 *   - nerfb200_occupancy_pack reads sigma (L, N, N, N), level k's sigma grid over level k's box; each level is marked
 *     with its inner cells empty, dilated within the level and packed with its inner cells cleared;
 *   - nerfb200_occupancy_popcount counts the occupied cells of every level;
 *   - nerfb200_cull_count walks each level's box in turn, so a culled ray has no point the rule finds occupied;
 *   - the density grid update runs steps 1-5 level by level on the level's non-inner cells in cell order (inner cells
 *     keep density 0 and bit 0), drawing cell c of level k with element 3 k + a (level 0: the one-level points),
 *     dilates within each level and advances the key once; nerfb200_density_points numbers the cells it evaluates
 *     level 0's first, then each further level's non-inner cells, in cell order;
 *   - the workspaces are those of one level (reused level by level). */
#define NERFB200_GRID_N(N, levels) ((int64_t)(N) + ((int64_t)(levels) - 1) * ((int64_t)1 << 32))

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_H_ */
