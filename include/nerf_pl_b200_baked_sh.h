/* nerf_pl_b200 — view-dependent baked volumes: degree-2 spherical harmonics of the colour per lattice point, stored in
 * the sparse bricks of nerf_pl_b200_baked.h and ray-marched without the MLP (DESIGN.md §10k).
 *
 * Entries of libnerf_pl_b200.so with the conventions of nerf_pl_b200.h (device pointers unless the name ends in
 * `_host`, `stream` last, 0 / NERFB200_E* / cudaError_t returns, nerfb200_last_error()).
 *
 * The fit.  D = 64 unit directions on a Fibonacci sphere, d_j = (sqrt(1 - z_j^2) cos phi_j, sqrt(1 - z_j^2) sin phi_j,
 * z_j) with z_j = 1 - (2 j + 1) / 64 and phi_j = j pi (3 - sqrt 5), made in float64 and rounded to float32.  Y is the
 * 64 x 9 matrix of PlenOctrees' eval_sh basis of degree 2 at those directions,
 *   [C0, -C1 y, C1 z, -C1 x, C2_0 x y, C2_1 y z, C2_2 (2 z^2 - x^2 - y^2), C2_3 x z, C2_4 (x^2 - y^2)],
 * and P = pinv(Y) in float64, rounded to float32.  f_j(p), the network's sigmoid rgb at the raw position p with the
 * direction d_j entering as the render path's fp32 direction bias, gives the coefficients
 * c_{ch,m}(p) = sum_j P[m, j] f_{j,ch}(p), accumulated in float32 in j order.
 *
 * A point is 28 floats (7 float4): (c_r0, c_g0, c_b0, sigma), then c_{r,m}, c_{g,m}, c_{b,m} for m = 1..8; sigma is the
 * raw sigma of nerfb200_query_rgb_sigma, bit for bit.  A volume is laid out as in nerf_pl_b200_baked.h with 7 float4
 * per point: per stored brick its 9^3 points, then the int32 map; N is at most 1024.
 *
 * Bake:       nerfb200_sparse_mc_plan -> bricks_host = {active, march}; nerfb200_baked_sh_workspace_bytes(N, active,
 *             march) and nerfb200_baked_sh_bytes(N, march); nerfb200_baked_sh_bake.  Its sigma channel and its bricks
 *             are nerfb200_baked_bake's at the same arguments.
 * From grid:  nerfb200_baked_sh_from_grid_count -> bricks; nerfb200_baked_sh_bytes(N, bricks); nerfb200_baked_sh_from_grid.
 * Render:     nerfb200_baked_sh_render: one launch, no synchronisation, no workspace (it can be captured in a CUDA graph). */
#ifndef NERF_PL_B200_BAKED_SH_H_
#define NERF_PL_B200_BAKED_SH_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of a volume of `bricks` stored bricks at N: 81648 per brick plus 4 per brick of ceil(N / 8)^3 (0 for N outside
 * [2, 1024] or bricks outside [0, ceil(N / 8)^3]). */
size_t nerfb200_baked_sh_bytes(int64_t N, int64_t bricks);

/* Bytes of the bake's workspace for the plan's brick counts: the rows of one SH query, the row offsets and the SH
 * query's table (0 for a bad N or counts). */
size_t nerfb200_baked_sh_workspace_bytes(int64_t N, int64_t active, int64_t march);

/* The volume of the plan's march bricks: the 28 floats of nerfb200_query_rgb_sh at every point
 * nerfb200_rgb_sigma_grid_masked evaluates, 0 at every other point.  The arguments are nerfb200_baked_bake's, N in
 * [2, 1024], ws of nerfb200_baked_sh_workspace_bytes and volume_bytes nerfb200_baked_sh_bytes(N, march).  Reads the
 * plan's counts back, so it synchronises. */
int nerfb200_baked_sh_bake(const void* packed, int64_t N, const double ranges_host[6], const uint32_t* bits,
                           int64_t occ_N, const double occ_ranges_host[6], void* plan_ws, size_t plan_bytes,
                           const int64_t bricks_host[2], void* ws, size_t bytes, void* volume, size_t volume_bytes,
                           void* stream);

/* The bricks a volume of the dense (N, N, N, 28) grid stores: those whose 9^3 points hold a sigma (float 3) with
 * max(sigma, 0) non-zero (NaN and +inf included).  N in [2, 1024]; plan_ws of
 * nerfb200_sparse_mc_plan_workspace_bytes(N).  bricks_host receives the count; it synchronises. */
int nerfb200_baked_sh_from_grid_count(const float* grid, int64_t N, void* plan_ws, size_t plan_bytes,
                                      int64_t bricks_host[1], void* stream);

/* The volume of those bricks, each holding the grid's values at its 9^3 points (0 past the lattice).  bricks: the
 * count's; volume_bytes: nerfb200_baked_sh_bytes(N, bricks).  Reads the count back, so it synchronises. */
int nerfb200_baked_sh_from_grid(const float* grid, int64_t N, void* plan_ws, size_t plan_bytes, int64_t bricks,
                                void* volume, size_t volume_bytes, void* stream);

/* The dense (N, N, N, 28) grid of a volume: every point from its stored brick, 0 where the brick is not stored.
 * N in [2, 1024]. */
int nerfb200_baked_sh_to_dense(const void* volume, size_t volume_bytes, int64_t N, int64_t bricks, float* grid,
                               void* stream);

/* nerfb200_baked_render's rays, samples, skipping, early stop and compositing, with a sample's colour
 * clamp(sum_m cbar_{ch,m} Y_m(d / |d|), 0, 1): cbar the trilinear coefficients, d / |d| and Y in float32 once per ray.
 * A sample whose interpolated sigma gives alpha = 0 reads only the first float4 of its corners. */
int nerfb200_baked_sh_render(const void* volume, size_t volume_bytes, int64_t N, const double ranges_host[6],
                             int64_t bricks, const float* rays, int64_t n_rays, double step, int32_t white_back,
                             double early_stop, float* rgb, float* depth, float* opacity, void* stream);

/* Bytes of nerfb200_query_rgb_sh's workspace: the 64 x 128 fp32 direction biases and the projection weights. */
size_t nerfb200_query_rgb_sh_workspace_bytes(void);

/* out (n, 28), 16-byte aligned: the 28 floats of a point (above) of `packed` at the raw positions xyz (row stride
 * xyz_stride >= 3), one trunk pass per point.  ws: 16-byte aligned, of nerfb200_query_rgb_sh_workspace_bytes(). */
int nerfb200_query_rgb_sh(const float* xyz, int64_t n, int64_t xyz_stride, const void* packed, void* ws, size_t bytes,
                          float* out, void* stream);

/* The fit's float32 direction table (64 x 3) and P (9 x 64, row m). */
int nerfb200_sh_fit_host(float dirs_host[192], float proj_host[576]);

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_BAKED_SH_H_ */
