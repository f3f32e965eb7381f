/* nerf_pl_b200 — baked volumes: rgb and sigma stored in sparse bricks, ray-marched without the MLP (DESIGN.md §10j).
 *
 * Entries of libnerf_pl_b200.so with the conventions of nerf_pl_b200.h (device pointers unless the name ends in
 * `_host`, `stream` last, 0 / NERFB200_E* / cudaError_t returns, nerfb200_last_error()).  extract_mesh.ipynb bakes
 * [sigmoid rgb, raw sigma] on an N^3 lattice with the direction 0 and the Unity project ray-marches it; these entries
 * keep that lattice on the device, store only its useful bricks and render views from it.
 *
 * The lattice is rgb_sigma_grid's: dense[i, j, k] is the value at (x_j, y_i, z_k), x = linspace(xmin, xmax, N) in
 * float32, likewise y and z.  It is split into bricks of 8^3 points, and the bricks are those of the sparse marching
 * cubes' plan (nerf_pl_b200_sparse_mc.h): a volume stores the plan's march bricks (the active bricks and their
 * neighbours at -1 along any subset of the axes).  A volume is one buffer of nerfb200_baked_bytes(N, bricks): per
 * stored brick its 9^3 points (the +1 apron copied from the neighbours) as float4 [r, g, b, sigma], then an int32 map
 * of the ceil(N / 8)^3 bricks holding each one's slot or -1.
 *
 * Bake:       nerfb200_sparse_mc_plan -> bricks_host = {active, march}; nerfb200_baked_workspace_bytes(N, active, march)
 *             and nerfb200_baked_bytes(N, march); nerfb200_baked_bake.  nerfb200_baked_to_dense of the result equals
 *             nerfb200_rgb_sigma_grid_masked at the same N, box and occupancy grid, bit for bit.
 * From grid:  nerfb200_baked_from_grid_count -> bricks; nerfb200_baked_bytes(N, bricks); nerfb200_baked_from_grid.
 * Render:     nerfb200_baked_render: one launch, no synchronisation, no workspace (it can be captured in a CUDA graph). */
#ifndef NERF_PL_B200_BAKED_H_
#define NERF_PL_B200_BAKED_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of a volume of `bricks` stored bricks at N: 11664 per brick plus 4 per brick of ceil(N / 8)^3 (0 for N outside
 * [2, 2048] or bricks outside [0, ceil(N / 8)^3]). */
size_t nerfb200_baked_bytes(int64_t N, int64_t bricks);

/* Bytes of the bake's workspace for the plan's brick counts: the rows of one rgb + sigma query and the row offsets
 * (0 for a bad N or counts). */
size_t nerfb200_baked_workspace_bytes(int64_t N, int64_t active, int64_t march);

/* The volume of the plan's march bricks: [sigmoid rgb, raw sigma] of `packed` with the direction 0 at every point
 * nerfb200_rgb_sigma_grid_masked evaluates (nerfb200_query_rgb_sigma on compacted rows), (0, 0, 0, 0) at every other
 * point.  N, ranges_host and the occupancy grid (bits, occ_N with NERFB200_GRID_N's levels, occ_ranges_host) are the
 * plan's, plan_ws the workspace it filled and bricks_host its {active, march}.  volume_bytes must be
 * nerfb200_baked_bytes(N, march).  Reads the plan's counts back, so it synchronises. */
int nerfb200_baked_bake(const void* packed, int64_t N, const double ranges_host[6], const uint32_t* bits, int64_t occ_N,
                        const double occ_ranges_host[6], void* plan_ws, size_t plan_bytes, const int64_t bricks_host[2],
                        void* ws, size_t bytes, void* volume, size_t volume_bytes, void* stream);

/* The bricks a volume of the dense (N, N, N, 4) grid `rgbsigma` stores: those whose 9^3 points hold a sigma with
 * max(sigma, 0) non-zero (NaN and +inf included).  N in [2, 1625]; plan_ws of nerfb200_sparse_mc_plan_workspace_bytes(N)
 * keeps their list for nerfb200_baked_from_grid.  bricks_host receives the count; it synchronises. */
int nerfb200_baked_from_grid_count(const float* rgbsigma, int64_t N, void* plan_ws, size_t plan_bytes,
                                   int64_t bricks_host[1], void* stream);

/* The volume of those bricks, each holding the grid's values at its 9^3 points (0 past the lattice).  bricks: the
 * count's; volume_bytes: nerfb200_baked_bytes(N, bricks).  Reads the count back, so it synchronises. */
int nerfb200_baked_from_grid(const float* rgbsigma, int64_t N, void* plan_ws, size_t plan_bytes, int64_t bricks,
                             void* volume, size_t volume_bytes, void* stream);

/* The dense (N, N, N, 4) grid of a volume: every point from its stored brick, (0, 0, 0, 0) where the brick is not
 * stored.  N in [2, 1625]. */
int nerfb200_baked_to_dense(const void* volume, size_t volume_bytes, int64_t N, int64_t bricks, float* rgbsigma,
                            void* stream);

/* rgb (n, 3), depth (n) and opacity (n) of the rays (n, 8) [o, d, near, far] through the volume over the box
 * ranges_host (finite, min != max, in float32): samples t_k = near + (k + 1/2) s / |d| for k < floor((far - near) |d| / s)
 * (none for far <= near or a non-finite value), trilinear rgb and max(sigma, 0) in index coordinates, 0 outside the box
 * and outside the stored bricks, alpha = 1 - exp(-sigma s), composited in float32 in sample order (DESIGN.md §10j).
 * step: s > 0 and finite; white_back: 0 or 1; early_stop in [0, 1]: a ray ends after the first sample with T below it. */
int nerfb200_baked_render(const void* volume, size_t volume_bytes, int64_t N, const double ranges_host[6], int64_t bricks,
                          const float* rays, int64_t n_rays, double step, int32_t white_back, double early_stop,
                          float* rgb, float* depth, float* opacity, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_BAKED_H_ */
