/* nerf_pl_b200 — C ABI, empty-space skipping at render time.
 *
 * An occupancy bit field is built once from a dense sigma grid of the trained network; before a render the rays
 * are classified against it and the live ones compacted (in order) into an ordinary (n_live, 8) ray tensor for
 * nerfb200_render_rays; afterwards the compacted results are scattered back over the value a ray through vacuum
 * renders.  The render kernel itself is untouched.  The reference has no counterpart.
 * Conventions of nerf_pl_b200.h (which includes this header): device pointers unless `_host`, `stream` last,
 * 0 = ok, negative = invalid argument.  Adding these entries changed no struct: NERFB200_ABI_VERSION stays 3.
 * What culling guarantees and what it does not: DESIGN.md section 10, "Empty-space skipping".
 *
 * AXIS ORDER.  The sigma grid is nerfb200_sigma_grid's, sigma[i, j, k] = sigma(x_j, y_i, z_k) (the first index is
 * y).  The occupancy grid undoes that: cell (cx, cy, cz), each in [0, N - 1), spans
 * [x_cx, x_cx+1] x [y_cy, y_cy+1] x [z_cz, z_cz+1] with x_j = linspace(x_range, N)[j] etc.  Its flat index is
 * c = (cz * (N-1) + cy) * (N-1) + cx (x fastest) and it is bit c % 32 of word c / 32; ceil((N-1)^3 / 32) words,
 * the bits past the last cell 0.
 */
#ifndef NERF_PL_B200_OCCUPANCY_H_
#define NERF_PL_B200_OCCUPANCY_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

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

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_OCCUPANCY_H_ */
