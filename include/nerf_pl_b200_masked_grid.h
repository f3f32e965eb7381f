/* nerf_pl_b200 — mesh and Unity-volume grids through an occupancy grid.
 *
 * Companion of nerf_pl_b200.h: the same library, return codes, nerfb200_last_error() and conventions (DEVICE
 * pointers unless the name ends in `_host`, `stream` a cudaStream_t as void*, no allocation).  Definition and
 * guarantees: DESIGN.md "Grids through an occupancy grid".
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
#ifndef NERF_PL_B200_MASKED_GRID_H_
#define NERF_PL_B200_MASKED_GRID_H_

#include "nerf_pl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

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

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_MASKED_GRID_H_ */
