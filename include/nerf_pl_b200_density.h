/* nerf_pl_b200 — the density grid: an occupancy grid kept current during training.
 *
 * Companion of nerf_pl_b200.h: the same library, return codes, nerfb200_last_error() and conventions (DEVICE
 * pointers unless the name ends in `_host`, `stream` a cudaStream_t as void*, no allocation).  Definition and
 * guarantees: DESIGN.md "Keeping the grid current during training".
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
#ifndef NERF_PL_B200_DENSITY_H_
#define NERF_PL_B200_DENSITY_H_

#include "nerf_pl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

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

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_DENSITY_H_ */
