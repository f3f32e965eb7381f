/* nerf_pl_b200 — sparse marching cubes through an occupancy grid (DESIGN.md §10i).
 *
 * Entries of libnerf_pl_b200.so with the conventions of nerf_pl_b200.h (device pointers unless the name ends in
 * `_host`, `stream` last, 0 / NERFB200_E* / cudaError_t returns, nerfb200_last_error()).  nerf_pl_b200.h keeps the
 * entries of the dense pipeline; this header adds the sparse route of extract_color_mesh.py's marching cubes
 * (mcubes.marching_cubes at --N_grid up to 2048).
 *
 * Replaces: marching_cubes(sigma_grid_masked(N, ranges, occupancy grid), threshold) — nerfb200_sigma_grid_masked
 * then nerfb200_mc_count / nerfb200_mc_emit — without the N^3 sigma grid.  The vertices and triangles are the same,
 * bit for bit and in the same order (vertices by the flat index q of the edge's lower endpoint, then axis; triangles
 * by flat cell index, then case-table order), for every threshold, NaN and +-inf included.  N in [2, 2048] (the dense
 * entries stop at 4e8 points).  The mesh grid and the occupancy grid (bits, occ_N with NERFB200_GRID_N's levels,
 * occ_ranges_host) are those of nerfb200_sigma_grid_masked.
 *
 * The lattice is split into bricks of 8^3 points.  A brick is *active* if it holds an evaluated point, a *march*
 * brick if it or a neighbour at +1 along any subset of the axes is active.  Three steps, each sized by the last:
 *   1. plan:  active and march bricks from the occupancy bits -> bricks_host = {active, march};
 *   2. count: sigma at the evaluated points (nerfb200_query_sigma on compacted rows, stored per active brick), then
 *             the vertices and triangles per march brick -> counts_host = {V, T};
 *   3. emit:  their keys, radix-sorted, resolved to (V, 3) float64 index-space vertices and (T, 3) int32 triangles.
 * plan, count and emit take the same N (and count the same grids) and the plan workspace the plan filled; count and
 * emit take the workspace count filled.  Every call reads its counts back, so it synchronises. */
#ifndef NERF_PL_B200_SPARSE_MC_H_
#define NERF_PL_B200_SPARSE_MC_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of the plan workspace at N points per axis: the brick map and lists, 21 B per brick of ceil(N / 8)^3
 * (0 for N outside [2, 2048]). */
size_t nerfb200_sparse_mc_plan_workspace_bytes(int64_t N);

/* Candidate bricks from the occupancy bits (never missing a brick with an evaluated point), the exact rule of
 * nerfb200_sigma_grid_masked on every point of a candidate, and the active and march bricks.  bricks_host receives
 * {active, march}. */
int nerfb200_sparse_mc_plan(int64_t N, const double ranges_host[6], const uint32_t* bits, int64_t occ_N,
                            const double occ_ranges_host[6], void* plan_ws, size_t plan_bytes, int64_t bricks_host[2],
                            void* stream);

/* Bytes of the count / emit workspace for the plan's brick counts: 2 KiB per active brick (its sigma values), 20 B
 * per march brick and the rows of one point query (0 for a bad N or counts). */
size_t nerfb200_sparse_mc_workspace_bytes(int64_t N, int64_t active, int64_t march);

/* sigma at every evaluated point of the active bricks, max(sigma, 0) exactly as nerfb200_sigma_grid_masked writes it,
 * then the vertex and triangle counts at `threshold`: counts_host = {V, T}.  bricks_host: the plan's.  V or T of
 * 2^31 or more returns NERFB200_EUNSUPPORTED. */
int nerfb200_sparse_mc_count(const void* packed, int64_t N, const double ranges_host[6], const uint32_t* bits,
                             int64_t occ_N, const double occ_ranges_host[6], double threshold, void* plan_ws,
                             size_t plan_bytes, const int64_t bricks_host[2], void* ws, size_t bytes,
                             int64_t counts_host[2], void* stream);

/* Bytes of the emit workspace for V vertices and T triangles: their sort keys, twice, and the sort's scratch (0 for
 * counts outside [0, 2^31)). */
size_t nerfb200_sparse_mc_emit_workspace_bytes(int64_t n_vertices, int64_t n_triangles);

/* vertices (V, 3) float64 and triangles (T, 3) int32 at `threshold` (count's): mcubes.marching_cubes' output, as
 * nerfb200_mc_emit writes it for the dense masked grid.  counts_host: count's {V, T}. */
int nerfb200_sparse_mc_emit(int64_t N, double threshold, void* plan_ws, size_t plan_bytes,
                            const int64_t bricks_host[2], void* ws, size_t bytes, const int64_t counts_host[2],
                            void* emit_ws, size_t emit_bytes, double* vertices, int32_t* triangles, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_SPARSE_MC_H_ */
