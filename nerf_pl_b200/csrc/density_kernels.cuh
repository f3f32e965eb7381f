// The density grid: an occupancy grid kept current during training.  Each cell holds a float density that decays
// and is refreshed from one jittered point in the cell per update (the scheme of Instant-NGP-style occupancy grids);
// the bit field it feeds is the OccupancyGrid one (occupancy_kernels.cuh), so every skipping path reads it as is.
// Rule and guarantees: DESIGN.md §10d.  An update from a network f with key s:
//   1. u_a = philox_uniform(s, ray = c, i = a, stream = 2), a = 0, 1, 2 (streams 0 and 1 are the render kernel's);
//   2. p_a = float32(lo_a + (double(cell_a) + double(u_a)) * ((hi_a - lo_a) / M)), each double operation rounded on
//      its own (no contraction), so a float64 replica reproduces the point bit for bit;
//   3. sigma_c = nerfb200_query_sigma(f, p) (the fused sigma-only MLP);
//   4. density_c <- fmaxf(float32(decay * density_c), sigma_c > 0 ? sigma_c : 0) (a NaN sigma counts as 0);
//   5. occupied iff double(density_c) > threshold, dilated by occ_dilate_axis_kernel and packed by occ_pack_kernel;
//   6. key <- key + 1 on the device.
// Cells are c = (cz * M + cy) * M + cx with M = N - 1 cells per axis, x fastest, as in occupancy_kernels.cuh.
//
// A cascade (DESIGN.md §10h) runs steps 1-5 per level k on level k's box, for its non-inner cells only, with
// element 3 k + a in step 1, so level 0 draws the points of a one-level grid.  Inner cells keep density 0 and bit 0.
// The launches see a level's non-inner cells by rank, in cell order (noninner_cell).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "render_kernel.cuh"
#include "occupancy_kernels.cuh"

namespace nerfb200 {

struct DensityBox {
  double lo[3], hi[3];    // the level's box, from ranges_host: a reversed range (lo > hi) walks its axis downwards
  long long M;            // cells per axis
  int level;
  long long ia, ib;       // the level's inner cells [ia, ib)^3; ia = ib = 0 at level 0
};

// The cell of rank r among the non-inner cells of a level, in cell order: z slabs below, through and above the
// hole, and inside a slab through the hole the rows below, through and above it.  The identity without a hole.
__device__ __forceinline__ long long noninner_cell(const DensityBox& b, long long r) {
  const long long M = b.M, n = b.ib - b.ia, F = M * M, H = F - n * n, R = M - n;
  long long cz;
  if (r < b.ia * F) return r;
  r -= b.ia * F;
  if (r >= n * H) return (b.ib * F) + (r - n * H);
  cz = b.ia + r / H;
  r %= H;
  long long cy, cx;
  if (r < b.ia * M) {
    cy = r / M; cx = r % M;
  } else if ((r -= b.ia * M) < n * R) {
    cy = b.ia + r / R; cx = r % R;
    if (cx >= b.ia) cx += n;
  } else {
    r -= n * R;
    cy = b.ib + r / M; cx = r % M;
  }
  return (cz * M + cy) * M + cx;
}

// Steps 1-2 for the level's non-inner cells of rank [start, start + count): xyz[i] is the point of rank start + i.
// The key is read from device memory, so a captured graph sees each update's key.  c < 1624^3 < 2^32: the cell
// index is the Philox ray counter.
__global__ void density_points_kernel(DensityBox b, const long long* __restrict__ key, long long start, long long count,
                                      float* __restrict__ xyz) {
  const unsigned long long s = static_cast<unsigned long long>(*key);
  const double m = static_cast<double>(b.M);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    const long long c = noninner_cell(b, start + i);
    const long long cell[3] = {c % b.M, (c / b.M) % b.M, c / (b.M * b.M)};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double u = static_cast<double>(
          philox_uniform(s, static_cast<uint32_t>(c), static_cast<uint32_t>(3 * b.level + a), 2u));
      const double step = __ddiv_rn(__dsub_rn(b.hi[a], b.lo[a]), m);
      const double v = __dadd_rn(b.lo[a], __dmul_rn(__dadd_rn(static_cast<double>(cell[a]), u), step));
      xyz[i * 3 + a] = __double2float_rn(v);
    }
  }
}

// Steps 4-5 (before the dilation) for the level's non-inner cells of rank [start, start + count), whose sigma is
// sigma[0, count): the decayed maximum and the occupancy byte.  density and occ are the level's.  With key_bump (the
// last chunk of an update) one thread does step 6; every point launch of the update is ahead of it in the stream.
__global__ void density_decay_kernel(const float* __restrict__ sigma, DensityBox b, long long start, long long count,
                                     float decay, double thr, float* __restrict__ density, uint8_t* __restrict__ occ,
                                     long long* __restrict__ key_bump) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    const long long c = noninner_cell(b, start + i);
    const float s = sigma[i];
    const float d = fmaxf(__fmul_rn(decay, density[c]), s > 0.f ? s : 0.f);
    density[c] = d;
    occ[c] = static_cast<double>(d) > thr;
  }
  if (key_bump && blockIdx.x == 0 && threadIdx.x == 0) *key_bump += 1;
}

}  // namespace nerfb200
