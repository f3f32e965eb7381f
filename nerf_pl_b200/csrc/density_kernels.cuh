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
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "render_kernel.cuh"

namespace nerfb200 {

struct DensityBox {
  double lo[3], hi[3];    // ranges_host: a reversed range (lo > hi) walks its axis downwards
  long long M;            // cells per axis
};

// Steps 1-2 for cells [start, start + count): xyz[i] is the point of cell start + i.  The key is read from device
// memory, so a captured graph sees each update's key.  c < 1624^3 < 2^32: the cell index is the Philox ray counter.
__global__ void density_points_kernel(DensityBox b, const long long* __restrict__ key, long long start, long long count,
                                      float* __restrict__ xyz) {
  const unsigned long long s = static_cast<unsigned long long>(*key);
  const double m = static_cast<double>(b.M);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    const long long c = start + i;
    const long long cell[3] = {c % b.M, (c / b.M) % b.M, c / (b.M * b.M)};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double u = static_cast<double>(philox_uniform(s, static_cast<uint32_t>(c), static_cast<uint32_t>(a), 2u));
      const double step = __ddiv_rn(__dsub_rn(b.hi[a], b.lo[a]), m);
      const double v = __dadd_rn(b.lo[a], __dmul_rn(__dadd_rn(static_cast<double>(cell[a]), u), step));
      xyz[i * 3 + a] = __double2float_rn(v);
    }
  }
}

// Steps 4-5 (before the dilation) for cells [start, start + count), whose sigma is sigma[0, count): the decayed
// maximum and the occupancy byte.  With key_bump (the last chunk of an update) one thread does step 6; every point
// launch of the update is ahead of it in the stream.
__global__ void density_decay_kernel(const float* __restrict__ sigma, long long start, long long count, float decay,
                                     double thr, float* __restrict__ density, uint8_t* __restrict__ occ,
                                     long long* __restrict__ key_bump) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    const long long c = start + i;
    const float s = sigma[i];
    const float d = fmaxf(__fmul_rn(decay, density[c]), s > 0.f ? s : 0.f);
    density[c] = d;
    occ[c] = static_cast<double>(d) > thr;
  }
  if (key_bump && blockIdx.x == 0 && threadIdx.x == 0) *key_bump += 1;
}

}  // namespace nerfb200
