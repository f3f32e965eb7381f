// Mesh and Unity-volume grids through an occupancy grid (DESIGN.md "Grids through an occupancy grid").  A lattice
// point of the dense mesh grid is evaluated iff its fp32 position (mesh_grid_positions_kernel's) passes
// point_occupied, the rule of skip="samples"; every other point gets the output 0 and never reaches the MLP.
//
// Per chunk of lattice indices [start, start + count):  classify (zeros for empty points, evaluated points per tile)
// -> exclusive scan of the tile counts -> emit (evaluated positions and indices, increasing index) -> the existing
// point query on the compacted rows -> scatter.  Classify and emit work on fixed tiles of kMaskTile points, so the
// compacted order and every output byte are independent of the launch shape.
#pragma once
#include <cub/cub.cuh>

#include "mesh_kernels.cuh"
#include "sample_skip_kernels.cuh"

namespace nerfb200 {

constexpr int kMaskThreads = 256;
constexpr int kMaskTile = 16 * kMaskThreads;

struct MaskedGridParams {
  double lo[3], hi[3];         // the mesh grid's x, y, z ranges
  long long N, start, count;   // N points per axis; the chunk [start, start + count) of flat indices
  SkipGrid occ;
  int channels;                // 1: max(sigma, 0); 4: [rgb, raw sigma]
  float* out;                  // (N^3, channels)
  unsigned long long* tcnt;    // (tiles + 1) evaluated points per tile of the chunk
  unsigned long long* tofs;    // (tiles + 1) exclusive scan of tcnt
  float* xyz;                  // (evaluated, 3) compacted positions
  long long* idx;              // (evaluated) their flat indices
  float* vals;                 // (evaluated, channels) the query's outputs
};

// Point t of the chunk: its flat index q, position x (np.meshgrid 'xy' order, as mesh_grid_positions_kernel) and
// whether it is evaluated.
__device__ __forceinline__ bool masked_point(const MaskedGridParams& p, long long t, long long& q, float x[3]) {
  q = p.start + t;
  const long long NN = p.N * p.N;
  const long long i = q / NN, j = (q / p.N) % p.N, k = q % p.N;
  x[0] = mesh_linspace(p.lo[0], p.hi[0], p.N, j);
  x[1] = mesh_linspace(p.lo[1], p.hi[1], p.N, i);
  x[2] = mesh_linspace(p.lo[2], p.hi[2], p.N, k);
  return point_occupied(p.occ, x);
}

__global__ void __launch_bounds__(kMaskThreads) masked_grid_classify_kernel(MaskedGridParams p) {
  using Reduce = cub::BlockReduce<int, kMaskThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  const long long tiles = (p.count + kMaskTile - 1) / kMaskTile;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    int n = 0;
    for (int r = 0; r < kMaskTile / kMaskThreads; ++r) {
      const long long t = tile * kMaskTile + r * kMaskThreads + threadIdx.x;
      if (t >= p.count) break;
      long long q;
      float x[3];
      if (masked_point(p, t, q, x)) {
        ++n;
      } else if (p.channels == 4) {
        reinterpret_cast<float4*>(p.out)[q] = make_float4(0.f, 0.f, 0.f, 0.f);
      } else {
        p.out[q] = 0.f;
      }
    }
    const int total = Reduce(tmp).Sum(n);
    if (threadIdx.x == 0) p.tcnt[tile] = static_cast<unsigned long long>(total);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kMaskThreads) masked_grid_emit_kernel(MaskedGridParams p) {
  using Scan = cub::BlockScan<int, kMaskThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const long long tiles = (p.count + kMaskTile - 1) / kMaskTile;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    unsigned long long base = p.tofs[tile];
    for (int r = 0; r < kMaskTile / kMaskThreads; ++r) {
      const long long t = tile * kMaskTile + r * kMaskThreads + threadIdx.x;
      long long q = 0;
      float x[3] = {0.f, 0.f, 0.f};
      int keep = 0;
      if (t < p.count) keep = masked_point(p, t, q, x) ? 1 : 0;
      int rank, total;
      Scan(tmp).ExclusiveSum(keep, rank, total);
      if (keep) {
        const unsigned long long row = base + static_cast<unsigned long long>(rank);
        p.xyz[row * 3 + 0] = x[0];
        p.xyz[row * 3 + 1] = x[1];
        p.xyz[row * 3 + 2] = x[2];
        p.idx[row] = q;
      }
      base += static_cast<unsigned long long>(total);
      __syncthreads();
    }
  }
}

// Row r of the query to its lattice point: max(sigma, 0) as mesh_relu_kernel leaves it (NaN and -0.0 pass through),
// or the four channels as they are.
__global__ void masked_grid_scatter_kernel(MaskedGridParams p, long long rows) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
    const long long q = p.idx[r];
    if (p.channels == 4) {
      reinterpret_cast<float4*>(p.out)[q] = reinterpret_cast<const float4*>(p.vals)[r];
    } else {
      const float v = p.vals[r];
      p.out[q] = v < 0.f ? 0.f : v;
    }
  }
}

}  // namespace nerfb200
