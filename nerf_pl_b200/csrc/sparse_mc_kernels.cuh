// Marching cubes through an occupancy grid without the dense sigma grid (DESIGN.md §10i).  The N^3 lattice is split
// into bricks of 8^3 points, brick (I, J, K) holding points (8 I + a, 8 J + b, 8 K + c).
//
//   plan:   candidate bricks from the occupancy bits (a superset of the bricks with an evaluated point), the exact
//           masked rule (masked_point) on every point of a candidate, the active bricks (some point evaluated) and
//           their brick map, and the march bricks (an active brick or one of its lower neighbours);
//   sigma:  the evaluated points of the active bricks, compacted, through the point query; max(sigma, 0) is stored
//           per active brick, every other point reads +0.0;
//   march:  per march brick, the vertices (key 3 q + axis) and triangles (key 5 c + t) of the dense kernels' rules,
//           counted, emitted, radix-sorted, then resolved to positions and vertex ids.
//
// A point the grid does not let through is +0.0 in the dense masked route too, and a cell whose corners are all such
// points is uniform for any threshold, so marching the march bricks finds every vertex and triangle of the dense
// route; sorting the unique keys puts them in its order.
#pragma once
#include <cstdint>
#include <cub/cub.cuh>

#include "masked_grid_kernels.cuh"
#include "mesh_kernels.cuh"

namespace nerfb200 {

constexpr int kBrick = 8;
constexpr int kBrickPoints = kBrick * kBrick * kBrick;
constexpr int kBrickHalo = kBrick + 1;
// Above this many bit-field words per level, a brick is a candidate without looking (the exact rule decides).
constexpr long long kBrickProbeWords = 512;

struct SparseMcParams {
  MaskedGridParams m;             // the mesh grid (lo, hi, N; start 0) and the occupancy grid: masked_point
  long long nb;                   // bricks per axis, ceil(N / 8)
  double thr;
  int* map;                       // (nb^3) a brick's slot among the active bricks, or -1
  uint8_t* flag;                  // (nb^3) candidate, then active, then march flags
  int* cnt;                       // (nb^3) evaluated points of a candidate brick; 0 elsewhere
  int* cand;                      // (nb^3) candidate bricks, increasing
  int* active;                    // (nb^3) active bricks, increasing
  int* march;                     // (nb^3) march bricks, increasing
  int* nsel;                      // [candidates, active, march]
  // sigma
  unsigned long long* rofs;       // (A + 1) the active bricks' first rows
  float* vals;                    // (A, 512) max(sigma, 0) per active brick, +0.0 where not evaluated
  long long slot0, slots;         // the chunk of active bricks being queried
  float* xyz;                     // (rows, 3) the chunk's evaluated positions
  long long* dst;                 // (rows) their index in vals
  float* out;                     // (rows) the query's sigma
  // march
  unsigned* bcnt;                 // (Mb + 1) vertices | triangles << 16 of each march brick
  unsigned long long* vofs;       // (Mb + 1) first vertex key of each march brick
  unsigned long long* tofs;       // (Mb + 1) first triangle key of each march brick
  unsigned long long* vkeys;      // (V) 3 q + axis
  unsigned long long* tkeys;      // (T) 5 c + t
  long long n_verts, n_tris;
  double* vertices;               // (V, 3) index space
  int* triangles;                 // (T, 3)
};

__device__ __forceinline__ void brick_coords(long long b, long long nb, long long& I, long long& J, long long& K) {
  I = b / (nb * nb);
  J = (b / nb) % nb;
  K = b % nb;
}

// Point l of a brick: its offsets (a, b, c) along (i, j, k).
__device__ __forceinline__ void brick_point(int l, int& a, int& b, int& c) {
  a = l >> 6;
  b = (l >> 3) & 7;
  c = l & 7;
}

// ---- 1. plan ------------------------------------------------------------------------------------------------------
// Whether any point of the brick can pass point_occupied.  Per axis, the brick's positions lie in [mn, mx] (a NaN
// position is never evaluated and is left out); grid coordinates are monotone in the position, so in each level the
// points' coordinates lie in [v(mn), v(mx)] and the cells point_occupied checks for them in
// [floor(v0) - 1, floor(v1)] clipped to the level.  Any occupied bit there, in any level, makes a candidate.
__device__ __forceinline__ bool brick_candidate(const SparseMcParams& p, long long I, long long J, long long K) {
  const MaskedGridParams& m = p.m;
  const SkipGrid& g = m.occ;
  const long long first[3] = {J * kBrick, I * kBrick, K * kBrick};   // x takes j, y takes i, z takes k
  double mn[3], mx[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    bool any = false;
    for (int t = 0; t < kBrick && first[a] + t < m.N; ++t) {
      const double x = static_cast<double>(mesh_linspace(m.lo[a], m.hi[a], m.N, first[a] + t));
      if (x != x) continue;
      mn[a] = any ? fmin(mn[a], x) : x;
      mx[a] = any ? fmax(mx[a], x) : x;
      any = true;
    }
    if (!any) return false;
  }
  const double Md = static_cast<double>(g.M);
  for (int k = 0; k < g.levels; ++k) {
    long long c0[3], c1[3];
    bool in = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      double v0 = (mn[a] - g.lo[k][a]) * g.scale[k][a], v1 = (mx[a] - g.lo[k][a]) * g.scale[k][a];
      if (v0 > v1) { const double s = v0; v0 = v1; v1 = s; }
      if (!(v1 >= 0.0 && v0 <= Md)) { in = false; continue; }
      v0 = v0 > 0.0 ? v0 : 0.0;
      v1 = v1 < Md ? v1 : Md;
      const long long f0 = static_cast<long long>(floor(v0)), f1 = static_cast<long long>(floor(v1));
      c0[a] = f0 > 0 ? f0 - 1 : 0;
      c1[a] = f1 < g.M - 1 ? f1 : g.M - 1;
    }
    if (!in) continue;
    const long long rows = (c1[1] - c0[1] + 1) * (c1[2] - c0[2] + 1);
    if (rows * ((c1[0] - c0[0]) / 32 + 2) > kBrickProbeWords) return true;
    const uint32_t* bits = g.bits + k * g.words;
    for (long long cz = c0[2]; cz <= c1[2]; ++cz)
      for (long long cy = c0[1]; cy <= c1[1]; ++cy) {
        const long long s = (cz * g.M + cy) * g.M + c0[0], e = s + (c1[0] - c0[0]);   // bits [s, e]
        for (long long w = s >> 5; w <= e >> 5; ++w) {
          uint32_t word = __ldg(bits + w);
          if (w == (s >> 5)) word &= ~0u << (s & 31);
          if (w == (e >> 5) && (e & 31) != 31) word &= (1u << ((e & 31) + 1)) - 1u;
          if (word) return true;
        }
      }
  }
  return false;
}

__global__ void smc_candidate_kernel(SparseMcParams p) {
  const long long B = p.nb * p.nb * p.nb;
  for (long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x; b < B; b += (long long)gridDim.x * blockDim.x) {
    long long I, J, K;
    brick_coords(b, p.nb, I, J, K);
    p.flag[b] = brick_candidate(p, I, J, K);
    p.cnt[b] = 0;
    p.map[b] = -1;
  }
}

// Point l of brick (I, J, K): whether it lies in the lattice and masked_point evaluates it; q its flat index.
__device__ __forceinline__ bool brick_evaluated(const SparseMcParams& p, long long I, long long J, long long K, int l,
                                                long long& q, float x[3]) {
  int a, b, c;
  brick_point(l, a, b, c);
  const long long i = I * kBrick + a, j = J * kBrick + b, k = K * kBrick + c;
  if (i >= p.m.N || j >= p.m.N || k >= p.m.N) return false;
  return masked_point(p.m, (i * p.m.N + j) * p.m.N + k, q, x);
}

// One CTA of kBrickPoints threads per candidate brick: its evaluated points by the exact rule.
__global__ void __launch_bounds__(kBrickPoints) smc_classify_kernel(SparseMcParams p) {
  const int n = p.nsel[0];
  for (int s = blockIdx.x; s < n; s += gridDim.x) {
    const long long b = p.cand[s];
    long long I, J, K, q;
    brick_coords(b, p.nb, I, J, K);
    float x[3];
    const int ev = __syncthreads_count(brick_evaluated(p, I, J, K, threadIdx.x, q, x));
    if (threadIdx.x == 0) {
      p.cnt[b] = ev;
      p.flag[b] = ev > 0;
    }
  }
}

__global__ void smc_map_kernel(SparseMcParams p) {
  const int n = p.nsel[1];
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) p.map[p.active[s]] = s;
}

// A brick is marched iff it or one of its neighbours at +1 along any subset of the axes is active: a cell's corners
// and an edge's upper endpoint lie in those bricks.
__global__ void smc_march_flag_kernel(SparseMcParams p) {
  const long long B = p.nb * p.nb * p.nb;
  for (long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x; b < B; b += (long long)gridDim.x * blockDim.x) {
    long long I, J, K;
    brick_coords(b, p.nb, I, J, K);
    bool any = false;
#pragma unroll
    for (int d = 0; d < 8; ++d) {
      const long long i = I + (d & 1), j = J + ((d >> 1) & 1), k = K + ((d >> 2) & 1);
      if (i < p.nb && j < p.nb && k < p.nb) any |= p.map[(i * p.nb + j) * p.nb + k] >= 0;
    }
    p.flag[b] = any;
  }
}

// ---- 2. sigma -----------------------------------------------------------------------------------------------------
// Evaluated points of each active brick (and a 0 past the last), for the scan that gives rofs.
__global__ void smc_row_counts_kernel(SparseMcParams p, unsigned long long* rcnt) {
  const long long n = p.nsel[1];
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s <= n; s += (long long)gridDim.x * blockDim.x)
    rcnt[s] = s < n ? static_cast<unsigned long long>(p.cnt[p.active[s]]) : 0ull;
}

// One CTA per active brick of the chunk: its evaluated points in brick order at rows rofs[slot] - rofs[slot0] + rank.
__global__ void __launch_bounds__(kBrickPoints) smc_sigma_emit_kernel(SparseMcParams p) {
  __shared__ int warp_ofs[kBrickPoints / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long s = p.slot0 + blockIdx.x; s < p.slot0 + p.slots; s += gridDim.x) {
    long long I, J, K, q;
    brick_coords(p.active[s], p.nb, I, J, K);
    float x[3];
    const bool ev = brick_evaluated(p, I, J, K, threadIdx.x, q, x);
    const unsigned ballot = __ballot_sync(0xffffffffu, ev);
    if (lane == 0) warp_ofs[warp] = __popc(ballot);
    __syncthreads();
    if (ev) {
      int rank = __popc(ballot & ((1u << lane) - 1u));
      for (int w = 0; w < warp; ++w) rank += warp_ofs[w];
      const unsigned long long row = p.rofs[s] - p.rofs[p.slot0] + static_cast<unsigned long long>(rank);
      p.xyz[row * 3 + 0] = x[0];
      p.xyz[row * 3 + 1] = x[1];
      p.xyz[row * 3 + 2] = x[2];
      p.dst[row] = s * kBrickPoints + threadIdx.x;
    }
    __syncthreads();
  }
}

// Row r to its point: max(sigma, 0) as masked_grid_scatter_kernel writes it (NaN and -0.0 pass through).
__global__ void smc_sigma_scatter_kernel(SparseMcParams p, long long rows) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
    const float v = p.out[r];
    p.vals[p.dst[r]] = v < 0.f ? 0.f : v;
  }
}

// ---- 3. march -----------------------------------------------------------------------------------------------------
// The value of lattice point (i, j, k) as the dense masked grid holds it.
__device__ __forceinline__ float smc_value(const SparseMcParams& p, long long i, long long j, long long k) {
  if (i >= p.m.N || j >= p.m.N || k >= p.m.N) return 0.f;
  const int s = p.map[((i >> 3) * p.nb + (j >> 3)) * p.nb + (k >> 3)];
  return s < 0 ? 0.f : p.vals[static_cast<long long>(s) * kBrickPoints + (((i & 7) * kBrick + (j & 7)) * kBrick + (k & 7))];
}

// The march brick's points and their +1 neighbours, 9^3 values, in shared memory; then point l's vertex edges and,
// for a cell of the lattice, its cube index.  Returns vertices | triangles << 16.
__device__ __forceinline__ unsigned smc_brick_point(const SparseMcParams& p, long long I, long long J, long long K,
                                                    float* tile, unsigned& emask, unsigned& cube) {
  for (int t = threadIdx.x; t < kBrickHalo * kBrickHalo * kBrickHalo; t += blockDim.x) {
    const int a = t / (kBrickHalo * kBrickHalo), b = (t / kBrickHalo) % kBrickHalo, c = t % kBrickHalo;
    tile[t] = smc_value(p, I * kBrick + a, J * kBrick + b, K * kBrick + c);
  }
  __syncthreads();
  const long long i0 = I * kBrick, j0 = J * kBrick, k0 = K * kBrick, N = p.m.N;
  const auto in = [&](long long i, long long j, long long k) {
    return mc_inside(tile[((i - i0) * kBrickHalo + (j - j0)) * kBrickHalo + (k - k0)], p.thr);
  };
  int a, b, c;
  brick_point(threadIdx.x, a, b, c);
  const long long i = i0 + a, j = j0 + b, k = k0 + c;
  emask = 0;
  cube = 0;
  unsigned nv = 0, nt = 0;
  if (i < N && j < N && k < N) {
    emask = mc_edge_mask(in, i, j, k, N, N, N);
    nv = __popc(emask);
  }
  if (i < N - 1 && j < N - 1 && k < N - 1) {
    cube = mc_cube(in, i, j, k);
    nt = nb_mc_tri_count[cube];
  }
  return nv | (nt << 16);
}

__global__ void __launch_bounds__(kBrickPoints) smc_march_count_kernel(SparseMcParams p) {
  using Reduce = cub::BlockReduce<unsigned, kBrickPoints>;
  __shared__ typename Reduce::TempStorage tmp;
  __shared__ float tile[kBrickHalo * kBrickHalo * kBrickHalo];
  const int n = p.nsel[2];
  for (int s = blockIdx.x; s < n; s += gridDim.x) {
    long long I, J, K;
    brick_coords(p.march[s], p.nb, I, J, K);
    unsigned emask, cube;
    const unsigned both = smc_brick_point(p, I, J, K, tile, emask, cube);
    const unsigned total = Reduce(tmp).Sum(both);   // at most 3 * 512 vertices and 5 * 512 triangles: no carry
    if (threadIdx.x == 0) p.bcnt[s] = total;
    __syncthreads();
  }
}

// bcnt -> the separate vertex and triangle counts, for the two scans
struct SmcVerts {
  __host__ __device__ unsigned long long operator()(unsigned v) const { return v & 0xffffu; }
};
struct SmcTris {
  __host__ __device__ unsigned long long operator()(unsigned v) const { return v >> 16; }
};

__global__ void __launch_bounds__(kBrickPoints) smc_march_emit_kernel(SparseMcParams p) {
  using Scan = cub::BlockScan<unsigned, kBrickPoints>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ float tile[kBrickHalo * kBrickHalo * kBrickHalo];
  const int n = p.nsel[2];
  const long long N = p.m.N, M = N - 1;
  for (int s = blockIdx.x; s < n; s += gridDim.x) {
    long long I, J, K;
    brick_coords(p.march[s], p.nb, I, J, K);
    unsigned emask, cube;
    const unsigned both = smc_brick_point(p, I, J, K, tile, emask, cube);
    unsigned rank;
    Scan(tmp).ExclusiveSum(both, rank);
    int a, b, c;
    brick_point(threadIdx.x, a, b, c);
    const long long i = I * kBrick + a, j = J * kBrick + b, k = K * kBrick + c;
    unsigned long long v = p.vofs[s] + (rank & 0xffffu), t = p.tofs[s] + (rank >> 16);
    const unsigned long long q = static_cast<unsigned long long>((i * N + j) * N + k);
#pragma unroll
    for (int ax = 0; ax < 3; ++ax)
      if (emask & (1u << ax)) p.vkeys[v++] = 3ull * q + ax;
    const int nt = (both >> 16);
    if (nt) {
      const unsigned long long cell = static_cast<unsigned long long>((i * M + j) * M + k);
      for (int r = 0; r < nt; ++r) p.tkeys[t + r] = 5ull * cell + r;
    }
    __syncthreads();
  }
}

// Sorted vertex key -> its position: the edge from q along the key's axis, as mc_emit_vertices_kernel places it.
__global__ void smc_vertices_kernel(SparseMcParams p) {
  const long long N = p.m.N;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < p.n_verts; v += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = p.vkeys[v];
    const long long q = static_cast<long long>(key / 3);
    const int axis = static_cast<int>(key % 3);
    const long long i = q / (N * N), j = (q / N) % N, k = q % N;
    const float f1 = smc_value(p, i + (axis == 0), j + (axis == 1), k + (axis == 2));
    mc_vertex(i, j, k, axis, p.thr, smc_value(p, i, j, k), f1, p.vertices + v * 3);
  }
}

__device__ __forceinline__ long long lower_bound_u64(const unsigned long long* a, long long n, unsigned long long v) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Sorted triangle key 5 c + t -> triangle t of cell c in table order, each corner the id of its edge's vertex (the
// rank of its key among the sorted vertex keys).
__global__ void smc_triangles_kernel(SparseMcParams p) {
  const long long N = p.m.N, M = N - 1;
  const auto in = [&](long long i, long long j, long long k) { return mc_inside(smc_value(p, i, j, k), p.thr); };
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < p.n_tris; t += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = p.tkeys[t];
    const long long c = static_cast<long long>(key / 5);
    const int r = static_cast<int>(key % 5);
    const long long i = c / (M * M), j = (c / M) % M, k = c % M;
    const unsigned cube = mc_cube(in, i, j, k);
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      long long d[3];
      const int axis = mc_edge_endpoint(nb_mc_tri_edges[cube][r * 3 + s], d);
      const long long q = ((i + d[0]) * N + (j + d[1])) * N + (k + d[2]);
      p.triangles[t * 3 + s] = static_cast<int>(lower_bound_u64(p.vkeys, p.n_verts, 3ull * q + axis));
    }
  }
}

}  // namespace nerfb200
