// Empty-space skipping at render time: an occupancy bit field built from a dense sigma grid, rays classified
// against it by a cell walk over closed cells grown by a sample's float32 rounding, the live rays compacted in
// order, and the rendered results scattered back over a vacuum background.  The render kernel is not involved:
// these kernels run in front of and behind it.
// Conventions and the conservativeness argument: DESIGN.md "Empty-space skipping".
//
// AXIS ORDER.  The sigma grid is the one of nerfb200_sigma_grid: sigma[i, j, k] = sigma(x_j, y_i, z_k), flat
// (i * N + j) * N + k (np.meshgrid's 'xy' indexing: the FIRST index is y).  The occupancy grid undoes it: cell
// (cx, cy, cz) spans [x_cx, x_cx+1] x [y_cy, y_cy+1] x [z_cz, z_cz+1] with x_j = linspace(x_range, N)[j] etc.,
// its corners are sigma[cy + dy, cx + dx, cz + dz], its flat index is c = (cz * M + cy) * M + cx with M = N - 1
// (x fastest), and it is bit c % 32 of word c / 32.  The bits past the last cell are 0.
//
// CASCADE (DESIGN.md §10h).  A grid of L levels holds L such bit fields, level k's ceil(M^3 / 32) words after level
// k - 1's.  Level 0 is the given box; level k >= 1 has the same centre and 2^k times its half-extent.  A point
// belongs to the smallest level whose closed box contains it; a cell of level k >= 1 whose closed box lies inside
// level k - 1's (an *inner* cell, inner_cell) is never reached by that rule and is always 0.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace nerfb200 {

constexpr int kMaxLevels = 8;

// The occupancy grid as its readers take it: point_occupied (sample_skip_kernels.cuh) and the cell walk below.
struct SkipGrid {
  const uint32_t* bits;   // level k's bit field at bits + k * words
  long long M, words;     // cells per axis; words per level
  int levels;
  double lo[kMaxLevels][3], scale[kMaxLevels][3];   // level k's grid coordinate g = (x - lo) * scale; box [0, M]^3
};

// Level k - 1's box is [M/4, 3M/4] on each axis of level k's grid coordinates, so cell index a of level k >= 1 is
// inside it on that axis iff 4 a >= M and 4 (a + 1) <= 3 M: a in [inner_lo(M), inner_hi(M)).  A cell is inner iff
// all three of its indices are.  Level 0 passes an empty range (0, 0).
__host__ __device__ __forceinline__ long long inner_lo(long long M) { return (M + 3) / 4; }
__host__ __device__ __forceinline__ long long inner_hi(long long M) { return 3 * M / 4; }
__device__ __forceinline__ bool inner_cell(long long cx, long long cy, long long cz, long long ia, long long ib) {
  return cx >= ia && cx < ib && cy >= ia && cy < ib && cz >= ia && cz < ib;
}

// ---- 1. sigma grid -> cells -> dilation -> bits ---------------------------------------------------------
// A cell is occupied iff a corner has sigma > thr, which is "the largest of its 8 corners > thr" with a NaN
// corner counting as not above.  The comparison is made in double, as marching cubes makes it.  The inner cells
// [ia, ib)^3 of a cascade level are empty, so they dilate nothing.
__global__ void occ_cells_kernel(const float* __restrict__ sigma, long long N, double thr, long long ia, long long ib,
                                 uint8_t* __restrict__ occ) {
  const long long M = N - 1, C = M * M * M;
  for (long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    const long long cx = c % M, cy = (c / M) % M, cz = c / (M * M);
    bool any = false;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const long long j = cx + (q & 1), i = cy + ((q >> 1) & 1), k = cz + ((q >> 2) & 1);
      any |= static_cast<double>(sigma[(i * N + j) * N + k]) > thr;
    }
    occ[c] = any && !inner_cell(cx, cy, cz, ia, ib);
  }
}

// One axis of the Chebyshev dilation (a box dilation is separable): out = OR of in over [-r, r] along the axis
// of stride `stride` cells, clipped to the grid.
__global__ void occ_dilate_axis_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, long long M,
                                       long long stride, int r) {
  const long long C = M * M * M;
  for (long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    const long long a = (c / stride) % M;
    const long long lo = a - r < 0 ? 0 : a - r, hi = a + r > M - 1 ? M - 1 : a + r;
    uint8_t v = 0;
    for (long long b = lo; b <= hi && !v; ++b) v = in[c + (b - a) * stride];
    out[c] = v;
  }
}

// 32 cells per word by warp ballot.  The launch has a multiple of 32 threads and every lane of a warp runs the
// same number of rounds (the bound is rounded up to a whole word).  The inner cells [ia, ib)^3 are cleared, which
// the dilation may have set.
__global__ void occ_pack_kernel(const uint8_t* __restrict__ occ, long long M, long long ia, long long ib,
                                uint32_t* __restrict__ bits) {
  const long long C = M * M * M, C_pad = (C + 31) / 32 * 32;
  for (long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x; c < C_pad; c += (long long)gridDim.x * blockDim.x) {
    const bool on = c < C && occ[c] != 0 && !(ia < ib && inner_cell(c % M, (c / M) % M, c / (M * M), ia, ib));
    const unsigned w = __ballot_sync(0xffffffffu, on);
    if ((threadIdx.x & 31) == 0) bits[c >> 5] = w;
  }
}

__global__ void occ_popcount_kernel(const uint32_t* __restrict__ bits, long long n_words, unsigned long long* total) {
  unsigned long long s = 0;
  for (long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x; w < n_words; w += (long long)gridDim.x * blockDim.x)
    s += __popc(bits[w]);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(total, s);
}

// ---- 2. ray classification -------------------------------------------------------------------------------
struct CullParams {
  const float* rays;      // (n, 8) [o, d, near, far]
  long long n;
  SkipGrid grid;
  uint8_t* flag;          // (n)
  int* tcnt;              // live rays of each tile
  long long* tofs;        // exclusive scan of tcnt, n_tiles + 1
  long long* live_idx;
  float* live_rays;
};

constexpr int kCullTile = 256;   // rays per tile = threads per block

// Whether the segment o + t d, t in [t0, t1] meets cell c's closed box grown by del[a] on each axis: a slab test in
// grid coordinates.  A zero direction component has del = 0 and tests its coordinate against [c, c + 1] exactly.
__device__ __forceinline__ bool cull_grown_cell_meets(int cx, int cy, int cz, const double o[3], const double d[3],
                                                      const double inv[3], const double del[3], double t0, double t1) {
  const int c[3] = {cx, cy, cz};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double lo = static_cast<double>(c[a]), hi = static_cast<double>(c[a] + 1);
    if (d[a] == 0.0) {
      if (o[a] < lo || o[a] > hi) return false;
    } else {
      const double ta = (lo - del[a] - o[a]) * inv[a], tb = (hi + del[a] - o[a]) * inv[a];
      t0 = fmax(t0, fmin(ta, tb));
      t1 = fmin(t1, fmax(ta, tb));
    }
  }
  return t0 <= t1;
}

// Whether level k calls the segment o + t d, t in [near, far] (v: a finite ray with far > near) live: whether it meets
// the closed box of an occupied cell grown by del_a = 2^-22 |scale_a| (|o_a| + |d_a| max(|near|, |far|)) grid units
// on each axis a (0 where d_a = 0), which covers the float32 rounding of every sample point the renderer places on
// the segment (DESIGN.md §10 "Live").  A level with del_a >= 1/2 on some axis is live wherever its grown box meets
// the segment.
//
// Amanatides-Woo in grid coordinates, in double, over the segment clipped to the grown box; each boundary time is
// recomputed from the cell index, so no error accumulates along the walk.  The walk runs on the lattice extended by
// a ring of empty cells -1 and M, which holds the part of the segment in the grown margin outside the box.  At each
// visited cell it takes, on each axis whose face the segment comes within del_a of inside the cell (within
// del_a / |d_a| of the time it crosses that face), the neighbour across that face: every cell cell + s with s_a in
// {-1, 0, 1} so allowed is a candidate, and an occupied candidate is confirmed by a slab test against its grown box.
// With del < 1 every cell whose grown box meets the segment is a candidate of some visited cell, so the result is
// the grown-box rule.  A segment usually enters and leaves a cell across faces, whose single-axis neighbours are
// the previous and next visited cells; those are not probed twice, so a step reads one bit unless the segment
// passes near an edge.
__device__ __forceinline__ bool cull_level_live(const SkipGrid& g, int k, const float v[8]) {
  const double M = static_cast<double>(g.M);
  const uint32_t* bits = g.bits + k * g.words;
  const double tmax = fmax(fabs(static_cast<double>(v[6])), fabs(static_cast<double>(v[7])));
  double o[3], d[3], inv[3], del[3];
  double t0 = v[6], t1 = v[7];
  bool coarse = false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    o[a] = (static_cast<double>(v[a]) - g.lo[k][a]) * g.scale[k][a];
    d[a] = static_cast<double>(v[3 + a]) * g.scale[k][a];
    if (d[a] == 0.0) {
      inv[a] = 0.0;
      del[a] = 0.0;
      if (o[a] < 0.0 || o[a] > M) return false;
    } else {
      inv[a] = 1.0 / d[a];
      // rounded as written (no contraction), so that tests/occupancy_ref.py restates it bit for bit
      const double ao = fabs(static_cast<double>(v[a])), ad = fabs(static_cast<double>(v[3 + a]));
      del[a] = __dmul_rn(0x1p-22 * fabs(g.scale[k][a]), __dadd_rn(ao, __dmul_rn(ad, tmax)));
      coarse |= del[a] >= 0.5;
      const double ta = (0.0 - del[a] - o[a]) * inv[a], tb = (M + del[a] - o[a]) * inv[a];
      t0 = fmax(t0, fmin(ta, tb));
      t1 = fmin(t1, fmax(ta, tb));
    }
  }
  if (!(t0 <= t1)) return false;
  if (coarse) return true;
  // cell indices in [-1, M] (M <= 1624) fit an int; only the flat bit index needs 64 bits
  const int Mi = static_cast<int>(g.M);
  int cell[3];
  double tnext[3], eps[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double f = floor(__dadd_rn(o[a], __dmul_rn(t0, d[a])));
    cell[a] = static_cast<int>(fmin(fmax(f, -1.0), M));
    eps[a] = __dmul_rn(del[a], fabs(inv[a]));   // del_a grid units in time along the ray
  }
  const double inf = __longlong_as_double(0x7ff0000000000000LL);
  const int steps = 3 * (Mi + 2) + 3;
  double te = t0;   // when the segment entered the current cell
  int entry = -1;   // the axis it entered across (-1: the first cell)
  for (int s = 0; s < steps; ++s) {
    double tlow[3];   // when the segment crosses the cell's face behind it on each axis
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      tnext[a] = d[a] == 0.0 ? inf : (static_cast<double>(cell[a] + (d[a] > 0.0 ? 1 : 0)) - o[a]) * inv[a];
      tlow[a] = d[a] == 0.0 ? -inf : (static_cast<double>(cell[a] + (d[a] > 0.0 ? 0 : 1)) - o[a]) * inv[a];
    }
    const int ax = tnext[0] <= tnext[1] ? (tnext[0] <= tnext[2] ? 0 : 2) : (tnext[1] <= tnext[2] ? 1 : 2);
    const double tmin = fmin(fmin(tnext[0], tnext[1]), tnext[2]);   // tnext[ax], without indexing by a variable
    const bool more = tmin <= t1;
    const double tx = fmin(tmin, t1);
    // The faces the segment comes within del_a of while inside the cell: the one behind it (back) if it entered
    // within eps_a of crossing it, the one ahead (ahead) if it leaves within eps_a of crossing that.  A zero
    // component sits at o_a: on the cell's low face iff o_a == cell_a.
    bool back[3], ahead[3];
    unsigned wide = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      back[a] = d[a] == 0.0 ? o[a] - static_cast<double>(cell[a]) <= 0.0 : te - tlow[a] <= eps[a];
      ahead[a] = d[a] == 0.0 ? static_cast<double>(cell[a] + 1) - o[a] <= 0.0 : tnext[a] - tx <= eps[a];
      wide |= (back[a] || ahead[a] ? 1u : 0u) << a;
    }
    // The cell the walk came from and the one it goes to next are visited cells, probed on their own visits: a
    // single-axis offset onto one of them is dropped (offsets combined with another axis are kept).
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const bool alone = !(wide & ~(1u << a));
      if (a == entry && alone) back[a] = false;
      if (a == ax && more && alone) ahead[a] = false;
    }
    int s0[3], s1[3];   // offsets on the cell's own axes: -1 toward lower indices, +1 toward higher
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const bool lower = d[a] < 0.0 ? ahead[a] : back[a], upper = d[a] < 0.0 ? back[a] : ahead[a];
      s0[a] = lower ? -1 : 0;
      s1[a] = upper ? 1 : 0;
    }
    // scalar loop indices: an index array would live in local memory
    const int x0 = max(cell[0] + s0[0], 0), x1 = min(cell[0] + s1[0], Mi - 1);
    const int y0 = max(cell[1] + s0[1], 0), y1 = min(cell[1] + s1[1], Mi - 1);
    const int z0 = max(cell[2] + s0[2], 0), z1 = min(cell[2] + s1[2], Mi - 1);
    for (int cz = z0; cz <= z1; ++cz)
      for (int cy = y0; cy <= y1; ++cy)
        for (int cx = x0; cx <= x1; ++cx) {
          const long long b = (static_cast<long long>(cz) * g.M + cy) * g.M + cx;
          if (((bits[b >> 5] >> (b & 31)) & 1u) && cull_grown_cell_meets(cx, cy, cz, o, d, inv, del, t0, t1))
            return true;
        }
    if (!more) return false;
    // unrolled over the axis so that the per-axis arrays stay in registers
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (a != ax) continue;
      cell[a] += d[a] > 0.0 ? 1 : -1;
      if (cell[a] < -1 || cell[a] > Mi) return false;
    }
    entry = ax;
    te = tmin;
  }
  return false;
}

// Live iff the segment crosses an occupied cell of some level: the walk of each level's box in turn.  Inner cells
// are 0, so this finds every cell point_occupied can find.  A ray the walk cannot judge (a non-finite value,
// far <= near) is live: the renderer then sees it unchanged.
__device__ __forceinline__ bool cull_ray_live(const CullParams& p, const float* r) {
  float v[8];
#pragma unroll
  for (int a = 0; a < 8; ++a) v[a] = r[a];
  bool finite = true;
#pragma unroll
  for (int a = 0; a < 8; ++a) finite &= isfinite(v[a]);
  if (!finite || !(v[7] > v[6])) return true;
  for (int k = 0; k < p.grid.levels; ++k)
    if (cull_level_live(p.grid, k, v)) return true;
  return false;
}

// One tile of kCullTile rays per round: the flags and the tile's live count.
__global__ void cull_classify_kernel(CullParams p) {
  const long long n_tiles = (p.n + kCullTile - 1) / kCullTile;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long i = tile * kCullTile + threadIdx.x;
    const bool live = i < p.n && cull_ray_live(p, p.rays + i * 8);
    if (i < p.n) p.flag[i] = live;
    const int cnt = __syncthreads_count(live);
    if (threadIdx.x == 0) p.tcnt[tile] = cnt;
  }
}

// Exclusive scan of the tile counts by one block of 1024 threads, 1024 tiles per round with a running carry;
// tofs[n_tiles] is the total.
__global__ void cull_scan_kernel(const int* __restrict__ tcnt, long long* __restrict__ tofs, long long n_tiles) {
  __shared__ long long warp_sum[32];
  __shared__ long long carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (long long base = 0; base < n_tiles; base += 1024) {
    const long long i = base + threadIdx.x;
    const long long own = i < n_tiles ? tcnt[i] : 0;
    long long incl = own;
    for (int o = 1; o < 32; o <<= 1) {
      const long long up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      long long w = warp_sum[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const long long up = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += up;
      }
      warp_sum[lane] = w;   // inclusive over the warps
    }
    __syncthreads();
    const long long before = carry + (warp ? warp_sum[warp - 1] : 0) + incl - own;
    if (i < n_tiles) tofs[i] = before;
    __syncthreads();
    if (threadIdx.x == 1023) carry = before + own;
    __syncthreads();
  }
  if (threadIdx.x == 0) tofs[n_tiles] = carry;
}

// The stable compaction: live ray i goes to row tofs[tile] + (live rays before it in the tile), so live_idx is
// increasing.  The index and the 32-byte ray are written in the same pass.
__global__ void cull_emit_kernel(CullParams p) {
  __shared__ int warp_cnt[kCullTile / 32];
  const long long n_tiles = (p.n + kCullTile - 1) / kCullTile;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long i = tile * kCullTile + threadIdx.x;
    const bool live = i < p.n && p.flag[i] != 0;
    const unsigned m = __ballot_sync(0xffffffffu, live);
    if (lane == 0) warp_cnt[warp] = __popc(m);
    __syncthreads();
    if (live) {
      long long row = p.tofs[tile] + __popc(m & ((1u << lane) - 1u));
      for (int w = 0; w < warp; ++w) row += warp_cnt[w];
      p.live_idx[row] = i;
      const float4* src = reinterpret_cast<const float4*>(p.rays + i * 8);
      float4* dst = reinterpret_cast<float4*>(p.live_rays + row * 8);
      dst[0] = src[0];
      dst[1] = src[1];
    }
    __syncthreads();
  }
}

// ---- 3. scatter with background fill ------------------------------------------------------------------
// The six result tensors of a render in the order rgb_coarse, depth_coarse, opacity_coarse, rgb_fine, depth_fine,
// opacity_fine; a NULL pair is skipped.
struct ScatterParams {
  const float* src[6];    // compacted (n_live, 3) / (n_live)
  float* dst[6];          // full size
  const long long* live_idx;
  long long n_live, n;
  float bg;               // rgb of a ray through vacuum: 1 with white_back, else 0 (depth and opacity: 0)
};

// One thread per output ray: its row among the live rays by binary search of the increasing live_idx, then every
// key is written once, from the render or from the vacuum value.
__global__ void scatter_results_kernel(ScatterParams p) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
    long long lo = 0, hi = p.n_live;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (p.live_idx[mid] < i) lo = mid + 1; else hi = mid;
    }
    const bool live = lo < p.n_live && p.live_idx[lo] == i;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      if (!p.dst[k]) continue;
      if (k % 3 == 0) {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) p.dst[k][i * 3 + ch] = live ? p.src[k][lo * 3 + ch] : p.bg;
      } else {
        p.dst[k][i] = live ? p.src[k][lo] : 0.f;
      }
    }
  }
}

}  // namespace nerfb200
