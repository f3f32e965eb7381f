// Coloured-mesh extraction (extract_color_mesh.py): dense grid positions, marching cubes, largest-cluster
// filter and occlusion-aware vertex colours.  The two MLP-bound stages (the sigma query and the occlusion
// renders) go through the existing launchers; everything here is memory-bound integer / fp64 work.
// Algorithms, conventions and the reference's quirks: DESIGN.md "Coloured mesh extraction".
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include "mc_table.h"

namespace nerfb200 {

// ---- 1. dense grid (extract_color_mesh.py:113-123) -----------------------------------------------
// np.linspace(lo, hi, N) in float64 (y = j * step + lo, last = hi) followed by the FloatTensor cast;
// __dmul_rn / __dadd_rn keep the two roundings numpy does (no FMA contraction).
__device__ __forceinline__ float mesh_linspace(double lo, double hi, long long N, long long j) {
  if (j == N - 1) return static_cast<float>(hi);
  const double step = __ddiv_rn(__dsub_rn(hi, lo), static_cast<double>(N - 1));
  return __double2float_rn(__dadd_rn(__dmul_rn(static_cast<double>(j), step), lo));
}

struct GridParams {
  double lo[3], hi[3];   // x, y, z ranges
  long long N, start, count;
  float* xyz;            // (count, 3)
};

// np.stack(np.meshgrid(x, y, z), -1).reshape(-1, 3): 'xy' indexing, flat point p = (i*N + j)*N + k
// holds (x_j, y_i, z_k).
__global__ void mesh_grid_positions_kernel(GridParams p) {
  const long long NN = p.N * p.N;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < p.count;
       t += (long long)gridDim.x * blockDim.x) {
    const long long q = p.start + t;
    const long long i = q / NN, j = (q / p.N) % p.N, k = q % p.N;
    p.xyz[t * 3 + 0] = mesh_linspace(p.lo[0], p.hi[0], p.N, j);
    p.xyz[t * 3 + 1] = mesh_linspace(p.lo[1], p.hi[1], p.N, i);
    p.xyz[t * 3 + 2] = mesh_linspace(p.lo[2], p.hi[2], p.N, k);
  }
}

// np.maximum(sigma, 0): NaN and -0.0 pass through as numpy leaves them.
__global__ void mesh_relu_kernel(float* s, long long n) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const float v = s[t];
    if (v < 0.f) s[t] = 0.f;
  }
}

// ---- 2. marching cubes (extract_color_mesh.py:144 mcubes.marching_cubes) ---------------------------
struct McParams {
  const float* sigma;
  long long n0, n1, n2;   // grid shape, C order
  double thr;
  uint8_t* vcnt;          // (P + 1) vertices owned by each grid point (its +axis edges)
  int* vofs;              // (P + 1) exclusive scan of vcnt
  uint8_t* ccnt;          // (C + 1) triangles of each cell
  int* cofs;              // (C + 1) exclusive scan of ccnt
  double* vertices;       // (V, 3) index space
  int* triangles;         // (T, 3)
};

// The rules of marching cubes on any value source, shared by the dense kernels below and the sparse ones
// (sparse_mc_kernels.cuh).  `in(i, j, k)` says whether point (i, j, k) is inside: double(value) > thr.
__device__ __forceinline__ bool mc_inside(float v, double thr) { return static_cast<double>(v) > thr; }

// bit a set: the edge from (i,j,k) along axis a exists in an (n0, n1, n2) grid and changes sign
template <class In>
__device__ __forceinline__ unsigned mc_edge_mask(const In& in, long long i, long long j, long long k, long long n0,
                                                 long long n1, long long n2) {
  const bool c = in(i, j, k);
  unsigned m = 0;
  if (i + 1 < n0 && in(i + 1, j, k) != c) m |= 1u;
  if (j + 1 < n1 && in(i, j + 1, k) != c) m |= 2u;
  if (k + 1 < n2 && in(i, j, k + 1) != c) m |= 4u;
  return m;
}

// bit c set: corner (i + (c & 1), j + (c >> 1 & 1), k + (c >> 2 & 1)) of cell (i, j, k) is inside
template <class In>
__device__ __forceinline__ unsigned mc_cube(const In& in, long long i, long long j, long long k) {
  unsigned cube = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c)
    if (in(i + (c & 1), j + ((c >> 1) & 1), k + ((c >> 2) & 1))) cube |= 1u << c;
  return cube;
}

// Edge e of the case table (nb_mc_tri_edges): its axis and the offset d of its lower endpoint from the cell's corner.
__device__ __forceinline__ int mc_edge_endpoint(int e, long long d[3]) {
  const int axis = e >> 2, r = e & 3;
  const int o1 = axis == 0 ? 1 : 0, o2 = axis == 2 ? 1 : 2;   // the two other axes, increasing
  d[0] = d[1] = d[2] = 0;
  d[o1] = r & 1;
  d[o2] = r >> 1;
  return axis;
}

// The vertex on the edge from (i, j, k) along `axis` with values f0 -> f1: a + (thr - f0)/(f1 - f0) on that axis,
// in double.
__device__ __forceinline__ void mc_vertex(long long i, long long j, long long k, int axis, double thr, float f0,
                                          float f1, double* out) {
  const double a = static_cast<double>(f0), b = static_cast<double>(f1);
  const double t = __ddiv_rn(__dsub_rn(thr, a), __dsub_rn(b, a));
  double pos[3] = {static_cast<double>(i), static_cast<double>(j), static_cast<double>(k)};
  pos[axis] = __dadd_rn(pos[axis], t);
  out[0] = pos[0];
  out[1] = pos[1];
  out[2] = pos[2];
}

__device__ __forceinline__ bool mc_in(const McParams& p, long long i, long long j, long long k) {
  return mc_inside(p.sigma[(i * p.n1 + j) * p.n2 + k], p.thr);
}

__device__ __forceinline__ unsigned mc_point_mask(const McParams& p, long long i, long long j, long long k) {
  return mc_edge_mask([&](long long a, long long b, long long c) { return mc_in(p, a, b, c); }, i, j, k, p.n0, p.n1,
                      p.n2);
}

__device__ __forceinline__ unsigned mc_cube_index(const McParams& p, long long i, long long j, long long k) {
  return mc_cube([&](long long a, long long b, long long c) { return mc_in(p, a, b, c); }, i, j, k);
}

__global__ void mc_classify_kernel(McParams p) {
  const long long P = p.n0 * p.n1 * p.n2;
  const long long m0 = p.n0 - 1, m1 = p.n1 - 1, m2 = p.n2 - 1;
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < P; q += (long long)gridDim.x * blockDim.x) {
    const long long i = q / (p.n1 * p.n2), j = (q / p.n2) % p.n1, k = q % p.n2;
    p.vcnt[q] = static_cast<uint8_t>(__popc(mc_point_mask(p, i, j, k)));
    if (i < m0 && j < m1 && k < m2)
      p.ccnt[(i * m1 + j) * m2 + k] = nb_mc_tri_count[mc_cube_index(p, i, j, k)];
  }
}

// Vertices in order of their lower endpoint's linear index, then edge axis; position a + (thr - f0)/(f1 - f0)
// along the edge, in double.
__global__ void mc_emit_vertices_kernel(McParams p) {
  const long long P = p.n0 * p.n1 * p.n2;
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < P; q += (long long)gridDim.x * blockDim.x) {
    if (p.vcnt[q] == 0) continue;
    const long long i = q / (p.n1 * p.n2), j = (q / p.n2) % p.n1, k = q % p.n2;
    const unsigned m = mc_point_mask(p, i, j, k);
    long long v = p.vofs[q];
    const long long step[3] = {p.n1 * p.n2, p.n2, 1};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!(m & (1u << a))) continue;
      mc_vertex(i, j, k, a, p.thr, p.sigma[q], p.sigma[q + step[a]], p.vertices + v * 3);
      ++v;
    }
  }
}

// Triangles in cell order, then table order.
__global__ void mc_emit_triangles_kernel(McParams p) {
  const long long m0 = p.n0 - 1, m1 = p.n1 - 1, m2 = p.n2 - 1;
  const long long C = m0 * m1 * m2;
  for (long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x; c < C; c += (long long)gridDim.x * blockDim.x) {
    const int nt = p.ccnt[c];
    if (nt == 0) continue;
    const long long i = c / (m1 * m2), j = (c / m2) % m1, k = c % m2;
    const unsigned cube = mc_cube_index(p, i, j, k);
    long long out = p.cofs[c];
    for (int t = 0; t < nt; ++t) {
      for (int s = 0; s < 3; ++s) {
        long long d[3];
        const int axis = mc_edge_endpoint(nb_mc_tri_edges[cube][t * 3 + s], d);
        const long long qi = i + d[0], qj = j + d[1], qk = k + d[2];
        const unsigned below = mc_point_mask(p, qi, qj, qk) & ((1u << axis) - 1u);
        p.triangles[out * 3 + s] = p.vofs[(qi * p.n1 + qj) * p.n2 + qk] + __popc(below);
      }
      ++out;
    }
  }
}

// ---- 3. index space -> world as extract_color_mesh.py:148-154 does it ------------------------------
// vertices_ = (v / N).astype(float32); x = (ymax-ymin)*v1 + ymin; y = (xmax-xmin)*v0 + xmin; z likewise.
// The scalars are float64 differences cast to float32 (numpy's weak-scalar promotion); the products and
// sums are float32 without contraction.
struct ToWorldParams {
  const double* v;
  long long n;
  double N;
  float scale[3], offset[3];   // per output column
  float* out;
};
__global__ void mesh_to_world_kernel(ToWorldParams p) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < p.n; t += (long long)gridDim.x * blockDim.x) {
    const float a0 = __double2float_rn(__ddiv_rn(p.v[t * 3 + 0], p.N));
    const float a1 = __double2float_rn(__ddiv_rn(p.v[t * 3 + 1], p.N));
    const float a2 = __double2float_rn(__ddiv_rn(p.v[t * 3 + 2], p.N));
    p.out[t * 3 + 0] = __fadd_rn(__fmul_rn(p.scale[0], a1), p.offset[0]);
    p.out[t * 3 + 1] = __fadd_rn(__fmul_rn(p.scale[1], a0), p.offset[1]);
    p.out[t * 3 + 2] = __fadd_rn(__fmul_rn(p.scale[2], a2), p.offset[2]);
  }
}

// ---- 4. largest cluster (extract_color_mesh.py:163-171) --------------------------------------------
// Triangles sharing an edge are joined.  The edges of all triangles are radix-sorted by (vmin, vmax); equal
// neighbours in the sorted list are united.  Union-find hooks the larger root under the smaller one (CAS),
// so parent[x] <= x always holds and every component's root is its lowest-indexed triangle, whatever the
// scheduling: the labels, counts and the chosen component are deterministic.
struct ClusterParams {
  const int* tris;
  long long n_tris, n_verts;
  unsigned long long* keys;
  int* vals;
  int* parent;
  int* count;
  unsigned long long* best;   // (count << 32) | ~label, max-reduced
  uint8_t* tflag;             // (T + 1)
  int* tofs;                  // (T + 1)
  uint8_t* vflag;             // (V + 1)
  int* vofs;                  // (V + 1)
  const float* vin;
  float* vout;
  int* tout;
};

__global__ void cluster_edges_kernel(ClusterParams p) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < p.n_tris; t += (long long)gridDim.x * blockDim.x) {
    const int a[3] = {p.tris[t * 3], p.tris[t * 3 + 1], p.tris[t * 3 + 2]};
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      const unsigned u = static_cast<unsigned>(a[e]), w = static_cast<unsigned>(a[(e + 1) % 3]);
      const unsigned lo = u < w ? u : w, hi = u < w ? w : u;
      p.keys[t * 3 + e] = (static_cast<unsigned long long>(lo) << 32) | hi;
      p.vals[t * 3 + e] = static_cast<int>(t);
    }
    p.parent[t] = static_cast<int>(t);
    p.count[t] = 0;
  }
}

__device__ __forceinline__ int uf_find(int* parent, int x) {
  while (true) {
    const int px = *reinterpret_cast<volatile int*>(&parent[x]);
    if (px == x) return x;
    const int gp = *reinterpret_cast<volatile int*>(&parent[px]);
    if (gp != px) parent[x] = gp;   // path halving: gp is an ancestor, parent values only ever decrease
    x = gp;
  }
}

__global__ void cluster_union_kernel(ClusterParams p) {
  const long long E = p.n_tris * 3;
  for (long long s = 1 + blockIdx.x * (long long)blockDim.x + threadIdx.x; s < E; s += (long long)gridDim.x * blockDim.x) {
    if (p.keys[s] != p.keys[s - 1]) continue;
    int a = p.vals[s], b = p.vals[s - 1];
    while (true) {
      a = uf_find(p.parent, a);
      b = uf_find(p.parent, b);
      if (a == b) break;
      const int hi = a > b ? a : b, lo = a > b ? b : a;
      if (atomicCAS(&p.parent[hi], hi, lo) == hi) break;
    }
  }
}

__global__ void cluster_label_kernel(ClusterParams p) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < p.n_tris; t += (long long)gridDim.x * blockDim.x) {
    const int r = uf_find(p.parent, static_cast<int>(t));
    atomicAdd(&p.count[r], 1);
  }
}

// after cluster_label_kernel (a kernel boundary later) every parent chain is final; store the roots
__global__ void cluster_best_kernel(ClusterParams p) {
  unsigned long long key = 0;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < p.n_tris; t += (long long)gridDim.x * blockDim.x) {
    const int r = uf_find(p.parent, static_cast<int>(t));
    if (r == t) {
      const unsigned long long k = (static_cast<unsigned long long>(p.count[t]) << 32) | (0xffffffffu - static_cast<unsigned>(t));
      key = k > key ? k : key;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
    key = other > key ? other : key;
  }
  if ((threadIdx.x & 31) == 0 && key) atomicMax(p.best, key);
}

__global__ void cluster_flag_kernel(ClusterParams p) {
  const int label = static_cast<int>(0xffffffffu - static_cast<unsigned>(*p.best & 0xffffffffull));
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < p.n_tris; t += (long long)gridDim.x * blockDim.x) {
    const bool keep = uf_find(p.parent, static_cast<int>(t)) == label;
    p.tflag[t] = keep;
    if (keep) {
      p.vflag[p.tris[t * 3 + 0]] = 1;
      p.vflag[p.tris[t * 3 + 1]] = 1;
      p.vflag[p.tris[t * 3 + 2]] = 1;
    }
  }
}

// remove_triangles_by_index + remove_unreferenced_vertices: both lists keep their order
__global__ void cluster_emit_kernel(ClusterParams p) {
  const long long n = p.n_tris > p.n_verts ? p.n_tris : p.n_verts;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    if (t < p.n_verts && p.vflag[t]) {
      const long long o = p.vofs[t];
      p.vout[o * 3 + 0] = p.vin[t * 3 + 0];
      p.vout[o * 3 + 1] = p.vin[t * 3 + 1];
      p.vout[o * 3 + 2] = p.vin[t * 3 + 2];
    }
    if (t < p.n_tris && p.tflag[t]) {
      const long long o = p.tofs[t];
      p.tout[o * 3 + 0] = p.vofs[p.tris[t * 3 + 0]];
      p.tout[o * 3 + 1] = p.vofs[p.tris[t * 3 + 1]];
      p.tout[o * 3 + 2] = p.vofs[p.tris[t * 3 + 2]];
    }
  }
}

// ---- 5. vertex colours (extract_color_mesh.py:206-284) ---------------------------------------------
// cv2.remap(image, mx, my, INTER_LINEAR) on a uint8 HxWx3 image, BORDER_CONSTANT 0: coordinates to 1/32
// pixel (cvRound = round half to even), 15-bit weights (32 - fy)(32 - fx)*32 ... (they sum to 2^15 exactly
// for the linear kernel), (sum + 2^14) >> 15.
__device__ __forceinline__ void remap_bilinear_u8(const uint8_t* img, int H, int W, float x, float y, uint8_t* out) {
  if (!(x == x) || !(y == y)) { out[0] = out[1] = out[2] = 0; return; }
  const int ix = __float2int_rn(x * 32.f), iy = __float2int_rn(y * 32.f);
  const int X = ix >> 5, Y = iy >> 5, fx = ix & 31, fy = iy & 31;
  if (X >= W || Y >= H || X < -1 || Y < -1) { out[0] = out[1] = out[2] = 0; return; }
  const int w[4] = {(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32};
  int acc[3] = {0, 0, 0};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int xx = X + (t & 1), yy = Y + (t >> 1);
    if (xx < 0 || yy < 0 || xx >= W || yy >= H) continue;
    const uint8_t* px = img + (static_cast<long long>(yy) * W + xx) * 3;
    acc[0] += px[0] * w[t];
    acc[1] += px[1] * w[t];
    acc[2] += px[2] * w[t];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int v = (acc[c] + (1 << 14)) >> 15;
    out[c] = static_cast<uint8_t>(v < 0 ? 0 : v > 255 ? 255 : v);
  }
}

__global__ void remap_bilinear_kernel(const uint8_t* img, int H, int W, const float* xy, long long n, uint8_t* out) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x)
    remap_bilinear_u8(img, H, W, xy[t * 2], xy[t * 2 + 1], out + t * 3);
}

struct ColorProjectParams {
  const float* vertices;   // (n, 3) world
  long long n;
  double w2c[12];          // np.linalg.inv(c2w4)[:3], float64
  float origin[3];         // FloatTensor(pose[:, -1])
  float focal;             // K is float32
  int W, H;
  const uint8_t* image;    // (H, W, 3)
  float near;
  uint8_t* colors;         // (n, 3)
  double* depth;           // (n)
  float* rays;             // (n, 8)
};

// :222-262 for one view.  P_w2c @ [v, 1] is summed in the order x, y, z, 1 in float64 without contraction
// (numpy's matmul goes through BLAS, whose order is its own); then the y / z flip, K (float32 entries,
// principal point (W/2, H/2)), depth = z + 1e-5, the float32 cast and the clip to the image.
__global__ void color_project_kernel(ColorProjectParams p) {
  const double cx = static_cast<double>(static_cast<float>(p.W * 0.5)), cy = static_cast<double>(static_cast<float>(p.H * 0.5));
  const double f = static_cast<double>(p.focal);
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < p.n; t += (long long)gridDim.x * blockDim.x) {
    const float vx = p.vertices[t * 3], vy = p.vertices[t * 3 + 1], vz = p.vertices[t * 3 + 2];
    double c[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      double s = __dmul_rn(p.w2c[r * 4 + 0], static_cast<double>(vx));
      s = __dadd_rn(s, __dmul_rn(p.w2c[r * 4 + 1], static_cast<double>(vy)));
      s = __dadd_rn(s, __dmul_rn(p.w2c[r * 4 + 2], static_cast<double>(vz)));
      c[r] = __dadd_rn(s, p.w2c[r * 4 + 3]);
    }
    c[1] = -c[1];
    c[2] = -c[2];
    const double u = __dadd_rn(__dmul_rn(f, c[0]), __dmul_rn(cx, c[2]));
    const double v = __dadd_rn(__dmul_rn(f, c[1]), __dmul_rn(cy, c[2]));
    const double depth = __dadd_rn(c[2], 1e-5);
    float x = __double2float_rn(__ddiv_rn(u, depth)), y = __double2float_rn(__ddiv_rn(v, depth));
    // np.clip keeps NaN
    x = x < 0.f ? 0.f : x > static_cast<float>(p.W - 1) ? static_cast<float>(p.W - 1) : x;
    y = y < 0.f ? 0.f : y > static_cast<float>(p.H - 1) ? static_cast<float>(p.H - 1) : y;
    remap_bilinear_u8(p.image, p.H, p.W, x, y, p.colors + t * 3);
    p.depth[t] = depth;
    // :255-262 rays [o, (v - o)/||v - o||, near, float32(depth)]
    const float dx = __fsub_rn(vx, p.origin[0]), dy = __fsub_rn(vy, p.origin[1]), dz = __fsub_rn(vz, p.origin[2]);
    const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    float* ray = p.rays + t * 8;
    ray[0] = p.origin[0]; ray[1] = p.origin[1]; ray[2] = p.origin[2];
    ray[3] = __fdiv_rn(dx, nrm); ray[4] = __fdiv_rn(dy, nrm); ray[5] = __fdiv_rn(dz, nrm);
    ray[6] = p.near;
    ray[7] = __double2float_rn(depth);
  }
}

// :269-277 in float64: w = 0.1/depth + (nan_to_num(opacity) < occ_threshold); sum += colour * w; wsum += w.
// nan_to_num(opacity, 1) passes 1 as `copy`, so NaN becomes 0 (and counts as not occluded); the comparison
// is float32 (numpy compares a float32 array with a Python float in float32).
__global__ void color_accumulate_kernel(const uint8_t* colors, const double* depth, const float* opacity, long long n,
                                        float occ_threshold, double* sum4) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    float op = opacity[t];
    if (op != op) op = 0.f;
    const double w = __dadd_rn(__ddiv_rn(0.1, depth[t]), op < occ_threshold ? 1.0 : 0.0);
    double* s = sum4 + t * 4;
    s[0] = __dadd_rn(s[0], __dmul_rn(static_cast<double>(colors[t * 3 + 0]), w));
    s[1] = __dadd_rn(s[1], __dmul_rn(static_cast<double>(colors[t * 3 + 1]), w));
    s[2] = __dadd_rn(s[2], __dmul_rn(static_cast<double>(colors[t * 3 + 2]), w));
    s[3] = __dadd_rn(s[3], w);
  }
}

// :283-284 (sum / wsum).astype(uint8): truncation.  A quotient outside [0, 256) only arises from negative
// weights (a vertex behind a camera); it keeps the low byte of its integer part, as x86 numpy does, NaN -> 0.
__global__ void color_finalize_kernel(const double* sum4, long long n, uint8_t* out) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double q = __ddiv_rn(sum4[t * 4 + c], sum4[t * 4 + 3]);
      out[t * 3 + c] = (q == q && fabs(q) < 9.0e18) ? static_cast<uint8_t>(static_cast<long long>(q) & 255) : 0;
    }
  }
}

// ---- 6. Unity volume (extract_mesh.ipynb "Generate .vol file for volume rendering in Unity") --------------
// Per point of the (N^3, 4) [rgb, raw sigma] grid: a = 1 - exp(fl32(c) * max(sigma, 0)) in float32, the product
// rounded once and exp taken in double then rounded to float32 (correctly rounded; numpy's SIMD float32 exp is
// not).  Kept where a > 0, as (i, r << 24 + g << 16 + b << 8 + trunc(a * 255)) with r = trunc(rgb * 255).
// Count / emit work on fixed tiles of kVolTile points, so the output order (increasing i) and the bytes do not
// depend on the launch shape.
constexpr int kVolThreads = 256;
constexpr int kVolTile = 16 * kVolThreads;

struct VolumeParams {
  const float4* rgbsigma;      // (P, 4)
  long long P;
  float c;                     // float32(-(xmax - xmin) / N), rounded on the host
  unsigned long long* tcnt;    // (tiles + 1) kept points per tile
  unsigned long long* tofs;    // (tiles + 1) exclusive scan of tcnt
  uint2* out;                  // (M) [i, s]
};

__device__ __forceinline__ bool volume_point(const float4 v, float c, uint32_t& s) {
  const float sg = v.w < 0.f ? 0.f : v.w;                       // np.maximum(sigma, 0): NaN stays NaN
  const float a = __fsub_rn(1.f, __double2float_rn(exp(static_cast<double>(__fmul_rn(c, sg)))));
  if (!(a > 0.f)) return false;
  const uint32_t r = static_cast<uint32_t>(__fmul_rn(v.x, 255.f));
  const uint32_t g = static_cast<uint32_t>(__fmul_rn(v.y, 255.f));
  const uint32_t b = static_cast<uint32_t>(__fmul_rn(v.z, 255.f));
  s = (r << 24) + (g << 16) + (b << 8) + static_cast<uint32_t>(__fmul_rn(a, 255.f));
  return true;
}

__global__ void __launch_bounds__(kVolThreads) volume_count_kernel(VolumeParams p) {
  using Reduce = cub::BlockReduce<int, kVolThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  const long long tiles = (p.P + kVolTile - 1) / kVolTile;
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    int n = 0;
#pragma unroll 4
    for (int r = 0; r < kVolTile / kVolThreads; ++r) {
      const long long q = t * kVolTile + r * kVolThreads + threadIdx.x;
      uint32_t s;
      if (q < p.P && volume_point(__ldg(p.rgbsigma + q), p.c, s)) ++n;
    }
    const int total = Reduce(tmp).Sum(n);
    if (threadIdx.x == 0) p.tcnt[t] = static_cast<unsigned long long>(total);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kVolThreads) volume_emit_kernel(VolumeParams p) {
  using Scan = cub::BlockScan<int, kVolThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const long long tiles = (p.P + kVolTile - 1) / kVolTile;
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    unsigned long long base = p.tofs[t];
    for (int r = 0; r < kVolTile / kVolThreads; ++r) {
      const long long q = t * kVolTile + r * kVolThreads + threadIdx.x;
      uint32_t s = 0;
      const int keep = (q < p.P && volume_point(__ldg(p.rgbsigma + q), p.c, s)) ? 1 : 0;
      int rank, total;
      Scan(tmp).ExclusiveSum(keep, rank, total);
      if (keep) p.out[base + rank] = make_uint2(static_cast<uint32_t>(q), s);
      base += static_cast<unsigned long long>(total);
      __syncthreads();
    }
  }
}

// ---- 7. vertex-normal colours (extract_color_mesh.py:187-203, --use_vertex_normal) -----------------
// Open3D TriangleMesh::ComputeVertexNormals() on a mesh without normals, in float64:
//   n_t = (v1 - v0) x (v2 - v0), Eigen's component formula, no contraction;
//   each vertex sums the n_t of its corners in increasing triangle index (corner order within a triangle);
//   normalize(): s = (x^2 + y^2) + z^2, divide by sqrt(s) when s > 0; then a NaN x becomes (0, 0, 1).
// The order comes from a stable radix sort of the 3T corners keyed by vertex (the values are triangle ids, so
// each vertex's segment lists its triangles in increasing order); no floating-point atomics anywhere.
struct NormalsParams {
  const float* vertices;   // (V, 3)
  const int* tris;         // (T, 3)
  long long n_verts, n_tris;
  int* keys;               // (3T) corner -> vertex, V for an index outside [0, V)
  int* vals;               // (3T) corner -> triangle
  double* tri_n;           // (T, 3) unnormalised triangle normals
  int* bad;                // set to 1 when an index is outside [0, V)
  double* normals;         // (V, 3)
};

// Reads the indices first and checks them before any vertex is addressed; a triangle with an index outside
// [0, V) flags `bad` and gets a zero normal, and its corners sort after every valid one.
__global__ void normals_triangle_kernel(NormalsParams p) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < p.n_tris; t += (long long)gridDim.x * blockDim.x) {
    int a[3];
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      a[c] = p.tris[t * 3 + c];
      const bool in = a[c] >= 0 && a[c] < p.n_verts;
      ok = ok && in;
      p.keys[t * 3 + c] = in ? a[c] : static_cast<int>(p.n_verts);
      p.vals[t * 3 + c] = static_cast<int>(t);
    }
    double n[3] = {0.0, 0.0, 0.0};
    if (ok) {
      double e1[3], e2[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double v0 = static_cast<double>(p.vertices[static_cast<long long>(a[0]) * 3 + c]);
        e1[c] = __dsub_rn(static_cast<double>(p.vertices[static_cast<long long>(a[1]) * 3 + c]), v0);
        e2[c] = __dsub_rn(static_cast<double>(p.vertices[static_cast<long long>(a[2]) * 3 + c]), v0);
      }
      n[0] = __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1]));
      n[1] = __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2]));
      n[2] = __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]));
    } else {
      *p.bad = 1;
    }
    p.tri_n[t * 3 + 0] = n[0];
    p.tri_n[t * 3 + 1] = n[1];
    p.tri_n[t * 3 + 2] = n[2];
  }
}

__device__ __forceinline__ long long lower_bound_i32(const int* a, long long n, int v) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// One thread per vertex: its segment of the sorted corners, summed in order, then Eigen's normalize().
__global__ void normals_vertex_kernel(NormalsParams p) {
  const long long E = p.n_tris * 3;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < p.n_verts; v += (long long)gridDim.x * blockDim.x) {
    const long long lo = lower_bound_i32(p.keys, E, static_cast<int>(v));
    double x = 0.0, y = 0.0, z = 0.0;
    for (long long s = lo; s < E && p.keys[s] == v; ++s) {
      const long long t = p.vals[s];
      x = __dadd_rn(x, p.tri_n[t * 3 + 0]);
      y = __dadd_rn(y, p.tri_n[t * 3 + 1]);
      z = __dadd_rn(z, p.tri_n[t * 3 + 2]);
    }
    const double sq = __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
    if (sq > 0.0) {
      const double r = __dsqrt_rn(sq);
      x = __ddiv_rn(x, r);
      y = __ddiv_rn(y, r);
      z = __ddiv_rn(z, r);
    }
    if (isnan(x)) { x = 0.0; y = 0.0; z = 1.0; }
    p.normals[v * 3 + 0] = x;
    p.normals[v * 3 + 1] = y;
    p.normals[v * 3 + 2] = z;
  }
}

// :190-193 rays [v - (d * near) * near_t, d, near, far] with d = fl32(normal), every operation fp32 as torch does
// it on the CPU (the scalars are fp32, rounded on the host).
__global__ void normal_rays_kernel(const float* vertices, const double* normals, long long n, float near, float far,
                                   float near_t, float* rays) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    float* ray = rays + t * 8;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float d = __double2float_rn(normals[t * 3 + c]);
      ray[c] = __fsub_rn(vertices[t * 3 + c], __fmul_rn(__fmul_rn(d, near), near_t));
      ray[3 + c] = d;
    }
    ray[6] = near;
    ray[7] = far;
  }
}

}  // namespace nerfb200
