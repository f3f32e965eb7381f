// A baked volume (DESIGN.md §10j): [sigmoid rgb, raw sigma] of the N^3 lattice of rgb_sigma_grid, stored in the
// bricks of the sparse marching cubes' plan (sparse_mc_kernels.cuh) and ray-marched without the MLP.
//
// Layout of one volume buffer (nerfb200_baked_bytes):
//   data:  (bricks, 9, 9, 9) float4 [r, g, b, sigma]: brick (I, J, K)'s points (8 I + a, 8 J + b, 8 K + c) for a, b, c
//          in [0, 8], so the +1 apron repeats the first points of the neighbours (0 where a neighbour is not stored,
//          and past the lattice); the order of the bricks is the order of their list (march bricks, increasing);
//   map:   (nb^3) int32 after the data: a brick's slot, or -1 where it is not stored.
//
// bake:       the plan's march bricks are stored; the evaluated points of the active bricks go through the rgb + sigma
//             query on compacted rows (the rows of the sparse marching cubes' sigma step) and are scattered into their
//             bricks, then every apron point is copied from its neighbour;
// from_grid:  a dense (N, N, N, 4) grid: the bricks whose 9^3 points hold a sigma with max(sigma, 0) != 0 are stored;
// render:     one thread per ray; samples at t_k = near + (k + 1/2) dt, each computed from k, looked up in the brick its
//             cell lies in.  A sample outside the box or in a brick that is not stored has sigma = 0, so alpha = 0:
//             such runs of samples are jumped over, and a jump is taken only after the last sample it skips is found
//             in the same brick as the first (see baked_skip), so skipping never changes a value.
//
// The kernels are templated on kW, the float4 count per point: 1 for the volume above, 7 for the view-dependent one
// of DESIGN.md §10k, whose point is (c_r0, c_g0, c_b0, sigma) and then c_{r,g,b; m} for m = 1..8 (degree-2 spherical
// harmonics of PlenOctrees' eval_sh); its render evaluates the colour at each ray's direction.
#pragma once
#include <cstdint>
#include <cub/cub.cuh>

#include "sparse_mc_kernels.cuh"

namespace nerfb200 {

constexpr int kBakedSide = kBrickHalo;                                   // 9 points per brick axis, apron included
constexpr int kBakedPoints = kBakedSide * kBakedSide * kBakedSide;       // 729
constexpr int kBakedThreads = 128;                                      // rays per CTA of the render
constexpr long long kBakedMaxSamples = 1LL << 40;                       // K is clamped here (far beyond any box)

__device__ __forceinline__ int baked_point(int a, int b, int c) { return (a * kBakedSide + b) * kBakedSide + c; }

// ---- bake -----------------------------------------------------------------------------------------------------------
// The stored bricks' slots: vmap (memset to -1 before) of list[s] = s.
__global__ void baked_map_kernel(const int* list, const int* count, int* vmap) {
  const int n = *count;
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) vmap[list[s]] = s;
}

// Row r of the point query (p.out holds kW float4 per row) to its point in its march brick's storage.
template <int kW>
__global__ void baked_scatter_kernel(SparseMcParams p, const int* vmap, float4* data, long long rows) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
    const long long dst = p.dst[r];
    const long long s = dst / kBrickPoints;
    int a, b, c;
    brick_point(static_cast<int>(dst % kBrickPoints), a, b, c);
    const long long m = vmap[p.active[s]];
#pragma unroll
    for (int w = 0; w < kW; ++w)
      data[(m * kBakedPoints + baked_point(a, b, c)) * kW + w] = reinterpret_cast<const float4*>(p.out)[r * kW + w];
  }
}

// Every apron point (a, b or c = 8) of every stored brick from its neighbour's first points, or 0 where the neighbour
// is not stored or lies past the lattice.  Reads interior points only, which the scatter wrote.
template <int kW>
__global__ void baked_apron_kernel(const int* list, const int* count, const int* vmap, long long nb, float4* data) {
  const long long n = static_cast<long long>(*count) * kBakedPoints;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long s = e / kBakedPoints;
    const int t = static_cast<int>(e % kBakedPoints);
    const int a = t / (kBakedSide * kBakedSide), b = (t / kBakedSide) % kBakedSide, c = t % kBakedSide;
    if (a < kBrick && b < kBrick && c < kBrick) continue;
    long long I, J, K;
    brick_coords(list[s], nb, I, J, K);
    I += a >> 3;
    J += b >> 3;
    K += c >> 3;
#pragma unroll
    for (int w = 0; w < kW; ++w) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (I < nb && J < nb && K < nb) {
        const long long m = vmap[(I * nb + J) * nb + K];
        if (m >= 0) v = data[(m * kBakedPoints + baked_point(a & 7, b & 7, c & 7)) * kW + w];
      }
      data[(s * kBakedPoints + t) * kW + w] = v;
    }
  }
}

// ---- from a dense grid ----------------------------------------------------------------------------------------------
// One CTA per brick: whether one of its 9^3 lattice points holds a sigma with max(sigma, 0) != 0 (NaN and +inf
// included), i.e. !(sigma <= 0).  Sigma is the w of a point's first float4.
template <int kW>
__global__ void __launch_bounds__(256) baked_grid_flag_kernel(const float4* grid, long long N, long long nb,
                                                              uint8_t* flag) {
  const long long B = nb * nb * nb;
  for (long long br = blockIdx.x; br < B; br += gridDim.x) {
    long long I, J, K;
    brick_coords(br, nb, I, J, K);
    bool any = false;
    for (int t = threadIdx.x; t < kBakedPoints; t += blockDim.x) {
      const long long i = I * kBrick + t / (kBakedSide * kBakedSide), j = J * kBrick + (t / kBakedSide) % kBakedSide,
                      k = K * kBrick + t % kBakedSide;
      if (i < N && j < N && k < N) any |= !(grid[((i * N + j) * N + k) * kW].w <= 0.f);
    }
    any = __syncthreads_or(any);
    if (threadIdx.x == 0) flag[br] = any;
  }
}

// The 9^3 points of every stored brick from the dense grid, 0 past the lattice.
template <int kW>
__global__ void baked_grid_copy_kernel(const float4* grid, long long N, const int* list, const int* count, long long nb,
                                       float4* data) {
  const long long n = static_cast<long long>(*count) * kBakedPoints;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long s = e / kBakedPoints;
    const int t = static_cast<int>(e % kBakedPoints);
    long long I, J, K;
    brick_coords(list[s], nb, I, J, K);
    const long long i = I * kBrick + t / (kBakedSide * kBakedSide), j = J * kBrick + (t / kBakedSide) % kBakedSide,
                    k = K * kBrick + t % kBakedSide;
    const bool in = i < N && j < N && k < N;
#pragma unroll
    for (int w = 0; w < kW; ++w)
      data[e * kW + w] = in ? grid[((i * N + j) * N + k) * kW + w] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// ---- back to a dense grid -------------------------------------------------------------------------------------------
// Point (i, j, k) from the brick that holds it at a, b, c < 8; (0, 0, 0, 0) where that brick is not stored.
template <int kW>
__global__ void baked_to_dense_kernel(const float4* data, const int* vmap, long long N, long long nb, float4* out) {
  const long long total = N * N * N;
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < total; q += (long long)gridDim.x * blockDim.x) {
    const long long i = q / (N * N), j = (q / N) % N, k = q % N;
    const long long m = vmap[((i >> 3) * nb + (j >> 3)) * nb + (k >> 3)];
    const long long src = (m * kBakedPoints + baked_point(static_cast<int>(i & 7), static_cast<int>(j & 7),
                                                           static_cast<int>(k & 7))) * kW;
#pragma unroll
    for (int w = 0; w < kW; ++w) out[q * kW + w] = m < 0 ? make_float4(0.f, 0.f, 0.f, 0.f) : data[src + w];
  }
}

// ---- render ---------------------------------------------------------------------------------------------------------
struct BakedRenderParams {
  const float4* data;
  const int* map;
  int N, nb;
  float lo[3], scale[3];       // u_a = (p_a - lo_a) * scale_a, scale_a = (N - 1) / (hi_a - lo_a); x, y, z
  float step;                  // s, world units
  float eps;                   // early stop: a ray ends after the first sample with T < eps
  float white_back;
  const float* rays;           // (n, 8) [o, d, near, far]
  long long n;
  float* rgb;                  // (n, 3)
  float* depth;                // (n)
  float* opacity;              // (n)
};

// Sample k's depth and its index coordinates u (x, y, z), each operation rounded once in the order written (the float64
// reference repeats these float32 operations): t and every u_a are monotone in k.
__device__ __forceinline__ float baked_t(float near, float dt, long long k) {
  return __fadd_rn(near, __fmul_rn(__fadd_rn(__ll2float_rn(k), 0.5f), dt));
}

__device__ __forceinline__ float baked_u(const BakedRenderParams& r, int a, float o, float d, float t) {
  return __fmul_rn(__fsub_rn(__fadd_rn(o, __fmul_rn(t, d)), r.lo[a]), r.scale[a]);
}

// The brick coordinate of u along one axis: -1 below the box, nb above it, else the brick of the cell floor(u)
// clamped to [0, N - 2].  Monotone in u.
__device__ __forceinline__ int baked_axis_key(float u, int N, int nb) {
  if (!(u >= 0.f)) return -1;
  if (u > static_cast<float>(N - 1)) return nb;
  return min(static_cast<int>(u), N - 2) >> 3;
}

// The three axis keys of sample k packed in one int (each + 1 in 10 bits; nb <= 256).
__device__ __forceinline__ int baked_key(const BakedRenderParams& r, const float o[3], const float d[3], float near,
                                         float dt, long long k, float u[3], float& t) {
  t = baked_t(near, dt, k);
  int key = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    u[a] = baked_u(r, a, o[a], d[a], t);
    key = (key << 10) | (baked_axis_key(u[a], r.N, r.nb) + 1);
  }
  return key;
}

// Sample k of key `key` is empty (outside the box, or in a brick that is not stored): the next sample that may not be.
// Every axis key is monotone in k, so if sample kc > k has the same three keys, so has every sample between them, and
// all of k .. kc are empty.  kc is estimated from where the ray leaves the brick (or enters the box), one sample early,
// and checked; halved towards k when the check fails; k + 1 if no candidate holds.  An axis that stays out of the box
// for good (moving away from it, or not moving) ends the ray.
__device__ __forceinline__ long long baked_skip(const BakedRenderParams& r, const float o[3], const float d[3],
                                                float near, float dt, long long k, long long K, int key) {
  float t_exit = INFINITY;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int ka = ((key >> (10 * (2 - a))) & 1023) - 1;
    const float du = d[a] * r.scale[a];
    float bound;
    if (ka < 0) {
      if (!(du > 0.f)) return K;
      bound = 0.f;
    } else if (ka >= r.nb) {
      if (!(du < 0.f)) return K;
      bound = static_cast<float>(r.N - 1);
    } else if (du > 0.f) {
      bound = ka == r.nb - 1 ? static_cast<float>(r.N - 1) : static_cast<float>(kBrick * (ka + 1));
    } else if (du < 0.f) {
      bound = static_cast<float>(kBrick * ka);
    } else {
      continue;
    }
    t_exit = fminf(t_exit, (bound / r.scale[a] + r.lo[a] - o[a]) / d[a]);
  }
  const float kf = floorf((t_exit - near) / dt - 0.5f) - 1.f;
  long long kc = kf < static_cast<float>(K - 1) ? static_cast<long long>(kf) : K - 1;
  float u[3], t;
  for (int tries = 0; tries < 4 && kc > k; ++tries) {
    if (baked_key(r, o, d, near, dt, kc, u, t) == key) return kc + 1;
    kc = k + (kc - k) / 2;
  }
  return k + 1;
}

__device__ __forceinline__ float baked_sigma(float s) { return s < 0.f ? 0.f : s; }   // max(sigma, 0), NaN passes

__device__ __forceinline__ float baked_lerp(float a, float b, float f) {
  return __fadd_rn(__fmul_rn(__fsub_rn(1.f, f), a), __fmul_rn(f, b));
}

// PlenOctrees' eval_sh constants, degree 2.
constexpr float kShC0 = 0.28209479177387814f;
constexpr float kShC1 = 0.4886025119029199f;
constexpr float kShC2_0 = 1.0925484305920792f, kShC2_1 = -1.0925484305920792f, kShC2_2 = 0.31539156525252005f,
                kShC2_3 = -1.0925484305920792f, kShC2_4 = 0.5462742152960396f;

// The 9 basis values at the unit direction (x, y, z), each operation rounded once in the order written.
__device__ __forceinline__ void sh_basis(float x, float y, float z, float (&Y)[kShBasis]) {
  Y[0] = kShC0;
  Y[1] = -__fmul_rn(kShC1, y);
  Y[2] = __fmul_rn(kShC1, z);
  Y[3] = -__fmul_rn(kShC1, x);
  Y[4] = __fmul_rn(__fmul_rn(kShC2_0, x), y);
  Y[5] = __fmul_rn(__fmul_rn(kShC2_1, y), z);
  Y[6] = __fmul_rn(kShC2_2, __fsub_rn(__fsub_rn(__fmul_rn(2.f, __fmul_rn(z, z)), __fmul_rn(x, x)), __fmul_rn(y, y)));
  Y[7] = __fmul_rn(__fmul_rn(kShC2_3, x), z);
  Y[8] = __fmul_rn(kShC2_4, __fsub_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
}

// kW = 7: a sample's colour is clamp(sum_m cbar_{ch,m} Y_m(d / |d|), 0, 1), cbar the trilinear coefficients; the other
// six float4 of its corners are read only when alpha != 0.
template <int kW>
__global__ void __launch_bounds__(kBakedThreads) baked_render_kernel(BakedRenderParams r) {
  for (long long ray = blockIdx.x * (long long)blockDim.x + threadIdx.x; ray < r.n;
       ray += (long long)gridDim.x * blockDim.x) {
    const float* R = r.rays + ray * 8;
    const float o[3] = {R[0], R[1], R[2]}, d[3] = {R[3], R[4], R[5]};
    const float near = R[6], far = R[7];
    bool finite = true;
#pragma unroll
    for (int c = 0; c < 8; ++c) finite &= isfinite(R[c]);
    long long K = 0;
    float dt = 0.f;
    float Y[kShBasis];
    if (finite && far > near) {
      const float nd = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])),
                                            __fmul_rn(d[2], d[2])));
      if constexpr (kW > 1) sh_basis(__fdiv_rn(d[0], nd), __fdiv_rn(d[1], nd), __fdiv_rn(d[2], nd), Y);
      dt = __fdiv_rn(r.step, nd);
      if (dt > 0.f && isfinite(dt)) {
        const float kf = floorf(__fdiv_rn(__fsub_rn(far, near), dt));
        K = kf >= static_cast<float>(kBakedMaxSamples) ? kBakedMaxSamples : static_cast<long long>(kf);
      }
    }
    float T = 1.f, cr = 0.f, cg = 0.f, cb = 0.f, cd = 0.f, cw = 0.f;
    int last_key = -1, slot = -1;
    for (long long k = 0; k < K;) {
      float u[3], t;
      const int key = baked_key(r, o, d, near, dt, k, u, t);
      if (key != last_key) {
        last_key = key;
        const int kx = ((key >> 20) & 1023) - 1, ky = ((key >> 10) & 1023) - 1, kz = (key & 1023) - 1;
        const bool in = kx >= 0 && kx < r.nb && ky >= 0 && ky < r.nb && kz >= 0 && kz < r.nb;
        slot = in ? __ldg(r.map + (static_cast<long long>(ky) * r.nb + kx) * r.nb + kz) : -1;
      }
      if (slot < 0) {
        k = baked_skip(r, o, d, near, dt, k, K, key);
        continue;
      }
      // the cell: x takes j (axis 1), y takes i (axis 0), z takes k (axis 2)
      int cell[3];
      float f[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        cell[a] = min(static_cast<int>(u[a]), r.N - 2);
        f[a] = __fsub_rn(u[a], static_cast<float>(cell[a]));
      }
      const float4* p = r.data + (static_cast<long long>(slot) * kBakedPoints +
                                  baked_point(cell[1] & 7, cell[0] & 7, cell[2] & 7)) * kW;
      float4 v[8];
#pragma unroll
      for (int c = 0; c < 8; ++c)   // c: bit 2 along i (y), bit 1 along j (x), bit 0 along k (z)
        v[c] = __ldg(p + baked_point(c >> 2, (c >> 1) & 1, c & 1) * kW);
      float val[4];
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) {
        float x[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float4 w = v[c];
          x[c] = ch == 0 ? w.x : ch == 1 ? w.y : ch == 2 ? w.z : baked_sigma(w.w);
        }
        const float z00 = baked_lerp(x[0], x[1], f[2]), z01 = baked_lerp(x[2], x[3], f[2]);
        const float z10 = baked_lerp(x[4], x[5], f[2]), z11 = baked_lerp(x[6], x[7], f[2]);
        val[ch] = baked_lerp(baked_lerp(z00, z01, f[0]), baked_lerp(z10, z11, f[0]), f[1]);
      }
      const float alpha = __fsub_rn(1.f, expf(-__fmul_rn(val[3], r.step)));
      if (alpha != 0.f) {         // alpha = 0 leaves every sum and T as they are
        if constexpr (kW > 1) {
          float col[3];
#pragma unroll
          for (int ch = 0; ch < 3; ++ch) col[ch] = __fmul_rn(val[ch], Y[0]);
#pragma unroll
          for (int w4 = 1; w4 < kW; ++w4) {
#pragma unroll
            for (int c = 0; c < 8; ++c) v[c] = __ldg(p + baked_point(c >> 2, (c >> 1) & 1, c & 1) * kW + w4);
#pragma unroll
            for (int l = 0; l < 4; ++l) {
              float x[8];
#pragma unroll
              for (int c = 0; c < 8; ++c) x[c] = l == 0 ? v[c].x : l == 1 ? v[c].y : l == 2 ? v[c].z : v[c].w;
              const float z00 = baked_lerp(x[0], x[1], f[2]), z01 = baked_lerp(x[2], x[3], f[2]);
              const float z10 = baked_lerp(x[4], x[5], f[2]), z11 = baked_lerp(x[6], x[7], f[2]);
              const float cb = baked_lerp(baked_lerp(z00, z01, f[0]), baked_lerp(z10, z11, f[0]), f[1]);
              const int e = 4 * (w4 - 1) + l;      // coefficient 1 + e / 3 of channel e % 3
              col[e % 3] = __fmaf_rn(cb, Y[1 + e / 3], col[e % 3]);
            }
          }
#pragma unroll
          for (int ch = 0; ch < 3; ++ch) val[ch] = fminf(fmaxf(col[ch], 0.f), 1.f);
        }
        const float w = __fmul_rn(alpha, T);
        cr = __fadd_rn(cr, __fmul_rn(w, val[0]));
        cg = __fadd_rn(cg, __fmul_rn(w, val[1]));
        cb = __fadd_rn(cb, __fmul_rn(w, val[2]));
        cd = __fadd_rn(cd, __fmul_rn(w, t));
        cw = __fadd_rn(cw, w);
        T = __fmul_rn(T, __fsub_rn(1.f, alpha));
        if (T < r.eps) break;
      }
      ++k;
    }
    const float back = __fmul_rn(r.white_back, __fsub_rn(1.f, cw));
    r.rgb[ray * 3 + 0] = __fadd_rn(cr, back);
    r.rgb[ray * 3 + 1] = __fadd_rn(cg, back);
    r.rgb[ray * 3 + 2] = __fadd_rn(cb, back);
    r.depth[ray] = cd;
    r.opacity[ray] = cw;
  }
}

}  // namespace nerfb200
