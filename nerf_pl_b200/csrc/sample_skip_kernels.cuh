// Per-sample empty-space skipping (DESIGN.md "Skipping empty samples"), at render time and in training.  The rays of
// a pass are rendered sample by sample: a sample whose point lies in no occupied cell gets sigma = 0 and is not
// evaluated, the others go through the MLP as compacted rows (mlp_forward_kernel's compacted-sample mode, or its
// training mode).  Everything else reuses the render kernel's device functions (z_base, composite_ray,
// pdf_to_cdf_ray, inverse_cdf, merge_rank, dir_embed_term, dir_bias), so an evaluated sample has the fused kernel's
// sigma / rgb bit for bit and a ray with nothing to skip renders as render_rays renders it.
//
// One set of per-ray kernels serves both callers; the render path is the training path without the direction-row
// store.  With perturb > 0 a pass jitters the coarse depths and keeps them in the workspace (zc), with noise_std > 0
// it adds noise to the evaluated sigma, and the resampling uses the render kernel's sorted random u; training
// (train_skip_kernels.cuh) also writes the fp16 direction rows its MLP saves for the backward, rendering has
// test_time and live_flag.  A render in chunks keys a ray's in-kernel random numbers by its index in the whole call.
//
// Per chunk of rays:  classify (coarse) -> scan -> [emit -> direction bias -> coarse MLP] -> coarse stage
// (composite, resample, merge, classify fine) -> scan -> [emit -> fine MLP] -> fine stage (composite).
// The per-ray kernels run one warp per ray in grid-stride order, so no result depends on the launch shape.
#pragma once
#include "aux_kernels.cuh"
#include "occupancy_kernels.cuh"

namespace nerfb200 {

constexpr int kSkipMaskWords = kMaxSf / 32;   // evaluated-sample bits of one ray and pass: bit i of word w = sample 32 w + i
constexpr int kSkipWarps = 4;                 // rays (warps) per block of the per-ray kernels

struct SkipParams {
  const float* rays;            // (n, 8) [o, d, near, far], 16-byte aligned
  int n;
  const uint8_t* live_flag;     // nullable: a ray whose flag is 0 has every sample skipped
  int Sc, K, use_disp, white_back, test_time;
  // training's randomness: perturb = noise_std = 0 is the render path
  float perturb, noise_std;
  const float* perturb_rand;    // (n, Sc), null with perturb = 0 or in-kernel random numbers
  const float* noise[2];        // (n, Sc) / (n, Sf), null with noise_std = 0
  const float* u_rand;          // (n, K), as perturb_rand
  unsigned long long rng_seed;  // as RenderParams
  int rng_in_kernel;
  SkipGrid grid;
  const uint8_t* net[2];        // packed images (coarse, fine)
  // workspace
  uint32_t* mask[2];            // (n, kSkipMaskWords) evaluated samples of the coarse / fine pass
  int* cnt;                     // (n) evaluated samples of the current pass
  long long* ofs;               // (n + 1) exclusive scan of cnt; ofs[n] the total
  float* zc;                    // nullable (n, Sc) coarse depths, stored by the classification; null: z_base's
  float* zf;                    // (n, Sf) merged fine depths
  float* dirbias;               // (n, kSkipDirStride)
  __half* dirrow;               // nullable (n, 64) fp16 direction rows of the training MLP
  int* row_ray;                 // (rows) compacted samples: ray, depth
  float* row_z;
  const float* mlp_out;         // (rows, 4) rgb + sigma, or (rows) sigma
  // results, nullable as render_rays' (RenderParams)
  float* rgb_coarse; float* depth_coarse; float* opacity_coarse;
  float* rgb_fine; float* depth_fine; float* opacity_fine;
  float* z_coarse; float* z_fine; float* weights_coarse; float* weights_fine;
  float* samples[2];            // optional (n, S, 4): rgb + sigma of every sample of the pass, 0 where skipped
  uint32_t ray0;                // in-kernel random numbers: ray r of the launch draws as ray ray0 + r (a chunk's start)
};

__device__ __forceinline__ unsigned long long skip_key(const SkipParams& p) {
  return p.rng_in_kernel == 2 ? *reinterpret_cast<const unsigned long long*>(p.rng_seed) : p.rng_seed;
}

// Coarse depths of ray r, sample i: render_rays_kernel's setup_group expression (models/rendering.py:189-204), the
// uniform from the tensor or from Philox stream 0 with the render kernel's counters; z_base with perturb = 0.
__device__ __forceinline__ float skip_z(const SkipParams& p, int r, int i, float nr, float fr) {
  const int Sc = p.Sc;
  const bool ud = p.use_disp != 0;
  float z = z_base(nr, fr, i, Sc, ud);
  if (p.perturb > 0.f) {
    const float zl = (i > 0) ? z_base(nr, fr, i - 1, Sc, ud) : z;
    const float zu = (i < Sc - 1) ? z_base(nr, fr, i + 1, Sc, ud) : z;
    const float lower = (i > 0) ? __fmul_rn(0.5f, __fadd_rn(zl, z)) : z;
    const float upper = (i < Sc - 1) ? __fmul_rn(0.5f, __fadd_rn(z, zu)) : z;
    const float pu = p.rng_in_kernel
                         ? philox_uniform(skip_key(p), static_cast<uint32_t>(r) + p.ray0, static_cast<uint32_t>(i), 0u)
                         : __ldg(p.perturb_rand + static_cast<long long>(r) * Sc + i);
    const float pr = __fmul_rn(p.perturb, pu);
    z = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), pr));
  }
  return z;
}

__device__ __forceinline__ bool mask_bit(const uint32_t* m, int i) { return (m[i >> 5] >> (i & 31)) & 1u; }

// Whether the point x lies in the closed box of an occupied cell of its level: the smallest level whose closed box
// [0, M]^3 holds its grid coordinates.  In grid coordinates, compared in double; a coordinate on a cell boundary
// belongs to both cells, so a point on a shared face, edge or corner checks every cell that touches it.  Outside
// the last level's box (and for a NaN) nothing is occupied.
__device__ __forceinline__ bool point_occupied(const SkipGrid& g, const float x[3]) {
  const double Md = static_cast<double>(g.M);
  double v[3];
  int k = 0;
#pragma unroll 1
  for (;; ++k) {
    if (k == g.levels) return false;
    bool in = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      v[a] = (static_cast<double>(x[a]) - g.lo[k][a]) * g.scale[k][a];
      in &= v[a] >= 0.0 && v[a] <= Md;
    }
    if (in) break;
  }
  const uint32_t* bits = g.bits + k * g.words;
  long long c0[3], c1[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double f = floor(v[a]);
    const long long fl = static_cast<long long>(f);
    c1[a] = fl < g.M - 1 ? fl : g.M - 1;
    c0[a] = (f == v[a] && fl > 0) ? fl - 1 : c1[a];
  }
  for (long long cz = c0[2]; cz <= c1[2]; ++cz)
    for (long long cy = c0[1]; cy <= c1[1]; ++cy)
      for (long long cx = c0[0]; cx <= c1[0]; ++cx) {
        const long long c = (cz * g.M + cy) * g.M + cx;
        if ((__ldg(bits + (c >> 5)) >> (c & 31)) & 1u) return true;
      }
  return false;
}

// The ray's values and |d| as the render kernel computes them; `plain` is set when the ray is evaluated at every
// sample of both passes: a non-finite value or far <= near.
struct SkipRay { float o[3], d[3], near, far, dnorm; bool plain; };
__device__ __forceinline__ SkipRay load_skip_ray(const SkipParams& p, int r) {
  SkipRay s;
  const float* v = p.rays + static_cast<long long>(r) * 8;
  bool finite = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    s.o[a] = __ldg(v + a);
    s.d[a] = __ldg(v + 3 + a);
    finite &= isfinite(s.o[a]) && isfinite(s.d[a]);
  }
  s.near = __ldg(v + 6);
  s.far = __ldg(v + 7);
  finite &= isfinite(s.near) && isfinite(s.far);
  s.plain = !finite || !(s.far > s.near);
  s.dnorm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(s.d[0], s.d[0]), __fmul_rn(s.d[1], s.d[1])), __fmul_rn(s.d[2], s.d[2])));
  return s;
}

// Classify the S samples z[0..S) of one ray by one warp: mask words into m (global), returns the count.  A pass
// whose interval lengths delta_i |d| (delta_{S-1} = 1e10, composite_ray's) are not all finite is evaluated at every
// sample: sigma = 0 would not give such a sample a zero weight.
__device__ __forceinline__ int classify_ray(const SkipParams& p, const SkipRay& s, int r, int lane, int S, const float* z,
                                            uint32_t* m) {
  const bool dead = p.live_flag != nullptr && __ldg(p.live_flag + r) == 0;
  bool bad = false;
  for (int i = lane; i < S; i += 32) {
    const float delta = (i < S - 1) ? __fsub_rn(z[i + 1], z[i]) : 1e10f;
    bad |= !isfinite(__fmul_rn(delta, s.dnorm));
  }
  const bool all = s.plain || __any_sync(0xffffffffu, bad);
  int count = 0;
  for (int w = 0; w < (S >> 5); ++w) {
    const int i = 32 * w + lane;
    bool ev = false;
    if (!dead) {
      if (all) {
        ev = true;
      } else {
        float x[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) x[c] = __fadd_rn(s.o[c], __fmul_rn(s.d[c], z[i]));   // encode_row's point
        ev = point_occupied(p.grid, x);
      }
    }
    const uint32_t b = __ballot_sync(0xffffffffu, ev);
    if (lane == 0) m[w] = b;
    count += __popc(b);
  }
  return count;
}

// Shared memory of one warp of the per-ray stages.
struct alignas(16) SkipWarpScratch {
  float zc[kMaxSc];
  float zf[kMaxSf];
  float sigma[kMaxSf];          // overwritten in place by the weights
  float rgb[3][kMaxSf];
  float cdf[kMaxSc];
  float znew[kMaxImp];
};

// sigma (and rgb) of the S samples of a ray from the compacted MLP rows, 0 where skipped.
__device__ __forceinline__ void expand_ray(const SkipParams& p, int r, int lane, int S, const uint32_t* m, bool want_rgb,
                                           SkipWarpScratch& w, float* samples) {
  long long pos = p.ofs[r];
  for (int k = 0; k < (S >> 5); ++k) {
    const uint32_t b = m[k];
    const int i = 32 * k + lane;
    float sg = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f;
    if ((b >> lane) & 1u) {
      const long long row = pos + __popc(b & ((1u << lane) - 1u));
      if (want_rgb) {
        const float4 v = *reinterpret_cast<const float4*>(p.mlp_out + row * 4);
        c0 = v.x; c1 = v.y; c2 = v.z; sg = v.w;
      } else {
        sg = p.mlp_out[row];
      }
    }
    w.sigma[i] = sg;
    w.rgb[0][i] = c0; w.rgb[1][i] = c1; w.rgb[2][i] = c2;
    if (samples != nullptr)
      *reinterpret_cast<float4*>(samples + (static_cast<long long>(r) * S + i) * 4) = make_float4(c0, c1, c2, sg);
    pos += __popc(b);
  }
}

// sigma + noise of the evaluated samples of one pass (composite_ray's expression); skipped samples keep sigma = 0.
__device__ __forceinline__ void add_noise(const SkipParams& p, int pass, long long r, int lane, int S, const uint32_t* m,
                                          float* sigma) {
  if (p.noise_std <= 0.f) return;
  const float* nz = p.noise[pass] + r * S;
  for (int i = lane; i < S; i += 32)
    if (mask_bit(m, i)) sigma[i] = __fadd_rn(sigma[i], __fmul_rn(__ldg(nz + i), p.noise_std));
}

// The results of pass `pass` of ray r: the weights (composite_ray left them in wts), the opacity and, with want_rgb,
// the colour (on the white background with white_back) and the depth.
__device__ __forceinline__ void store_pass(const SkipParams& p, int pass, long long r, int lane, int S, const RayOut& o,
                                           bool want_rgb, const float* wts) {
  float* const weights = pass ? p.weights_fine : p.weights_coarse;
  if (weights != nullptr)
    for (int i = lane; i < S; i += 32) weights[r * S + i] = wts[i];
  if (lane == 0) {
    const float add = (p.white_back != 0) ? __fsub_rn(1.f, o.opac) : 0.f;
    (pass ? p.opacity_fine : p.opacity_coarse)[r] = o.opac;
    if (want_rgb) {
      float* const rgb = pass ? p.rgb_fine : p.rgb_coarse;
      rgb[3 * r + 0] = o.r + add;
      rgb[3 * r + 1] = o.g + add;
      rgb[3 * r + 2] = o.b + add;
      (pass ? p.depth_fine : p.depth_coarse)[r] = o.depth;
    }
  }
}

// Coarse classification: the coarse depths (skip_z; stored to zc and z_coarse when given), the count per ray and,
// with dirrow, the fp16 direction row the training MLP stores for the direction-slice wgrad (Embedding(3, 4)(d) as
// the render kernel computes it, columns 27..63 zero).
__global__ void __launch_bounds__(kSkipWarps * 32) skip_classify_kernel(SkipParams p) {
  __shared__ float zs[kSkipWarps][kMaxSc];
  __shared__ float de[kSkipWarps][28];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // n <= 2^22 (samples_shape_ok): int ray indices keep the loop state small across z_base's division calls
  for (int r = blockIdx.x * kSkipWarps + warp; r < p.n; r += gridDim.x * kSkipWarps) {
    // the depths first: the ray's other values are not live across those calls
    const float near = __ldg(p.rays + 8 * r + 6), far = __ldg(p.rays + 8 * r + 7);
    for (int i = lane; i < p.Sc; i += 32) {
      const float z = skip_z(p, r, i, near, far);
      zs[warp][i] = z;
      if (p.zc != nullptr) p.zc[static_cast<long long>(r) * p.Sc + i] = z;
      if (p.z_coarse != nullptr) p.z_coarse[static_cast<long long>(r) * p.Sc + i] = z;
    }
    if (p.dirrow != nullptr && lane < 15) dir_embed_term(lane, p.rays + 8 * r + 3, de[warp]);
    __syncwarp();
    const int c = classify_ray(p, load_skip_ray(p, r), r, lane, p.Sc, zs[warp], p.mask[0] + r * kSkipMaskWords);
    if (lane == 0) p.cnt[r] = c;
    if (p.dirrow != nullptr) {
      const float lo = (2 * lane < 27) ? de[warp][2 * lane] : 0.f, hi = (2 * lane + 1 < 27) ? de[warp][2 * lane + 1] : 0.f;
      reinterpret_cast<__half2*>(p.dirrow + static_cast<long long>(r) * 64)[lane] = __floats2half2_rn(lo, hi);
    }
    __syncwarp();
  }
}

// The rows of pass `pass`: evaluated sample i of ray r goes to row ofs[r] + (evaluated samples of r before i), so
// the rows are ray-major and in depth-index order.  The depths are zf's, or zc's (z_base's without zc) for pass 0.
__global__ void __launch_bounds__(kSkipWarps * 32) skip_emit_kernel(SkipParams p, int pass) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = pass ? p.Sc + p.K : p.Sc;
  const float* zb = pass ? p.zf : p.zc;
  for (long long r = static_cast<long long>(blockIdx.x) * kSkipWarps + warp; r < p.n;
       r += static_cast<long long>(gridDim.x) * kSkipWarps) {
    const uint32_t* m = p.mask[pass] + r * kSkipMaskWords;
    long long pos = p.ofs[r];
    const float near = __ldg(p.rays + r * 8 + 6), far = __ldg(p.rays + r * 8 + 7);
    for (int k = 0; k < (S >> 5); ++k) {
      const uint32_t b = m[k];
      const int i = 32 * k + lane;
      if ((b >> lane) & 1u) {
        const long long row = pos + __popc(b & ((1u << lane) - 1u));
        p.row_ray[row] = static_cast<int>(r);
        p.row_z[row] = zb != nullptr ? zb[r * S + i] : z_base(near, far, i, S, p.use_disp != 0);
      }
      pos += __popc(b);
    }
  }
}

// The render kernel's per-ray direction bias of the networks in [pass0, pass1), one block of kDirW threads per ray.
__global__ void __launch_bounds__(kDirW) skip_dir_bias_kernel(SkipParams p, int pass0, int pass1) {
  __shared__ float direnc[28];
  const int t = threadIdx.x;
  for (long long r = blockIdx.x; r < p.n; r += gridDim.x) {
    if (t < 15) dir_embed_term(t, p.rays + r * 8 + 3, direnc);
    __syncthreads();
    for (int pass = pass0; pass < pass1; ++pass) {
      const float* f32 = reinterpret_cast<const float*>(p.net[pass] + kHalfRegionBytes);
      p.dirbias[r * kSkipDirStride + pass * kDirW + t] = dir_bias(f32, __ldg(f32 + kF32Bias + 8 * 256 + t), t, direnc);
    }
    __syncthreads();
  }
}

// Coarse stage of one ray per warp: expand, noise, composite, results; then (K > 0) the inverse-CDF resampling with
// the render kernel's u (sorted random numbers, linspace with perturb = 0), the merge and the fine classification.
// The scratch allows 9 blocks per SM; the register bound keeps the training branches from allowing fewer.
__global__ void __launch_bounds__(kSkipWarps * 32, 9) skip_coarse_stage_kernel(SkipParams p) {
  __shared__ SkipWarpScratch scr[kSkipWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  SkipWarpScratch& w = scr[warp];
  const int Sc = p.Sc, K = p.K, Sf = Sc + K;
  const bool want_rgb = p.test_time == 0;
  for (long long r = static_cast<long long>(blockIdx.x) * kSkipWarps + warp; r < p.n;
       r += static_cast<long long>(gridDim.x) * kSkipWarps) {
    const uint32_t* m = p.mask[0] + r * kSkipMaskWords;
    if (p.zc != nullptr) {
      for (int i = lane; i < Sc; i += 32) w.zc[i] = p.zc[r * Sc + i];
    } else {
      const float near = __ldg(p.rays + r * 8 + 6), far = __ldg(p.rays + r * 8 + 7);
      for (int i = lane; i < Sc; i += 32) w.zc[i] = z_base(near, far, i, Sc, p.use_disp != 0);
    }
    expand_ray(p, static_cast<int>(r), lane, Sc, m, want_rgb, w, p.samples[0]);
    add_noise(p, 0, r, lane, Sc, m, w.sigma);
    __syncwarp();
    const RayOut o = composite_ray(lane, Sc, w.zc, w.sigma, w.rgb[0], w.rgb[1], w.rgb[2], nullptr, 0.f,
                                   load_skip_ray(p, static_cast<int>(r)).dnorm, want_rgb, w.sigma);
    __syncwarp();
    store_pass(p, 0, r, lane, Sc, o, want_rgb, w.sigma);
    if (K == 0) continue;
    pdf_to_cdf_ray(lane, Sc, w.sigma, w.cdf);
    // u: render_rays_kernel's ranking (a u's slot is the number of u's before it in torch.sort's order); the u's
    // are parked in w.zf, which the merge overwrites below
    if (p.perturb > 0.f) {
      const unsigned long long key = p.rng_in_kernel ? skip_key(p) : 0ull;
      for (int j = lane; j < K; j += 32)
        w.zf[j] = p.rng_in_kernel ? philox_uniform(key, static_cast<uint32_t>(r) + p.ray0, static_cast<uint32_t>(j), 1u)
                                  : __ldg(p.u_rand + r * K + j);
    }
    __syncwarp();
    for (int j = lane; j < K; j += 32) {
      float uj;
      int slot = j;
      if (p.perturb > 0.f) {
        uj = w.zf[j];
        slot = 0;
        if (p.rng_in_kernel) {       // philox_uniform is never NaN
          for (int q = 0; q < K; ++q) {
            const float uq = w.zf[q];
            slot += (uq < uj) || (uq == uj && q < j);
          }
        } else {
          for (int q = 0; q < K; ++q) {
            const float uq = w.zf[q];
            slot += sort_before(uq, uj) || (sort_tied(uq, uj) && q < j);
          }
        }
      } else {
        uj = linspace01(j, K);
      }
      w.znew[slot] = inverse_cdf(Sc, w.zc, w.cdf, uj);
    }
    __syncwarp();
    bool inv = false;
    for (int i = lane; i < Sf; i += 32) inv |= merge_flag(i, Sc, w.zc, w.znew);
    const bool any_inv = __any_sync(0xffffffffu, inv);
    for (int i = lane; i < Sf; i += 32) {
      const float v = (i < Sc) ? w.zc[i] : w.znew[i - Sc];
      w.zf[merge_rank(i, v, Sc, K, w.zc, w.znew, any_inv)] = v;
    }
    __syncwarp();
    for (int i = lane; i < Sf; i += 32) {
      p.zf[r * Sf + i] = w.zf[i];
      if (p.z_fine != nullptr) p.z_fine[r * Sf + i] = w.zf[i];
    }
    // reloaded here rather than kept live across the resampling's division calls
    const int c = classify_ray(p, load_skip_ray(p, static_cast<int>(r)), static_cast<int>(r), lane, Sf, w.zf,
                               p.mask[1] + r * kSkipMaskWords);
    if (lane == 0) p.cnt[r] = c;
    __syncwarp();
  }
}

// Fine stage of one ray per warp: expand, noise and composite the merged depths.
__global__ void __launch_bounds__(kSkipWarps * 32) skip_fine_stage_kernel(SkipParams p) {
  __shared__ SkipWarpScratch scr[kSkipWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  SkipWarpScratch& w = scr[warp];
  const int Sf = p.Sc + p.K;
  for (long long r = static_cast<long long>(blockIdx.x) * kSkipWarps + warp; r < p.n;
       r += static_cast<long long>(gridDim.x) * kSkipWarps) {
    const uint32_t* m = p.mask[1] + r * kSkipMaskWords;
    for (int i = lane; i < Sf; i += 32) w.zf[i] = p.zf[r * Sf + i];
    expand_ray(p, static_cast<int>(r), lane, Sf, m, true, w, p.samples[1]);
    add_noise(p, 1, r, lane, Sf, m, w.sigma);
    __syncwarp();
    const RayOut o = composite_ray(lane, Sf, w.zf, w.sigma, w.rgb[0], w.rgb[1], w.rgb[2], nullptr, 0.f,
                                   load_skip_ray(p, static_cast<int>(r)).dnorm, true, w.sigma);
    __syncwarp();
    store_pass(p, 1, r, lane, Sf, o, true, w.sigma);
    __syncwarp();
  }
}

}  // namespace nerfb200
