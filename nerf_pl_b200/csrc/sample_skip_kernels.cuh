// Per-sample empty-space skipping at render time (DESIGN.md "Skipping empty samples").  The live rays of a cull
// (occupancy_kernels.cuh) are rendered sample by sample: a sample whose point lies in no occupied cell gets
// sigma = 0 and is not evaluated, the others go through the MLP as compacted rows (mlp_forward_kernel's
// compacted-sample mode).  Everything else reuses the render kernel's device functions (z_base, composite_ray,
// pdf_to_cdf_ray, inverse_cdf, merge_rank, dir_embed_term, dir_bias), so an evaluated sample has the fused kernel's
// sigma / rgb bit for bit and a ray with nothing to skip renders as render_rays renders it.
//
// Per chunk of rays:  classify (coarse) -> scan -> [emit -> direction bias -> coarse MLP] -> coarse stage
// (composite, resample, merge, classify fine) -> scan -> [emit -> fine MLP] -> fine stage (composite).
// The per-ray kernels run one warp per ray in grid-stride order, so no result depends on the launch shape.
#pragma once
#include "aux_kernels.cuh"

namespace nerfb200 {

constexpr int kSkipMaskWords = kMaxSf / 32;   // evaluated-sample bits of one ray and pass: bit i of word w = sample 32 w + i
constexpr int kSkipWarps = 4;                 // rays (warps) per block of the per-ray kernels

struct SkipGrid {
  const uint32_t* bits;   // occupancy bit field (occupancy_kernels.cuh: cell (cz * M + cy) * M + cx)
  long long M;            // cells per axis
  double lo[3], scale[3]; // grid coordinate g = (x - lo) * scale; the box is [0, M]^3
};

struct SkipParams {
  const float* rays;            // (n, 8) [o, d, near, far], 16-byte aligned
  int n;
  const uint8_t* live_flag;     // nullable: a ray whose flag is 0 has every sample skipped
  int Sc, K, use_disp, white_back, test_time;
  SkipGrid grid;
  const uint8_t* net[2];        // packed images (coarse, fine)
  // workspace
  uint32_t* mask[2];            // (n, kSkipMaskWords) evaluated samples of the coarse / fine pass
  int* cnt;                     // (n) evaluated samples of the current pass
  long long* ofs;               // (n + 1) exclusive scan of cnt; ofs[n] the total
  float* zf;                    // (n, Sf) merged fine depths
  float* dirbias;               // (n, kSkipDirStride)
  int* row_ray;                 // (rows) compacted samples: ray, depth
  float* row_z;
  const float* mlp_out;         // (rows, 4) rgb + sigma, or (rows) sigma
  // results, nullable as render_rays' (RenderParams)
  float* rgb_coarse; float* depth_coarse; float* opacity_coarse;
  float* rgb_fine; float* depth_fine; float* opacity_fine;
  float* z_fine; float* weights_coarse; float* weights_fine;
  float* samples[2];            // optional (n, S, 4): rgb + sigma of every sample of the pass, 0 where skipped
};

// Whether the point x lies in the closed box of an occupied cell.  In grid coordinates, compared in double; a
// coordinate on a cell boundary belongs to both cells, so a point on a shared face, edge or corner checks every
// cell that touches it.  Outside the box [0, M]^3 (and for a NaN) nothing is occupied.
__device__ __forceinline__ bool point_occupied(const SkipGrid& g, const float x[3]) {
  long long c0[3], c1[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double v = (static_cast<double>(x[a]) - g.lo[a]) * g.scale[a];
    if (!(v >= 0.0 && v <= static_cast<double>(g.M))) return false;
    const double f = floor(v);
    const long long fl = static_cast<long long>(f);
    c1[a] = fl < g.M - 1 ? fl : g.M - 1;
    c0[a] = (f == v && fl > 0) ? fl - 1 : c1[a];
  }
  for (long long cz = c0[2]; cz <= c1[2]; ++cz)
    for (long long cy = c0[1]; cy <= c1[1]; ++cy)
      for (long long cx = c0[0]; cx <= c1[0]; ++cx) {
        const long long c = (cz * g.M + cy) * g.M + cx;
        if ((__ldg(g.bits + (c >> 5)) >> (c & 31)) & 1u) return true;
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

// Coarse classification: the coarse depths of render_rays (z_base, perturb = 0), count per ray.
__global__ void __launch_bounds__(kSkipWarps * 32) skip_classify_kernel(SkipParams p) {
  __shared__ float zs[kSkipWarps][kMaxSc];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // n <= 2^22 (nerfb200_render_samples): int ray indices keep the loop state small across z_base's division calls
  for (int r = blockIdx.x * kSkipWarps + warp; r < p.n; r += gridDim.x * kSkipWarps) {
    // the depths first: the ray's other values are not live across those calls
    const float near = __ldg(p.rays + 8 * r + 6), far = __ldg(p.rays + 8 * r + 7);
    for (int i = lane; i < p.Sc; i += 32) zs[warp][i] = z_base(near, far, i, p.Sc, p.use_disp != 0);
    __syncwarp();
    const int c = classify_ray(p, load_skip_ray(p, r), r, lane, p.Sc, zs[warp], p.mask[0] + r * kSkipMaskWords);
    if (lane == 0) p.cnt[r] = c;
    __syncwarp();
  }
}

// The rows of pass `pass`: evaluated sample i of ray r goes to row ofs[r] + (evaluated samples of r before i), so
// the rows are ray-major and in depth-index order.
__global__ void __launch_bounds__(kSkipWarps * 32) skip_emit_kernel(SkipParams p, int pass) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = pass ? p.Sc + p.K : p.Sc;
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
        p.row_z[row] = pass ? p.zf[r * S + i] : z_base(near, far, i, S, p.use_disp != 0);
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

// Coarse stage of one ray per warp: expand, composite, results; then (N_importance > 0) the deterministic inverse-CDF
// resampling, the merge and the classification of the fine samples.
__global__ void __launch_bounds__(kSkipWarps * 32) skip_coarse_stage_kernel(SkipParams p) {
  __shared__ SkipWarpScratch scr[kSkipWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  SkipWarpScratch& w = scr[warp];
  const int Sc = p.Sc, K = p.K, Sf = Sc + K;
  const bool want_rgb = p.test_time == 0;
  for (long long r = static_cast<long long>(blockIdx.x) * kSkipWarps + warp; r < p.n;
       r += static_cast<long long>(gridDim.x) * kSkipWarps) {
    const float near = __ldg(p.rays + r * 8 + 6), far = __ldg(p.rays + r * 8 + 7);
    for (int i = lane; i < Sc; i += 32) w.zc[i] = z_base(near, far, i, Sc, p.use_disp != 0);
    expand_ray(p, static_cast<int>(r), lane, Sc, p.mask[0] + r * kSkipMaskWords, want_rgb, w, p.samples[0]);
    __syncwarp();
    const RayOut o = composite_ray(lane, Sc, w.zc, w.sigma, w.rgb[0], w.rgb[1], w.rgb[2], nullptr, 0.f,
                                   load_skip_ray(p, static_cast<int>(r)).dnorm, want_rgb, w.sigma);
    __syncwarp();
    if (p.weights_coarse != nullptr)
      for (int i = lane; i < Sc; i += 32) p.weights_coarse[r * Sc + i] = w.sigma[i];
    if (lane == 0) {
      const float add = (p.white_back != 0) ? __fsub_rn(1.f, o.opac) : 0.f;
      p.opacity_coarse[r] = o.opac;
      if (want_rgb) {
        p.rgb_coarse[3 * r + 0] = o.r + add;
        p.rgb_coarse[3 * r + 1] = o.g + add;
        p.rgb_coarse[3 * r + 2] = o.b + add;
        p.depth_coarse[r] = o.depth;
      }
    }
    if (K == 0) continue;
    pdf_to_cdf_ray(lane, Sc, w.sigma, w.cdf);
    __syncwarp();
    for (int j = lane; j < K; j += 32) w.znew[j] = inverse_cdf(Sc, w.zc, w.cdf, linspace01(j, K));
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

// Fine stage of one ray per warp: expand and composite the merged depths.
__global__ void __launch_bounds__(kSkipWarps * 32) skip_fine_stage_kernel(SkipParams p) {
  __shared__ SkipWarpScratch scr[kSkipWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  SkipWarpScratch& w = scr[warp];
  const int Sf = p.Sc + p.K;
  for (long long r = static_cast<long long>(blockIdx.x) * kSkipWarps + warp; r < p.n;
       r += static_cast<long long>(gridDim.x) * kSkipWarps) {
    const SkipRay s = load_skip_ray(p, static_cast<int>(r));
    for (int i = lane; i < Sf; i += 32) w.zf[i] = p.zf[r * Sf + i];
    expand_ray(p, static_cast<int>(r), lane, Sf, p.mask[1] + r * kSkipMaskWords, true, w, p.samples[1]);
    __syncwarp();
    const RayOut o = composite_ray(lane, Sf, w.zf, w.sigma, w.rgb[0], w.rgb[1], w.rgb[2], nullptr, 0.f, s.dnorm, true,
                                   w.sigma);
    __syncwarp();
    if (p.weights_fine != nullptr)
      for (int i = lane; i < Sf; i += 32) p.weights_fine[r * Sf + i] = w.sigma[i];
    if (lane == 0) {
      const float add = (p.white_back != 0) ? __fsub_rn(1.f, o.opac) : 0.f;
      p.opacity_fine[r] = o.opac;
      p.rgb_fine[3 * r + 0] = o.r + add;
      p.rgb_fine[3 * r + 1] = o.g + add;
      p.rgb_fine[3 * r + 2] = o.b + add;
      p.depth_fine[r] = o.depth;
    }
    __syncwarp();
  }
}

}  // namespace nerfb200
