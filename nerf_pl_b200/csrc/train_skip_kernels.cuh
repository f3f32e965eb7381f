// The training step with empty samples skipped (DESIGN.md "Training with empty samples skipped").  The rule of
// sample_skip_kernels.cuh carried into training: the coarse depths are the render kernel's stratified depths with the
// perturb jitter, an evaluated sample gets the network's sigma + noise * noise_std, a skipped one sigma = 0 without
// noise (weight exactly 0, no gradient), and the resampling uses the render kernel's sorted random u.  The compacted
// rows go through mlp_forward_kernel<true, true>, which leaves in one NeRF.forward training workspace per network what
// nerfb200_nerf_backward's tail reads; the backward starts with train_skip_bwd_kernel, the compositing backward over
// the sparse sample lists.
//
// Forward:  classify (perturbed depths, direction rows) -> scan -> [emit -> direction bias -> coarse MLP] -> coarse
// stage (noise, composite, random resampling, merge, classify fine) -> scan -> [emit -> fine MLP] -> fine stage ->
// loss (mse_psnr_kernel).  One warp per ray in grid-stride order: no result depends on the launch shape.
#pragma once
#include "sample_skip_kernels.cuh"

namespace nerfb200 {

struct TrainSkipParams {
  SkipParams s;                 // s.ofs: the offsets of the pass a launch works on (ofs[pass] below)
  float perturb, noise_std;
  const float* perturb_rand;    // (n, Sc), null with perturb = 0 or in-kernel random numbers
  const float* noise[2];        // (n, Sc) / (n, Sf), null with noise_std = 0
  const float* u_rand;          // (n, K), as perturb_rand
  unsigned long long rng_seed;  // as RenderParams
  int rng_in_kernel;
  float* zc;                    // (n, Sc) coarse depths (workspace)
  __half* dirrow;               // (n, 64) fp16 direction rows (workspace)
  long long* ofs[2];            // (n + 1) exclusive scans of the evaluated samples of each pass (workspace)
  float* z_coarse;              // optional (n, Sc) copy of the coarse depths
};

__device__ __forceinline__ unsigned long long train_skip_key(const TrainSkipParams& t) {
  return t.rng_in_kernel == 2 ? *reinterpret_cast<const unsigned long long*>(t.rng_seed) : t.rng_seed;
}

// Coarse depths of ray r, sample i: render_rays_kernel's setup_group expression (models/rendering.py:189-204), the
// uniform from the tensor or from Philox stream 0 with the render kernel's counters.
__device__ __forceinline__ float train_skip_z(const TrainSkipParams& t, int r, int i, float nr, float fr) {
  const int Sc = t.s.Sc;
  const bool ud = t.s.use_disp != 0;
  float z = z_base(nr, fr, i, Sc, ud);
  if (t.perturb > 0.f) {
    const float zl = (i > 0) ? z_base(nr, fr, i - 1, Sc, ud) : z;
    const float zu = (i < Sc - 1) ? z_base(nr, fr, i + 1, Sc, ud) : z;
    const float lower = (i > 0) ? __fmul_rn(0.5f, __fadd_rn(zl, z)) : z;
    const float upper = (i < Sc - 1) ? __fmul_rn(0.5f, __fadd_rn(z, zu)) : z;
    const float pu = t.rng_in_kernel ? philox_uniform(train_skip_key(t), static_cast<uint32_t>(r), static_cast<uint32_t>(i), 0u)
                                     : __ldg(t.perturb_rand + static_cast<long long>(r) * Sc + i);
    const float pr = __fmul_rn(t.perturb, pu);
    z = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), pr));
  }
  return z;
}

__device__ __forceinline__ bool mask_bit(const uint32_t* m, int i) { return (m[i >> 5] >> (i & 31)) & 1u; }

// Per ray: the coarse depths, the coarse classification and count, and the fp16 direction row the training MLP
// stores for the direction-slice wgrad (Embedding(3, 4)(d) as the render kernel computes it, columns 27..63 zero).
__global__ void __launch_bounds__(kSkipWarps * 32) train_skip_classify_kernel(TrainSkipParams t) {
  __shared__ float zs[kSkipWarps][kMaxSc];
  __shared__ float de[kSkipWarps][28];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const SkipParams& p = t.s;
  for (int r = blockIdx.x * kSkipWarps + warp; r < p.n; r += gridDim.x * kSkipWarps) {
    const float near = __ldg(p.rays + 8 * r + 6), far = __ldg(p.rays + 8 * r + 7);
    for (int i = lane; i < p.Sc; i += 32) {
      const float z = train_skip_z(t, r, i, near, far);
      zs[warp][i] = z;
      t.zc[static_cast<long long>(r) * p.Sc + i] = z;
      if (t.z_coarse != nullptr) t.z_coarse[static_cast<long long>(r) * p.Sc + i] = z;
    }
    if (lane < 15) dir_embed_term(lane, p.rays + 8 * r + 3, de[warp]);
    __syncwarp();
    const int c = classify_ray(p, load_skip_ray(p, r), r, lane, p.Sc, zs[warp], p.mask[0] + r * kSkipMaskWords);
    if (lane == 0) p.cnt[r] = c;
    const float lo = (2 * lane < 27) ? de[warp][2 * lane] : 0.f, hi = (2 * lane + 1 < 27) ? de[warp][2 * lane + 1] : 0.f;
    reinterpret_cast<__half2*>(t.dirrow + static_cast<long long>(r) * 64)[lane] = __floats2half2_rn(lo, hi);
    __syncwarp();
  }
}

// The rows of pass `pass` (skip_emit_kernel's order), depths from the workspace.
__global__ void __launch_bounds__(kSkipWarps * 32) train_skip_emit_kernel(TrainSkipParams t, int pass) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const SkipParams& p = t.s;
  const int S = pass ? p.Sc + p.K : p.Sc;
  const float* zb = pass ? p.zf : t.zc;
  for (long long r = static_cast<long long>(blockIdx.x) * kSkipWarps + warp; r < p.n;
       r += static_cast<long long>(gridDim.x) * kSkipWarps) {
    const uint32_t* m = p.mask[pass] + r * kSkipMaskWords;
    long long pos = p.ofs[r];
    for (int k = 0; k < (S >> 5); ++k) {
      const uint32_t b = m[k];
      const int i = 32 * k + lane;
      if ((b >> lane) & 1u) {
        const long long row = pos + __popc(b & ((1u << lane) - 1u));
        p.row_ray[row] = static_cast<int>(r);
        p.row_z[row] = zb[r * S + i];
      }
      pos += __popc(b);
    }
  }
}

// sigma + noise of the evaluated samples of one pass (composite_ray's expression); skipped samples keep sigma = 0.
__device__ __forceinline__ void add_noise(const TrainSkipParams& t, int pass, long long r, int lane, int S,
                                          const uint32_t* m, float* sigma) {
  if (t.noise_std <= 0.f) return;
  const float* nz = t.noise[pass] + r * S;
  for (int i = lane; i < S; i += 32)
    if (mask_bit(m, i)) sigma[i] = __fadd_rn(sigma[i], __fmul_rn(__ldg(nz + i), t.noise_std));
}

// Coarse stage of one ray per warp: expand, noise, composite, results; then (K > 0) the inverse-CDF resampling with
// the render kernel's u (sorted random numbers, linspace with perturb = 0), the merge and the fine classification.
__global__ void __launch_bounds__(kSkipWarps * 32) train_skip_coarse_stage_kernel(TrainSkipParams t) {
  __shared__ SkipWarpScratch scr[kSkipWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  SkipWarpScratch& w = scr[warp];
  const SkipParams& p = t.s;
  const int Sc = p.Sc, K = p.K, Sf = Sc + K;
  for (long long r = static_cast<long long>(blockIdx.x) * kSkipWarps + warp; r < p.n;
       r += static_cast<long long>(gridDim.x) * kSkipWarps) {
    const uint32_t* m = p.mask[0] + r * kSkipMaskWords;
    for (int i = lane; i < Sc; i += 32) w.zc[i] = t.zc[r * Sc + i];
    expand_ray(p, static_cast<int>(r), lane, Sc, m, true, w, p.samples[0]);
    add_noise(t, 0, r, lane, Sc, m, w.sigma);
    __syncwarp();
    const RayOut o = composite_ray(lane, Sc, w.zc, w.sigma, w.rgb[0], w.rgb[1], w.rgb[2], nullptr, 0.f,
                                   load_skip_ray(p, static_cast<int>(r)).dnorm, true, w.sigma);
    __syncwarp();
    if (p.weights_coarse != nullptr)
      for (int i = lane; i < Sc; i += 32) p.weights_coarse[r * Sc + i] = w.sigma[i];
    if (lane == 0) {
      const float add = (p.white_back != 0) ? __fsub_rn(1.f, o.opac) : 0.f;
      p.opacity_coarse[r] = o.opac;
      p.rgb_coarse[3 * r + 0] = o.r + add;
      p.rgb_coarse[3 * r + 1] = o.g + add;
      p.rgb_coarse[3 * r + 2] = o.b + add;
      p.depth_coarse[r] = o.depth;
    }
    if (K == 0) continue;
    pdf_to_cdf_ray(lane, Sc, w.sigma, w.cdf);
    // u: render_rays_kernel's ranking (a u's slot is the number of u's before it in torch.sort's order); the u's
    // are parked in w.zf, which the merge overwrites below
    if (t.perturb > 0.f) {
      const unsigned long long key = t.rng_in_kernel ? train_skip_key(t) : 0ull;
      for (int j = lane; j < K; j += 32)
        w.zf[j] = t.rng_in_kernel ? philox_uniform(key, static_cast<uint32_t>(r), static_cast<uint32_t>(j), 1u)
                                  : __ldg(t.u_rand + r * K + j);
    }
    __syncwarp();
    for (int j = lane; j < K; j += 32) {
      float uj;
      int slot = j;
      if (t.perturb > 0.f) {
        uj = w.zf[j];
        slot = 0;
        if (t.rng_in_kernel) {       // philox_uniform is never NaN
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
    const int c = classify_ray(p, load_skip_ray(p, static_cast<int>(r)), static_cast<int>(r), lane, Sf, w.zf,
                               p.mask[1] + r * kSkipMaskWords);
    if (lane == 0) p.cnt[r] = c;
    __syncwarp();
  }
}

// Fine stage of one ray per warp: expand, noise and composite the merged depths.
__global__ void __launch_bounds__(kSkipWarps * 32) train_skip_fine_stage_kernel(TrainSkipParams t) {
  __shared__ SkipWarpScratch scr[kSkipWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  SkipWarpScratch& w = scr[warp];
  const SkipParams& p = t.s;
  const int Sf = p.Sc + p.K;
  for (long long r = static_cast<long long>(blockIdx.x) * kSkipWarps + warp; r < p.n;
       r += static_cast<long long>(gridDim.x) * kSkipWarps) {
    const uint32_t* m = p.mask[1] + r * kSkipMaskWords;
    for (int i = lane; i < Sf; i += 32) w.zf[i] = p.zf[r * Sf + i];
    expand_ray(p, static_cast<int>(r), lane, Sf, m, true, w, p.samples[1]);
    add_noise(t, 1, r, lane, Sf, m, w.sigma);
    __syncwarp();
    const RayOut o = composite_ray(lane, Sf, w.zf, w.sigma, w.rgb[0], w.rgb[1], w.rgb[2], nullptr, 0.f,
                                   load_skip_ray(p, static_cast<int>(r)).dnorm, true, w.sigma);
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

// ------------------------------------------------------------------ sparse compositing backward
// composite_bwd_kernel's arithmetic (the fused MSE seed, white_back, noise, the ReLU mask) on one ray per warp, with
// sigma / rgb of an evaluated sample read from its compacted row and sigma = 0, rgb = 0 (no noise) for a skipped one.
// d sigma / d rgb_pre go to the evaluated rows only; rows n_rows .. n_pad - 1 (padding of the last MLP tile) get 0.
// n_rows is read on the device (the pass's total in ofs), n_pad is its multiple of 128.
// Also the amax words of the scale selection and status 103 for a non-finite per-sample gradient.
struct TrainSkipBwdParams {
  int n_rays, S;
  const long long* n_rows;      // device: the evaluated rows of the pass
  const float* rays;            // (n_rays, 8)
  const float* z;               // (n_rays, S) depths of the pass
  const uint32_t* mask;         // (n_rays, kSkipMaskWords)
  const long long* ofs;         // (n_rays + 1)
  const float* sigma;           // (n_pad) raw sigma of the rows
  const float* rgb;             // (n_pad, 3)
  const float* noise;           // (n_rays, S) or null
  float noise_std;
  int white_back;
  const float* rgb_out;         // (n_rays, 3) rendered colour of the pass
  const float* target;          // (n_rays, 3)
  const float* loss_grad;       // device scalar dL/dloss or null (= 1)
  float* dsigma;                // (n_pad)
  float* dprergb;               // (n_pad, 3)
  unsigned* amax_bits;          // [2]
  int* status;
};

__global__ void __launch_bounds__(kSkipWarps * 32) train_skip_bwd_kernel(const TrainSkipBwdParams p) {
  const int lane = threadIdx.x & 31;
  const int S = p.S, P = S >> 5;
  float amax = 0.f, amax_rgb = 0.f;
  bool nonfinite = false;
  const float lg = (p.loss_grad != nullptr) ? *p.loss_grad : 1.f;
  const float kseed = 2.f * lg / (3.f * static_cast<float>(p.n_rays));
  for (long long ray = static_cast<long long>(blockIdx.x) * kSkipWarps + (threadIdx.x >> 5); ray < p.n_rays;
       ray += static_cast<long long>(gridDim.x) * kSkipWarps) {
    const float* rr = p.rays + ray * 8;
    const float dx = rr[3], dy = rr[4], dz = rr[5];
    const float dnorm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    float g[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) g[c] = 0.f + kseed * (p.rgb_out[ray * 3 + c] - p.target[ray * 3 + c]);
    float go = 0.f;
    if (p.white_back) go -= g[0] + g[1] + g[2];
    const float* z = p.z + ray * S;
    const uint32_t* m = p.mask + ray * kSkipMaskWords;
    // the row of this lane's first sample: the ray's offset plus its evaluated samples before lane * P
    long long row0 = p.ofs[ray];
    const int i0 = lane * P;
    for (int w = 0; w < (i0 >> 5); ++w) row0 += __popc(m[w]);
    row0 += __popc(m[i0 >> 5] & ((1u << (i0 & 31)) - 1u));
    float alpha[6], tloc[6], om[6], dw[6], de[6], wgt[6], col[6][3];
    bool pos[6], ev[6];
    long long row[6];
    float prod = 1.f;
    long long rnext = row0;
    for (int q = 0; q < P; ++q) {
      const int i = i0 + q;
      ev[q] = mask_bit(m, i);
      row[q] = rnext;
      rnext += ev[q] ? 1 : 0;
      float delta = (i < S - 1) ? __fsub_rn(z[i + 1], z[i]) : 1e10f;
      delta = __fmul_rn(delta, dnorm);
      float s = 0.f;
      col[q][0] = col[q][1] = col[q][2] = 0.f;
      if (ev[q]) {
        s = p.sigma[row[q]];
        if (p.noise != nullptr) s = __fadd_rn(s, __fmul_rn(p.noise[ray * S + i], p.noise_std));
        col[q][0] = p.rgb[row[q] * 3]; col[q][1] = p.rgb[row[q] * 3 + 1]; col[q][2] = p.rgb[row[q] * 3 + 2];
      }
      const float e = expf(-__fmul_rn(delta, fmaxf(s, 0.f)));
      alpha[q] = __fsub_rn(1.f, e);
      om[q] = __fadd_rn(__fsub_rn(1.f, alpha[q]), 1e-10f);
      de[q] = delta * e;
      pos[q] = s > 0.f;
      tloc[q] = prod;
      prod = __fmul_rn(prod, om[q]);
      dw[q] = g[0] * col[q][0] + g[1] * col[q][1] + g[2] * col[q][2] + 0.f * z[i] + go;
    }
    float incl = prod;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl *= v;
    }
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.f;
    float asum = 0.f;
    for (int q = 0; q < P; ++q) {
      tloc[q] *= excl;
      wgt[q] = alpha[q] * tloc[q];
      asum += wgt[q] * dw[q];
    }
    float sincl = asum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float v = __shfl_down_sync(0xffffffffu, sincl, o);
      if (lane + o < 32) sincl += v;
    }
    float after = __shfl_down_sync(0xffffffffu, sincl, 1);
    if (lane == 31) after = 0.f;
    float run = after;
    for (int q = P - 1; q >= 0; --q) {
      const float dalpha = tloc[q] * dw[q] - run / om[q];
      run += wgt[q] * dw[q];
      if (!ev[q]) continue;
      const float ds = pos[q] ? dalpha * de[q] : 0.f;
      p.dsigma[row[q]] = ds;
      amax = fmaxf(amax, fabsf(ds));
      nonfinite |= !isfinite(ds);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float c = col[q][ch];
        const float dp = wgt[q] * g[ch] * c * (1.f - c);
        p.dprergb[row[q] * 3 + ch] = dp;
        amax_rgb = fmaxf(amax_rgb, fabsf(dp));
        nonfinite |= !isfinite(dp);
      }
    }
  }
  if (__any_sync(0xffffffffu, nonfinite) && lane == 0) report_fault(p.status, 103);
  const long long n_rows = *p.n_rows, n_pad = (n_rows + 127) / 128 * 128;
  for (long long i = n_rows + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_pad;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    p.dsigma[i] = 0.f;
    p.dprergb[3 * i] = 0.f; p.dprergb[3 * i + 1] = 0.f; p.dprergb[3 * i + 2] = 0.f;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    amax_rgb = fmaxf(amax_rgb, __shfl_xor_sync(0xffffffffu, amax_rgb, o));
  }
  if (lane == 0 && amax > 0.f && amax < 3e38f) atomicMax(p.amax_bits, __float_as_uint(amax));
  if (lane == 0 && amax_rgb > 0.f && amax_rgb < 3e38f) atomicMax(p.amax_bits + 1, __float_as_uint(amax_rgb));
}

// The evaluated sample counts of both passes (the totals of their scans; 0 for the fine pass without one).
__global__ void train_skip_counts_kernel(const long long* c0, const long long* c1, long long* out) {
  if (threadIdx.x == 0) {
    out[0] = *c0;
    out[1] = c1 != nullptr ? *c1 : 0;
  }
}

// dst[0 .. *rows * width) = src[...]: the optional per-row outputs of the backward, exactly the evaluated rows.
__global__ void train_skip_copy_rows_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                            const long long* __restrict__ rows, int width) {
  const long long total = *rows * width;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dst[i] = src[i];
}

}  // namespace nerfb200
