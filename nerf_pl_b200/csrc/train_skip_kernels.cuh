// The training step with empty samples skipped (DESIGN.md "Training with empty samples skipped").  The rule of
// sample_skip_kernels.cuh carried into training: the coarse depths are the render kernel's stratified depths with the
// perturb jitter, an evaluated sample gets the network's sigma + noise * noise_std, a skipped one sigma = 0 without
// noise (weight exactly 0, no gradient), and the resampling uses the render kernel's sorted random u.  The compacted
// rows go through mlp_forward_kernel<true, true>, which leaves in one NeRF.forward training workspace per network what
// nerfb200_nerf_backward's tail reads; the backward starts with train_skip_bwd_kernel, the compositing backward over
// the sparse sample lists.
//
// The forward runs the per-ray kernels of sample_skip_kernels.cuh with the training inputs set (perturb, noise, the
// random u, the zc and dirrow workspace) and ends with the loss (mse_psnr_kernel).  This file holds what only training
// has: the sparse compositing backward, the device copy of the sample counts and the per-row copies.
#pragma once
#include "sample_skip_kernels.cuh"

namespace nerfb200 {

// composite_bwd_kernel's arithmetic (its seed: upstream g_rgb / g_depth / g_opac and the fused MSE term, white_back,
// noise, the ReLU mask, in its evaluation order) on one ray per warp, with
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
  const float* g_rgb;           // (n_rays, 3) upstream gradient of the pass's colour or null
  const float* g_depth;         // (n_rays) or null
  const float* g_opac;          // (n_rays) or null
  const float* rgb_out;         // (n_rays, 3) rendered colour of the pass, used with `target`
  const float* target;          // (n_rays, 3) or null: adds the MSE seed 2 (rgb_out - target) / (3 n_rays) * loss_grad
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
  for (long long ray = static_cast<long long>(blockIdx.x) * kSkipWarps + (threadIdx.x >> 5); ray < p.n_rays;
       ray += static_cast<long long>(gridDim.x) * kSkipWarps) {
    const float* rr = p.rays + ray * 8;
    const float dx = rr[3], dy = rr[4], dz = rr[5];
    const float dnorm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    float g[3] = {0.f, 0.f, 0.f};
    if (p.g_rgb != nullptr) { g[0] = p.g_rgb[ray * 3]; g[1] = p.g_rgb[ray * 3 + 1]; g[2] = p.g_rgb[ray * 3 + 2]; }
    if (p.target != nullptr) {
      const float lg = (p.loss_grad != nullptr) ? *p.loss_grad : 1.f;
      const float k = 2.f * lg / (3.f * static_cast<float>(p.n_rays));
#pragma unroll
      for (int c = 0; c < 3; ++c) g[c] += k * (p.rgb_out[ray * 3 + c] - p.target[ray * 3 + c]);
    }
    const float gd = (p.g_depth != nullptr) ? p.g_depth[ray] : 0.f;
    float go = (p.g_opac != nullptr) ? p.g_opac[ray] : 0.f;
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
      dw[q] = g[0] * col[q][0] + g[1] * col[q][1] + g[2] * col[q][2] + gd * z[i] + go;
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
