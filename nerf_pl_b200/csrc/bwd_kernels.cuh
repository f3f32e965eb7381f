// Backward of the render_rays training step (reference: train.py:103-117 loss.backward() through
// models/rendering.py:143-170 and models/nerf.py:100-124), hand-written for sm_90a.
//
// The forward launch in "train" mode (render_kernel.cuh, kSave) leaves per sample in the training
// workspace: the encoded input, the 8 hidden activations (fp16, tiled layout of layout.h), the ReLU
// sign bits of the 8 hidden layers, the direction-layer output, raw sigma and rgb.  The backward is
//
//   composite_bwd_kernel  warp per ray: d(rgb, depth, opacity) [or the fused MSE seed] -> per-sample
//                         d sigma, d rgb_pre                                   (CUDA cores)
//   head_bwd_kernel       rgb head + ReLU of the direction layer: dd (tiled 16-bit), the rgb-head and
//                         direction-part weight gradients                      (CUDA cores)
//   chain_bwd_kernel      dgrad chain on the wgmma tile engine: per 128-sample tile
//                         dd -> dh8 -> dpre8 -> ... -> dpre1, activations in registers exactly like the
//                         forward, 30 transposed weight slices per tile; writes dpre_l (tiled)
//   wgrad_kernel          split-K wgmma GEMMs gW_l = dpre_l^T h_{l-1}: one CTA per (layer, sample
//                         range), both operands MN-major straight from the tiled arrays, fp32
//                         accumulators in registers per piece of the CTA's range, the pieces added in
//                         fp32; bias gradients as column sums on the CUDA cores of the same tiles
//   wgrad_reduce_kernel   fixed-order sum of the per-CTA partials into the .grad tensors
//   unfold_kernel         chain rule through the pack-time folding W' = W_dir[:, :256] W_final
//
// Per-sample gradients are fp16 with a power-of-two scale PER LAYER, chosen on the device in the
// same step (no state carried between steps, deterministic): level 0 (dd) from a bound on its
// largest element, |d rgb_pre|_max * max_n sum_c |W_rgb[c][n]|; levels 1..8 (dpre_8..dpre_1) from
// the largest elements a PROBE pass of the chain kernel sees on one tile per SM, spread evenly over
// each pass (no stores), each
// mapped to 64 (10 bits of headroom to the fp16 maximum, 20 bits of normal range below; gradients
// shrink or grow by orders of magnitude through 8 layers, one global scale costs precision in the
// deep layers: measured 4e-2 relative error at layer 1 vs 4e-3 with per-layer scales).
// Conversions saturate instead of producing inf; the weight gradients accumulate in fp32 and are
// un-scaled per layer by the reduction.
// fp16 rather than bf16 because the wgrad GEMM contracts the gradients with the forward's fp16
// activations and wgmma takes its two 16-bit operands in one type (f16 x f16 or bf16 x bf16, PTX ISA
// "wgmma.mma_async").
#pragma once
#include "render_kernel.cuh"

namespace nerfb200 {

__device__ __forceinline__ uint32_t cvt_bwd_x2(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
// packed fp16 add
__device__ __forceinline__ uint32_t bwd_add_x2(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("add.rn.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}

// ------------------------------------------------------------------------- compositing backward
// models/rendering.py:143-170 differentiated by hand (oracle/nerf_oracle_grad.py
// volume_render_backward is the executable statement of the same formulas):
//   w_i = alpha_i T_i,  T_i = prod_{j<i} (1 - alpha_j + 1e-10),  alpha_i = 1 - exp(-delta_i relu(s_i))
//   dL/dw_i     = <g_rgb, c_i> + g_depth z_i + g_opac - [white_back] sum_ch g_rgb
//   dL/dalpha_i = T_i dL/dw_i - (sum_{j>i} w_j dL/dw_j) / (1 - alpha_i + 1e-10)
//   dL/dsigma_i = dL/dalpha_i delta_i exp(-delta_i relu(s_i)) [s_i > 0]
//   dL/dc_i     = w_i g_rgb;  through the sigmoid: dL/dpre_i = dL/dc_i c_i (1 - c_i)
// One warp per ray, each lane owns P = S / 32 consecutive samples.
struct CompBwdParams {
  int n_rays, S;
  long long n_pad;
  const float* z;
  const float* sigma;
  const float* rgb;
  const float* rays;
  long long ray_stride;
  const float* noise;       // (n_rays, S) or null
  float noise_std;
  int white_back;
  const float* g_rgb;       // (n_rays, 3) upstream gradient or null
  const float* g_depth;     // (n_rays) or null
  const float* g_opac;      // (n_rays) or null
  const float* rgb_out;     // (n_rays, 3) rendered colour, used with `target`
  const float* target;      // (n_rays, 3) or null: adds the MSE seed 2 (rgb_out - target) / (3 n_rays) * loss_grad
  const float* loss_grad;   // device scalar dL/dloss or null (= 1)
  float* dsigma;
  float* dprergb;
  unsigned* amax_bits;      // [2]: max |d sigma|, max |d rgb_pre| as float bits (scale selection) or null
  int* status;              // device status word: 103 when a per-sample gradient is not finite
};

__global__ void __launch_bounds__(128) composite_bwd_kernel(const CompBwdParams p) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const long long ray = static_cast<long long>(blockIdx.x) * wpb + (threadIdx.x >> 5);
  const int S = p.S, P = S >> 5;
  float amax = 0.f, amax_rgb = 0.f;
  bool nonfinite = false;
  if (ray < p.n_rays) {
    const float* rr = p.rays + ray * p.ray_stride;
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
    const long long g0 = ray * S;
    float alpha[6], tloc[6], om[6], dw[6], de[6], wgt[6];
    bool pos[6];
    float prod = 1.f;
    for (int q = 0; q < P; ++q) {
      const int i = lane * P + q;
      float delta = (i < S - 1) ? __fsub_rn(z[i + 1], z[i]) : 1e10f;
      delta = __fmul_rn(delta, dnorm);
      float s = p.sigma[g0 + i];
      if (p.noise != nullptr) s = __fadd_rn(s, __fmul_rn(p.noise[g0 + i], p.noise_std));
      const float e = expf(-__fmul_rn(delta, fmaxf(s, 0.f)));
      alpha[q] = __fsub_rn(1.f, e);
      om[q] = __fadd_rn(__fsub_rn(1.f, alpha[q]), 1e-10f);
      de[q] = delta * e;
      pos[q] = s > 0.f;
      tloc[q] = prod;
      prod = __fmul_rn(prod, om[q]);
      const float* c = p.rgb + (g0 + i) * 3;
      dw[q] = g[0] * c[0] + g[1] * c[1] + g[2] * c[2] + gd * z[i] + go;
    }
    float incl = prod;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl *= v;
    }
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.f;
    // suffix sums of a_i = w_i dL/dw_i (exclusive, from the far end)
    float asum = 0.f;
    for (int q = 0; q < P; ++q) {
      tloc[q] *= excl;                     // T_i
      wgt[q] = alpha[q] * tloc[q];         // w_i
      asum += wgt[q] * dw[q];
    }
    float sincl = asum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float v = __shfl_down_sync(0xffffffffu, sincl, o);
      if (lane + o < 32) sincl += v;
    }
    float after = __shfl_down_sync(0xffffffffu, sincl, 1);     // sum over lanes > this one
    if (lane == 31) after = 0.f;
    float run = after;
    for (int q = P - 1; q >= 0; --q) {
      const int i = lane * P + q;
      const float dalpha = tloc[q] * dw[q] - run / om[q];
      run += wgt[q] * dw[q];
      const float ds = pos[q] ? dalpha * de[q] : 0.f;
      p.dsigma[g0 + i] = ds;
      amax = fmaxf(amax, fabsf(ds));
      nonfinite |= !isfinite(ds);
      const float* c = p.rgb + (g0 + i) * 3;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float dp = wgt[q] * g[ch] * c[ch] * (1.f - c[ch]);
        p.dprergb[(g0 + i) * 3 + ch] = dp;
        amax_rgb = fmaxf(amax_rgb, fabsf(dp));
        nonfinite |= !isfinite(dp);
      }
    }
  }
  // A non-finite ray, colour or upstream gradient: the reference's gradients are NaN everywhere, but fmaxf above
  // drops NaN and the wgrad sums of the biases never see it, so say so instead of returning finite bias gradients.
  if (__any_sync(0xffffffffu, nonfinite) && lane == 0) report_fault(p.status, 103);
  // padding rows carry no gradient
  const long long n = static_cast<long long>(p.n_rays) * S;
  if (blockIdx.x == gridDim.x - 1)
    for (long long i = n + threadIdx.x; i < p.n_pad; i += blockDim.x) {
      p.dsigma[i] = 0.f;
      p.dprergb[3 * i] = 0.f; p.dprergb[3 * i + 1] = 0.f; p.dprergb[3 * i + 2] = 0.f;
    }
  if (p.amax_bits != nullptr) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      amax_rgb = fmaxf(amax_rgb, __shfl_xor_sync(0xffffffffu, amax_rgb, o));
    }
    if (lane == 0 && amax > 0.f && amax < 3e38f) atomicMax(p.amax_bits, __float_as_uint(amax));
    if (lane == 0 && amax_rgb > 0.f && amax_rgb < 3e38f) atomicMax(p.amax_bits + 1, __float_as_uint(amax_rgb));
  }
}

// ------------------------------------------------------------------------ NeRF.forward seed
// The backward of a direct NeRF.forward call (models/nerf.py:83-124, output [rgb, sigma]) starts from the
// upstream gradient g (n, 4) instead of from compositing:  d rgb_pre = g_rgb rgb (1 - rgb) through the sigmoid
// (models/nerf.py:120), d sigma = g_sigma.  Rows n .. n_pad - 1 (padding of the last tile) are written as zero.
// Also the amax words bwd_scale_kernel's phase 0 reads.  One thread per row.
struct MlpSeedParams {
  long long n, n_pad;
  const float* g;           // (n, 4) upstream gradient [rgb, sigma]
  const float* rgb;         // (n_pad, 3) stored sigmoid(rgb)
  float* dsigma;            // (n_pad)
  float* dprergb;           // (n_pad, 3)
  unsigned* amax_bits;      // [2]: max |d sigma|, max |d rgb_pre| as float bits
  int* status;              // device status word: 103 when a per-sample gradient is not finite
};
__global__ void __launch_bounds__(256) mlp_seed_kernel(const MlpSeedParams p) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  float amax = 0.f, amax_rgb = 0.f;
  bool nonfinite = false;
  if (i < p.n) {
    const float4 g = __ldg(reinterpret_cast<const float4*>(p.g) + i);
    const float gc[3] = {g.x, g.y, g.z};
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float c = p.rgb[i * 3 + ch];
      const float dp = gc[ch] * c * (1.f - c);
      p.dprergb[i * 3 + ch] = dp;
      amax_rgb = fmaxf(amax_rgb, fabsf(dp));
      nonfinite |= !isfinite(dp);
    }
    p.dsigma[i] = g.w;
    amax = fabsf(g.w);
    nonfinite |= !isfinite(g.w);
  } else if (i < p.n_pad) {
    p.dsigma[i] = 0.f;
    p.dprergb[3 * i] = 0.f; p.dprergb[3 * i + 1] = 0.f; p.dprergb[3 * i + 2] = 0.f;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    amax_rgb = fmaxf(amax_rgb, __shfl_xor_sync(0xffffffffu, amax_rgb, o));
  }
  const int lane = threadIdx.x & 31;
  if (__any_sync(0xffffffffu, nonfinite) && lane == 0) report_fault(p.status, 103);   // as composite_bwd_kernel
  if (lane == 0 && amax > 0.f && amax < 3e38f) atomicMax(p.amax_bits, __float_as_uint(amax));
  if (lane == 0 && amax_rgb > 0.f && amax_rgb < 3e38f) atomicMax(p.amax_bits + 1, __float_as_uint(amax_rgb));
}

// Per-pass, per-level scales (see the header comment).  Level v: 0 = dd, v = 1..8 = dpre_{9-v}.
//   phase 0 (before head_bwd / the probe): every level gets the level-0 scale
//            2^floor(log2(64 / max(|d rgb_pre|_max wmax_rgb, |d sigma|_max wmax_sigma)))
//   phase 1 (after the probe pass): levels 1..8 from the probe's per-level maxima (true, un-scaled
//            values), clamped to [2^-12, 2^40] x level 0; a level the probe saw nothing in keeps its
//            predecessor's scale.  Resets the statistics for the next step.
constexpr int kLevels = 9;
struct ScaleParams {
  int n_pass, phase;
  unsigned* amax;            // [2 passes][2]: |d sigma|, |d rgb_pre| maxima (float bits)
  unsigned* lamax;           // [2 passes][kLevels] probe maxima (float bits)
  float* lscale;             // [2][kLevels]
  float* linv;               // [2][kLevels]
  const float* w_rgb[2];     // live fp32 (3,128)
  const float* w_sigma[2];   // live fp32 (256)
};
__global__ void __launch_bounds__(128) bwd_scale_kernel(const ScaleParams p) {
  __shared__ float red[2][128];
  const int t = threadIdx.x;
  for (int ps = 0; ps < p.n_pass; ++ps) {
    if (p.phase == 0) {
      float wr = fabsf(p.w_rgb[ps][t]) + fabsf(p.w_rgb[ps][128 + t]) + fabsf(p.w_rgb[ps][256 + t]);
      float wsg = fmaxf(fabsf(p.w_sigma[ps][t]), fabsf(p.w_sigma[ps][128 + t]));
      red[0][t] = wr; red[1][t] = wsg;
      __syncthreads();
      for (int o = 64; o > 0; o >>= 1) {
        if (t < o) { red[0][t] = fmaxf(red[0][t], red[0][t + o]); red[1][t] = fmaxf(red[1][t], red[1][t + o]); }
        __syncthreads();
      }
      if (t < kLevels) {
        float s = 1.f;
        const float bound = fmaxf(__uint_as_float(p.amax[2 * ps + 1]) * red[0][0], __uint_as_float(p.amax[2 * ps]) * red[1][0]);
        if (bound > 0.f) s = exp2f(floorf(log2f(64.f / bound)));
        s = fminf(fmaxf(s, 1e-30f), 1e30f);
        p.lscale[ps * kLevels + t] = s;
        p.linv[ps * kLevels + t] = 1.f / s;
        p.lamax[ps * kLevels + t] = 0u;
      }
      __syncthreads();
      if (t < 2) p.amax[2 * ps + t] = 0u;
    } else if (t == 0) {
      const float s0 = p.lscale[ps * kLevels];
      float prev = s0;
      for (int v = 1; v < kLevels; ++v) {
        const float am = __uint_as_float(p.lamax[ps * kLevels + v]);
        float s = prev;
        if (am > 0.f) s = exp2f(floorf(log2f(64.f / am)));
        s = fminf(fmaxf(s, s0 * 2.44140625e-4f), s0 * 1.0995116e12f);
        p.lscale[ps * kLevels + v] = s;
        p.linv[ps * kLevels + v] = 1.f / s;
        p.lamax[ps * kLevels + v] = 0u;
        prev = s;
      }
    }
  }
}

// ------------------------------------------------------------------------ rgb head / dir ReLU
// models/nerf.py:119-120 backwards, per sample:  dd = (dpre_rgb W_rgb) * (d > 0)  -> tiled fp16 (the
// A operand of the chain kernel's first step and of the W' wgrad), plus the small weight gradients
// that contract over samples on the CUDA cores:
//   gW_rgb[c][n] = sum_s dpre_rgb[s][c] d[s][n]     gb_rgb[c] = sum_s dpre_rgb[s][c]
//   raysum[ray][n] = sum_{s in ray} dd[s][n]        (the direction is constant along a ray: the direction
//   part of gW_dir is sum_rays raysum[ray] (x) dir_enc[ray], dir_grad_kernel below)
//   gW_sigma[n] = sum_s dsigma[s] h8[s][n]          gb_sigma = sum_s dsigma[s]     (models/nerf.py:112)
// A streaming kernel (0.5 KB per sample): one warp per ray and pass, lane = 4 adjacent columns, 8-byte
// loads / stores of the tiled arrays, the sample loop unrolled so that 8 rows are in flight per warp.
// Per-block partials of gW_rgb / gb_rgb, summed in fixed order by wgrad_reduce_kernel.
constexpr int kHeadWarps = 4;
constexpr int kHeadPartRgbW = 0;            // [3][128]
constexpr int kHeadPartRgbB = 384;          // [4]
constexpr int kHeadPartSigW = 388;          // [256]
constexpr int kHeadPartSigB = 644;          // [4]
constexpr int kHeadPartFloats = 648;
struct HeadBwdParams {
  int n_rays, n_pass;
  PassBufs pass[2];
  const float* w_rgb[2];    // live fp32 (3,128)
  const float* lscale;      // [2][kLevels]: level 0 of each pass scales dd
  const float* rays;
  long long ray_stride;
  float* raysum[2];         // (n_rays, 128), or null (NeRF.forward backward: no per-ray direction)
  float* direnc;            // (n_rays, 28): Embedding(3,4)(rays_d), as the forward computes it, or null (same)
  float* part[2];           // [gridDim.x][kHeadPartFloats] per pass (blocks of the other pass write zeros)
};

// (A two-role variant - one warp streaming d, a second one h8, 24 warps per SM instead of 16 - measured 128 us
// against 88 us for this one: more warps in flight did not help, the extra address streams hurt.)
// The body of head_bwd_kernel and of head_bwd_dev_kernel over a HeadBwdParams `p`.  A macro rather than a device
// function: the plain kernel then compiles to the instructions it had before the planned variant existed.
#define NERFB200_HEAD_BWD_BODY                                                                                                      \
  __shared__ float red[kHeadWarps][kHeadPartFloats];                                                                                \
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;                                                                       \
  const long long unit = static_cast<long long>(blockIdx.x) * kHeadWarps + warp;  /* (pass, ray) */                                 \
  const int ps = unit >= p.n_rays ? 1 : 0;                                                                                          \
  const long long ray = unit - (ps ? p.n_rays : 0);                                                                                 \
  const bool active = ray < p.n_rays && ps < p.n_pass;                                                                              \
  float gw[3][4], gb[3] = {0.f, 0.f, 0.f}, rs[4] = {0.f, 0.f, 0.f, 0.f};                                                            \
  float gs[8], gsb = 0.f;  /* sigma head: this lane's 8 columns of h8 (one 16-byte chunk), sum of dsigma */                         \
_Pragma("unroll")                                                                                                                   \
  for (int c = 0; c < 3; ++c)                                                                                                       \
_Pragma("unroll")                                                                                                                   \
    for (int i = 0; i < 4; ++i) gw[c][i] = 0.f;                                                                                     \
_Pragma("unroll")                                                                                                                   \
  for (int i = 0; i < 8; ++i) gs[i] = 0.f;                                                                                          \
  if (active) {                                                                                                                     \
    const PassBufs& pb = p.pass[ps];                                                                                                \
    const int S = pb.S;                                                                                                             \
    const float scale = p.lscale[ps * kLevels];                                                                                     \
    float w[3][4];                                                                                                                  \
_Pragma("unroll")                                                                                                                   \
    for (int c = 0; c < 3; ++c)                                                                                                     \
_Pragma("unroll")                                                                                                                   \
      for (int i = 0; i < 4; ++i) w[c][i] = p.w_rgb[ps][c * 128 + 4 * lane + i];                                                    \
    if (ps == 0 && lane < 15 && p.direnc != nullptr) {  /* Embedding(3,4)(rays_d) exactly as render_kernel.cuh setup_group */       \
      const int cc = lane / 5, kk = lane % 5;                                                                                       \
      const float dv = p.rays[ray * p.ray_stride + 3 + cc];                                                                         \
      float* de = p.direnc + ray * 28;                                                                                              \
      if (kk == 4) {                                                                                                                \
        de[cc] = dv;                                                                                                                \
      } else {                                                                                                                      \
        float sn, cs;                                                                                                               \
        sincosf(__fmul_rn(static_cast<float>(1 << kk), dv), &sn, &cs);                                                              \
        de[3 + 6 * kk + cc] = sn;                                                                                                   \
        de[3 + 6 * kk + 3 + cc] = cs;                                                                                               \
      }                                                                                                                             \
    }                                                                                                                               \
    /* lane's 4 columns: column block lane / 16, 16-byte chunk (lane % 16) / 2, half (lane & 1) */                                  \
    const uint32_t fb = lane >> 4, ch = (lane & 15) >> 1, hf = (lane & 1) * 8;                                                      \
    const uint8_t* h8 = pb.act + 7ll * pb.n_pad * 512;                                                                              \
    const long long g0 = ray * S;                                                                                                   \
_Pragma("unroll 8")                                                                                                                 \
    for (int i = 0; i < S; ++i) {                                                                                                   \
      const long long g = g0 + i;                                                                                                   \
      const unsigned long long off = tiled_block_off(static_cast<unsigned long long>(g >> 6), fb, 2) + (g & 63) * 128 +             \
                                     ((ch ^ static_cast<uint32_t>(g & 7)) << 4) + hf;                                               \
      const uint2 dv2 = __ldg(reinterpret_cast<const uint2*>(pb.d + off));                                                          \
      /* h8 row: 32 lanes x 16 bytes, lane = (column block lane / 8, chunk lane % 8) */                                             \
      const uint4 hv = __ldg(reinterpret_cast<const uint4*>(                                                                        \
          h8 + tiled_block_off(static_cast<unsigned long long>(g >> 6), lane >> 3, 4) + (g & 63) * 128 +                            \
          (((lane & 7u) ^ static_cast<uint32_t>(g & 7)) << 4)));                                                                    \
      const float ds = __ldg(pb.dsigma + g);                                                                                        \
      {                                                                                                                             \
        const float2 a0 = __half22float2(*reinterpret_cast<const __half2*>(&hv.x));                                                 \
        const float2 a1 = __half22float2(*reinterpret_cast<const __half2*>(&hv.y));                                                 \
        const float2 a2 = __half22float2(*reinterpret_cast<const __half2*>(&hv.z));                                                 \
        const float2 a3 = __half22float2(*reinterpret_cast<const __half2*>(&hv.w));                                                 \
        gs[0] = fmaf(ds, a0.x, gs[0]); gs[1] = fmaf(ds, a0.y, gs[1]); gs[2] = fmaf(ds, a1.x, gs[2]); gs[3] = fmaf(ds, a1.y, gs[3]); \
        gs[4] = fmaf(ds, a2.x, gs[4]); gs[5] = fmaf(ds, a2.y, gs[5]); gs[6] = fmaf(ds, a3.x, gs[6]); gs[7] = fmaf(ds, a3.y, gs[7]); \
        gsb += ds;                                                                                                                  \
      }                                                                                                                             \
      const float q0 = __ldg(pb.dprergb + 3 * g), q1 = __ldg(pb.dprergb + 3 * g + 1), q2 = __ldg(pb.dprergb + 3 * g + 2);           \
      const float2 d01 = __half22float2(*reinterpret_cast<const __half2*>(&dv2.x));                                                 \
      const float2 d23 = __half22float2(*reinterpret_cast<const __half2*>(&dv2.y));                                                 \
      const float dv[4] = {d01.x, d01.y, d23.x, d23.y};                                                                             \
      float val[4];                                                                                                                 \
_Pragma("unroll")                                                                                                                   \
      for (int k = 0; k < 4; ++k) {                                                                                                 \
        gw[0][k] = fmaf(q0, dv[k], gw[0][k]);                                                                                       \
        gw[1][k] = fmaf(q1, dv[k], gw[1][k]);                                                                                       \
        gw[2][k] = fmaf(q2, dv[k], gw[2][k]);                                                                                       \
        val[k] = (dv[k] > 0.f) ? fmaf(q0, w[0][k], fmaf(q1, w[1][k], q2 * w[2][k])) : 0.f;                                          \
        rs[k] += val[k];                                                                                                            \
      }                                                                                                                             \
      gb[0] += q0; gb[1] += q1; gb[2] += q2;                                                                                        \
      *reinterpret_cast<uint2*>(pb.dd + off) = make_uint2(cvt_bwd_x2(val[0] * scale, val[1] * scale),                               \
                                                          cvt_bwd_x2(val[2] * scale, val[3] * scale));                              \
    }                                                                                                                               \
    if (p.raysum[ps] != nullptr)                                                                                                    \
      *reinterpret_cast<float4*>(p.raysum[ps] + ray * 128 + 4 * lane) = make_float4(rs[0], rs[1], rs[2], rs[3]);                    \
  }                                                                                                                                 \
  /* per-block partial of gW_rgb / gb_rgb: warps in fixed order */                                                                  \
_Pragma("unroll")                                                                                                                   \
  for (int c = 0; c < 3; ++c)                                                                                                       \
_Pragma("unroll")                                                                                                                   \
    for (int k = 0; k < 4; ++k) red[warp][c * 128 + 4 * lane + k] = gw[c][k];                                                       \
  if (lane < 4) red[warp][kHeadPartRgbB + lane] = (lane < 3) ? gb[lane] : 0.f;                                                      \
_Pragma("unroll")                                                                                                                   \
  for (int k = 0; k < 8; ++k) red[warp][kHeadPartSigW + 8 * lane + k] = gs[k];                                                      \
  if (lane < 4) red[warp][kHeadPartSigB + lane] = (lane == 0) ? gsb : 0.f;                                                          \
  __syncthreads();                                                                                                                  \
  /* a block's warps all belong to one pass unless it straddles the boundary: sum per pass */                                       \
  for (int q = 0; q < p.n_pass; ++q) {                                                                                              \
    float* out = p.part[q] + static_cast<long long>(blockIdx.x) * kHeadPartFloats;                                                  \
    for (int i = threadIdx.x; i < kHeadPartFloats; i += blockDim.x) {                                                               \
      float acc = 0.f;                                                                                                              \
      for (int wv = 0; wv < kHeadWarps; ++wv) {                                                                                     \
        const long long u = static_cast<long long>(blockIdx.x) * kHeadWarps + wv;                                                   \
        if ((u >= p.n_rays ? 1 : 0) == q) acc += red[wv][i];                                                                        \
      }                                                                                                                             \
      out[i] = acc;                                                                                                                 \
    }                                                                                                                               \
  }

__global__ void __launch_bounds__(kHeadWarps * 32) head_bwd_kernel(const HeadBwdParams p) { NERFB200_HEAD_BWD_BODY }
// The same with its parameters planned on the device (capi.cu train_skip_plan_kernel): launched at the grid of the
// carved worst case, the blocks past the plan's *grid return without writing.
__global__ void __launch_bounds__(kHeadWarps * 32) head_bwd_dev_kernel(const HeadBwdParams* __restrict__ pp,
                                                                        const int* __restrict__ grid) {
  if (static_cast<int>(blockIdx.x) >= *grid) return;
  const HeadBwdParams& p = *pp;
  NERFB200_HEAD_BWD_BODY
}

// gW_dir[n][256 + j] = sum_rays raysum[ray][n] dir_enc[ray][j]: block = 128 threads (n), blockIdx.x = ray slice,
// blockIdx.y = pass; per-slice partials [slice][n][27], summed by wgrad_reduce_kernel.
constexpr int kDirSlices = 64;
struct DirGradParams {
  int n_rays;
  const float* raysum[2];
  const float* direnc;
  float* part[2];           // [kDirSlices][128][27]
};
__global__ void __launch_bounds__(128) dir_grad_kernel(const DirGradParams p) {
  __shared__ float de[64][28];
  const int ps = blockIdx.y, n = threadIdx.x;
  const int per = (p.n_rays + kDirSlices - 1) / kDirSlices;
  const int r0 = blockIdx.x * per, r1 = min(r0 + per, p.n_rays);
  float acc[27];
#pragma unroll
  for (int j = 0; j < 27; ++j) acc[j] = 0.f;
  for (int base = r0; base < r1; base += 64) {
    const int cnt = min(64, r1 - base);
    __syncthreads();
    for (int i = n; i < cnt * 28; i += 128) de[i / 28][i % 28] = p.direnc[static_cast<long long>(base) * 28 + i];
    __syncthreads();
#pragma unroll 4
    for (int r = 0; r < cnt; ++r) {
      const float v = p.raysum[ps][static_cast<long long>(base + r) * 128 + n];
#pragma unroll
      for (int j = 0; j < 27; ++j) acc[j] = fmaf(v, de[r][j], acc[j]);
    }
  }
  float* out = p.part[ps] + (static_cast<long long>(blockIdx.x) * 128 + n) * 27;
#pragma unroll
  for (int j = 0; j < 27; ++j) out[j] = acc[j];
}

// ------------------------------------------------------------------------------ dgrad chain
// Per 128-sample tile, on the forward's tile engine (mlp_engine.cuh: same warp roles, same weight ring,
// same register-resident A operand between layers):
//   step 0     D = dd[128 x 128] . W'           (A from shared memory: the dd tile, 2 K blocks)
//              dh8 = D + dsigma (x) w_sigma ;  dpre8 = dh8 * relu'(h8)
//   step s>=1  D = dpre_l[128 x 256] . W_l      (A from registers, l = 8, 7, .., 2; for l = 5
//              only the hidden columns 63..318 of W_5)        dpre_{l-1} = D * relu'(h_{l-1})
// relu' comes from the sign bits the forward stored (64 per thread, row and layer; the backward thread
// of a row owns the same columns as the forward thread did).  Every dpre_l is also written to HBM (tiled
// 16-bit) for the wgrad kernel.  30 weight slices per tile, the same tensor work as layers 2-8 of the forward.
constexpr int kChainSteps = 8;
constexpr uint32_t kChA0 = 0;                          // 2 x [2 K blocks][128 x 64] 16-bit = 2 x 32 KiB
constexpr uint32_t kChA0Bytes = 32768;
constexpr uint32_t kChRing = 2 * kChA0Bytes;           // kStages x 32 KiB
constexpr uint32_t kChConsts = kChRing + kStages * kSliceBytes256;   // w_sigma of both networks (2 x 256 fp32)
constexpr uint32_t kChScratch = kChConsts + 2048;
constexpr uint32_t kChSmemTotal = kChScratch + 1024;

struct ChainScratch {
  Barriers bars;
  uint64_t a0_full[2];
  uint64_t a0_empty[2];
};
static_assert(sizeof(ChainScratch) <= 1024, "chain scratch");

struct ChainParams {
  PassBufs pass[2];
  const uint8_t* net[2];      // packed images (backward region at kOffBwd, w_sigma in the fp32 region)
  int n_pass;
  long long tiles[2];         // 128-sample tiles visited per pass (probe mode: a subset)
  long long head[2];          // the real pass visits tiles j < head of both passes first (the probe's tiles)
  long long span[2];          // 128-sample tiles of the pass; visit j of a pass is tile j * stride mod span
  long long stride[2];        // coprime to span (so the real pass visits every tile once), ~ span / probe tiles
  const float* lscale;        // [2][kLevels] per-level scales (bwd_scale_kernel)
  unsigned* lamax;            // probe mode: [2][kLevels] maxima of the un-scaled values per level
  int* status;
};

// Visit t of a chain launch -> (pass, tile): the first head[0] + head[1] visits are visits j < head of pass 0,
// then of pass 1, the rest the remaining visits of pass 0, then of pass 1; visit j of a pass is tile
// j * stride mod span.  In probe mode head == tiles, so only the first part exists.
__device__ __forceinline__ long long chain_tile(const ChainParams& p, long long t, int& ps) {
  long long j;
  if (t < p.head[0]) { ps = 0; j = t; }
  else if (t < p.head[0] + p.head[1]) { ps = 1; j = t - p.head[0]; }
  else if (t < p.tiles[0] + p.head[1]) { ps = 0; j = t - p.head[1]; }
  else { ps = 1; j = t - p.tiles[0]; }
  return j * p.stride[ps] % p.span[ps];
}

// One step of the chain for this thread's accumulator (2 rows x 64 columns).
//   kFirst: add the rank-1 sigma-head term
//   ratio = scale of the produced level / scale of the consumed level (a power of two)
//   kProbe: no HBM stores; returns the largest |value| (in units of the produced level's scale)
//   mw[s]: the ReLU sign bits of row s (epi_hidden's layout); h: the result, the next step's A operand
template <bool kFirst, bool kProbe>
__device__ __forceinline__ float chain_epi(const WgCtx& c, uint8_t* dpre, const long long (&g)[2], const uint2 (&mw)[2],
                                           const float (&dsig)[2], const float* wsig, float ratio,
                                           const float (&acc)[128], uint32_t (&h)[64]) {
  float vmax = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    float2 ws = make_float2(0.f, 0.f);
    if (kFirst) ws = *reinterpret_cast<const float2*>(wsig + 8 * j + 2 * c.q);
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      float a = acc[4 * j + 2 * s], b = acc[4 * j + 2 * s + 1];
      if (kFirst) {
        a = fmaf(dsig[s], ws.x, a);
        b = fmaf(dsig[s], ws.y, b);
      }
      a *= ratio;
      b *= ratio;
      const uint32_t bits = (((j >> 4) ? mw[s].y : mw[s].x) >> (2 * (j & 15))) & 3u;
      const uint32_t keep = ((bits & 1u) ? 0u : 0xFFFFu) | ((bits & 2u) ? 0u : 0xFFFF0000u);
      h[2 * j + s] = cvt_bwd_x2(a, b) & keep;
      if (kProbe) {
        if (!(bits & 1u)) vmax = fmaxf(vmax, fabsf(a));
        if (!(bits & 2u)) vmax = fmaxf(vmax, fabsf(b));
      }
    }
  }
  if (!kProbe) {
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int j = 0; j < 32; ++j) *reinterpret_cast<uint32_t*>(dpre + tiled_pair_off(g[s], 8 * j + 2 * c.q, 4)) = h[2 * j + s];
  }
  return vmax;
}

template <bool kProbe>
__device__ __forceinline__ void chain_bwd_body(const ChainParams& p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  ChainScratch* sc = reinterpret_cast<ChainScratch*>(smem + kChScratch);
  Barriers* bars = &sc->bars;
  if (threadIdx.x == 0) {
    for (int b = 0; b < 2; ++b) {
      mbar_init(smem_u32(&sc->a0_full[b]), 1);
      mbar_init(smem_u32(&sc->a0_empty[b]), kConsumerWGs * 4);
    }
  }
  if (!engine_setup(smem, bars)) {
    if (threadIdx.x == 0) report_fault(p.status, 101);
    return;
  }
  float* wsig_s = reinterpret_cast<float*>(smem + kChConsts);
  for (int i = threadIdx.x; i < 512; i += blockDim.x) {
    const int ps = i >> 8;
    wsig_s[i] = (ps < p.n_pass) ? reinterpret_cast<const float*>(p.net[ps] + kHalfRegionBytes)[kF32WSigma + (i & 255)] : 0.f;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long total = p.tiles[0] + (p.n_pass > 1 ? p.tiles[1] : 0);

  if (warp < kConsumerWarp0) {
    regs_dec<kRegsAux>();
    if (warp == kProducerWarp && lane == 0) {
      RingState rs;
      int it = 0;
      for (long long t = blockIdx.x; t < total; t += gridDim.x, ++it) {
        int ps;
        const long long tile = chain_tile(p, t, ps);
        const int b = it & 1;
        // the dd tile: rows 0..63 and 64..127 of column block kb are two 8 KiB blocks of the tiled array
        mbar_wait(smem_u32(&sc->a0_empty[b]), ((it >> 1) & 1) ^ 1, 31);
        const uint32_t full = smem_u32(&sc->a0_full[b]);
        mbar_arrive_expect_tx(full, kChA0Bytes);
        const uint32_t dst = smem_u32(smem + kChA0 + b * kChA0Bytes);
        const uint8_t* dd = p.pass[ps].dd;
#pragma unroll
        for (int kb = 0; kb < 2; ++kb)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
            bulk_g2s(dst + kb * 16384 + hh * 8192, dd + tiled_block_off(static_cast<unsigned long long>(tile * 2 + hh), kb, 2), 8192, full);
        const uint8_t* w = p.net[ps] + kOffBwd;
        for (int i = 0; i < kNumSlicesBwd; ++i) {
          mbar_wait(smem_u32(&bars->empty[rs.stage]), rs.phase ^ 1, 1);
          const uint32_t fl = smem_u32(&bars->full[rs.stage]);
          const uint32_t d2 = smem_u32(smem + kChRing + rs.stage * kSliceBytes256);
          mbar_arrive_expect_tx(fl, kSliceBytes256);
          const uint8_t* src = w + static_cast<size_t>(i) * kSliceBytes256;
#pragma unroll
          for (int cc = 0; cc < 4; ++cc) bulk_g2s(d2 + cc * 8192, src + cc * 8192, 8192, fl);
          rs.advance();
        }
      }
    }
  } else {
    regs_inc<kRegsConsumer>();
    WgCtx c;
    wg_init(c, smem, bars);
    const uint64_t ring_desc = make_desc_sw128(smem_u32(smem + kChRing));
    float acc[128];
    uint32_t h[64];
    float amx[2][8];      // probe mode only: per pass and level, in un-scaled units
#pragma unroll
    for (int i = 0; i < 8; ++i) { amx[0][i] = 0.f; amx[1][i] = 0.f; }
    int it = 0;
    for (long long t = blockIdx.x; t < total; t += gridDim.x, ++it) {
      int ps;
      const long long tile = chain_tile(p, t, ps);
      const int b = it & 1;
      const PassBufs& pb = p.pass[ps];
      const long long g[2] = {tile * 128 + c.row[0], tile * 128 + c.row[1]};
      const float* ls = p.lscale + ps * kLevels;
      float sc_in = ls[0];
      const float dsig[2] = {pb.dsigma[g[0]] * sc_in, pb.dsigma[g[1]] * sc_in};
      const float* wsig = wsig_s + ps * 256;
      float sc_out = ls[1];
      auto masks = [&](int idx, uint2 (&mw)[2]) {
#pragma unroll
        for (int s = 0; s < 2; ++s) mw[s] = __ldg(pb.mask + (static_cast<long long>(idx) * pb.n_pad + g[s]) * 4 + c.q);
      };
      auto dpre_of = [&](int idx) { return pb.dpre + static_cast<long long>(idx) * pb.n_pad * 512; };
      uint2 mw[2];
      masks(7, mw);
      mbar_wait(smem_u32(&sc->a0_full[b]), (it >> 1) & 1, 9);
      mma_layer<5>(c, acc, h, make_desc_sw128(smem_u32(smem + kChA0 + b * kChA0Bytes + c.wg * 8192)), ring_desc);
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&sc->a0_empty[b]));
      float m = chain_epi<true, kProbe>(c, dpre_of(7), g, mw, dsig, wsig, sc_out / sc_in, acc, h);
      if (kProbe) amx[ps][0] = fmaxf(amx[ps][0], m / sc_out);
      const float zero[2] = {0.f, 0.f};
#pragma unroll 1
      for (int s = 1; s < kChainSteps; ++s) {
        sc_in = sc_out;
        sc_out = ls[s + 1];
        masks(7 - s, mw);
        mma_layer<1>(c, acc, h, 0ull, ring_desc);
        m = chain_epi<false, kProbe>(c, dpre_of(7 - s), g, mw, zero, nullptr, sc_out / sc_in, acc, h);
        if (kProbe) amx[ps][s] = fmaxf(amx[ps][s], m / sc_out);
      }
    }
    if (kProbe) {
#pragma unroll
      for (int ps = 0; ps < 2; ++ps)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float v = amx[ps][i];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
          if (lane == 0 && v > 0.f && v < 3e38f) atomicMax(p.lamax + ps * kLevels + 1 + i, __float_as_uint(v));
        }
    }
  }
}
template <bool kProbe>
__global__ void __launch_bounds__(kThreads, 1) chain_bwd_kernel(const ChainParams p) { chain_bwd_body<kProbe>(p); }
// The same with its parameters planned on the device: launched at the grid of the carved worst case, a CTA whose
// first visit is past the plan's tiles visits none.
template <bool kProbe>
__global__ void __launch_bounds__(kThreads, 1) chain_bwd_dev_kernel(const ChainParams* __restrict__ p) {
  chain_bwd_body<kProbe>(*p);
}

// ------------------------------------------------------------------------------------ wgrad
// gW = A^T B over a range of 64-sample chunks:  A = a 16-bit gradient array (dpre_l or dd), B = an
// fp16 activation array (h_{l-1} or the encoded input), both in the tiled layout, i.e. already the
// MN-major SWIZZLE_128B operand image, so a chunk is staged with two plain bulk copies and the
// tensor core contracts over the samples.  The output rows are taken 128 at a time ("halves" of
// M = 256): per half and chunk, consumer warpgroup w accumulates
//   D_w[64 x N] += A[:, 64 (2 half + w) ..]^T[64 x 64] . B[64 x N]      4 x wgmma (K = 16 samples)
// in registers over one piece (a range of chunks) and writes it out, or adds it in fp32 to what the CTA's earlier
// pieces wrote, as the CTA's partial, which wgrad_reduce_kernel sums with the other CTAs' partials in a fixed
// order.  The kernel is HBM-bound by construction: the point of
// the layout is that it reads the operands with no transposition pass and no staging through
// registers.  Two more warps reduce the same shared-memory tiles on the CUDA cores: column sums of A
// (the bias gradients).
constexpr int kWgStages = 3;
constexpr uint32_t kWgABytes = 16384;                  // two column blocks of A
constexpr uint32_t kWgStageBytes = kWgABytes + 32768;  // A half + B chunk (<= 32 KiB)
constexpr uint32_t kWgScratch = kWgStages * kWgStageBytes;
constexpr uint32_t kWgSmemTotal = kWgScratch + 1024;
constexpr int kWgThreads = 3 * 128;                    // warpgroup 0: producer (warp 0), reductions (warps 2, 3)
constexpr int kWgReduceWarp0 = 2;

struct WgradJob {          // one piece: a (pass, layer) GEMM over a contiguous range of 64-sample chunks
  const uint8_t* a;        // tiled (n_pad, 64 a_fb) 16-bit gradient array
  const uint8_t* b;        // tiled (n_pad, 64 b_fb) fp16 activation array
  int a_fb;                // column blocks of A: 4 (M = 256, two halves) or 2 (M = 128)
  int b_fb;                // column blocks of B: N = 64 b_fb
  int chunk0, chunk1;      // 64-sample chunks chunk0, chunk0 + chunk_step, ... < chunk1
  int chunk_step;          // > 1: the CTAs of one GEMM interleave their chunks (they read one moving window of HBM)
  int add;                 // 1: add into the partial, which the CTA's previous piece wrote; 0: write it
  float* out;              // partial, TRANSPOSED: element (m, n) at out[n * 64 a_fb + m]
  float* bias_out;         // partial column sums of A (64 a_fb) or null
};

struct WgScratch {
  uint64_t full[kWgStages];
  uint64_t empty[kWgStages];
};

// CTA b works through pieces [cta_first[b], cta_first[b + 1]).  The host (capi.cu plan_wgrad) gives every
// (pass, layer) GEMM whole CTAs in proportion to the bytes it streams (at least one per GEMM); the CTAs of one
// GEMM take its chunks round-robin, each its share as consecutive pieces of a bounded length into one partial.
// CTAs do not synchronise with each other, so the grid may run in more than one wave.
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_kernel(const WgradJob* __restrict__ jobs,
                                                               const int* __restrict__ cta_first, int* status) {
  extern __shared__ __align__(1024) uint8_t smem[];
  WgScratch* sc = reinterpret_cast<WgScratch*>(smem + kWgScratch);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if ((smem_u32(smem) & 1023u) != 0) {
    if (threadIdx.x == 0) report_fault(status, 101);
    return;
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < kWgStages; ++i) {
      mbar_init(smem_u32(&sc->full[i]), 1);
      mbar_init(smem_u32(&sc->empty[i]), 8 + 2);     // the consumer warps + the two reduction warps
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int p0 = cta_first[blockIdx.x], p1 = cta_first[blockIdx.x + 1];

  if (warp == 0) {
    if (lane == 0) {
      uint32_t stage = 0, phase = 0;
      for (int pi = p0; pi < p1; ++pi) {
        const WgradJob job = jobs[pi];
        const uint32_t a_bytes = job.a_fb * kTileBlockBytes, b_bytes = job.b_fb * kTileBlockBytes;
        for (int hh = 0; hh < (job.a_fb >> 1); ++hh) {
          for (int c = job.chunk0; c < job.chunk1; c += job.chunk_step) {
            mbar_wait(smem_u32(&sc->empty[stage]), phase ^ 1, 51);
            const uint32_t full = smem_u32(&sc->full[stage]);
            const uint32_t dst = smem_u32(smem + stage * kWgStageBytes);
            mbar_arrive_expect_tx(full, kWgABytes + b_bytes);
            const uint8_t* sa = job.a + static_cast<unsigned long long>(c) * a_bytes + hh * kWgABytes;
            const uint8_t* sb = job.b + static_cast<unsigned long long>(c) * b_bytes;
            bulk_g2s(dst, sa, kWgABytes, full);
            bulk_g2s(dst + kWgABytes, sb, b_bytes, full);
            if (++stage == kWgStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ---- consumer warpgroups: warpgroup w owns output rows 64 (2 hh + w) .. + 63 of half hh
    const int ct = threadIdx.x - 128;
    const int w = ct >> 7, wi = (ct >> 5) & 3, q = lane & 3;
    uint32_t stage = 0, phase = 0;
    float acc[128];
    for (int pi = p0; pi < p1; ++pi) {
      const WgradJob job = jobs[pi];
      const int N = job.b_fb * 64, M = job.a_fb * 64;
      for (int hh = 0; hh < (job.a_fb >> 1); ++hh) {
#pragma unroll
        for (int i = 0; i < 128; ++i) acc[i] = 0.f;
        for (int c = job.chunk0; c < job.chunk1; c += job.chunk_step) {
          mbar_wait(smem_u32(&sc->full[stage]), phase, 52);
          const uint32_t base = smem_u32(smem + stage * kWgStageBytes);
          wgmma_fence();
#pragma unroll
          for (int j = 0; j < 4; ++j) {        // 16 samples = two 8-row groups = 2048 B per K step
            const uint64_t ad = make_desc_mn_sw128(base + w * 8192 + j * 2048, 8192, 1024);
            const uint64_t bd = make_desc_mn_sw128(base + kWgABytes + j * 2048, 8192, 1024);
            if (N == 256) wgmma_n256_ss_mn(acc, ad, bd, 1u);
            else wgmma_n64_ss_mn(reinterpret_cast<float(&)[32]>(acc), ad, bd, 1u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(acc);
          __syncwarp();
          if (lane == 0) mbar_arrive(smem_u32(&sc->empty[stage]));
          if (++stage == kWgStages) { stage = 0; phase ^= 1; }
        }
        // ---- drain: element (m, n) at out[n * M + m].  The element belongs to this thread in every piece of the
        // CTA, so its reductions (no value returned) add in program order: the sum is deterministic
        const int m0 = 64 * (2 * hh + w) + 16 * wi + (lane >> 2);
        if (job.add) {
#pragma unroll
          for (int i = 0; i < 128; ++i) {
            const int n = 8 * (i >> 2) + 2 * q + (i & 1);
            if (n < N) atomicAdd(job.out + static_cast<long long>(n) * M + m0 + 8 * ((i >> 1) & 1), acc[i]);
          }
        } else {
#pragma unroll
          for (int i = 0; i < 128; ++i) {
            const int n = 8 * (i >> 2) + 2 * q + (i & 1);
            if (n < N) job.out[static_cast<long long>(n) * M + m0 + 8 * ((i >> 1) & 1)] = acc[i];
          }
        }
      }
    }
  } else if (warp >= kWgReduceWarp0) {
    // ---- reduction warps.  Column sums of A (the bias gradient): warp wr owns column block 2 hh + wr,
    // lane = (logical 16-byte chunk c = lane % 8, row phase lane / 8): one LDS.128 covers 8 columns of one
    // row, the warp 4 rows (512 B, conflict-free).  8 rows are first summed in fp16 pairs (values are scaled
    // to <= 64, so <= 512; the rounding is far below what the sum over 1e5 samples averages out), then
    // converted and added in fp32 - a sixth of the instructions of a scalar fp32 loop.
    // These warps read every element of every stored gradient level (dd and dpre_1..8 are the A operands of
    // jobs with a bias), so they also check the levels' ranges: an element at the fp16 clamp (a tile whose
    // gradients the probe's scale did not cover, saturated by the chain kernel) or a pre-sum that overflowed
    // makes the weight gradients wrong; it is reported through the status word (code 102), not silently used.
    const int wr = warp - kWgReduceWarp0;
    const uint32_t rc = lane & 7, rph = lane >> 3;
    uint32_t stage = 0, phase = 0;
    __half2 vmax = __float2half2_rn(0.f);      // largest |element| this lane has seen
    bool overflow = false;
    for (int pi = p0; pi < p1; ++pi) {
      const WgradJob job = jobs[pi];
      const bool a_act = job.bias_out != nullptr;
      for (int hh = 0; hh < (job.a_fb >> 1); ++hh) {
        float sa[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) sa[i] = 0.f;
        for (int c = job.chunk0; c < job.chunk1; c += job.chunk_step) {
          mbar_wait(smem_u32(&sc->full[stage]), phase, 53);
          if (a_act) {
            const uint8_t* blk = smem + stage * kWgStageBytes + wr * kTileBlockBytes;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              uint32_t hacc[4] = {0u, 0u, 0u, 0u};
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const uint32_t r = static_cast<uint32_t>((half * 8 + i) * 4) + rph;
                const uint4 v = *reinterpret_cast<const uint4*>(blk + r * 128 + ((rc ^ (r & 7u)) << 4));
                hacc[0] = bwd_add_x2(hacc[0], v.x); hacc[1] = bwd_add_x2(hacc[1], v.y);
                hacc[2] = bwd_add_x2(hacc[2], v.z); hacc[3] = bwd_add_x2(hacc[3], v.w);
                vmax = __hmax2(vmax, __habs2(*reinterpret_cast<const __half2*>(&v.x)));
                vmax = __hmax2(vmax, __habs2(*reinterpret_cast<const __half2*>(&v.y)));
                vmax = __hmax2(vmax, __habs2(*reinterpret_cast<const __half2*>(&v.z)));
                vmax = __hmax2(vmax, __habs2(*reinterpret_cast<const __half2*>(&v.w)));
              }
#pragma unroll
              for (int qq = 0; qq < 4; ++qq) {
                const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hacc[qq]));
                sa[2 * qq] += f.x;
                sa[2 * qq + 1] += f.y;
              }
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(smem_u32(&sc->empty[stage]));
          if (++stage == kWgStages) { stage = 0; phase ^= 1; }
        }
        if (a_act) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {     // the four row phases hold partial sums of the same 8 columns
            sa[i] += __shfl_xor_sync(0xffffffffu, sa[i], 8);
            sa[i] += __shfl_xor_sync(0xffffffffu, sa[i], 16);
            overflow |= !isfinite(sa[i]);
          }
          if (rph == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              float* o = job.bias_out + (2 * hh + wr) * 64 + rc * 8 + i;
              if (job.add) atomicAdd(o, sa[i]);
              else *o = sa[i];
            }
          }
        }
      }
    }
    const float2 vm = __half22float2(vmax);
    overflow |= fmaxf(vm.x, vm.y) >= 65504.f;
    if (__any_sync(0xffffffffu, overflow) && lane == 0) report_fault(status, 102);
  }
}

// ------------------------------------------------------------------- partial sums -> gradients
// out[r][out_col0 + c] = mul * sum_s part[s * split_stride + r * part_ld + c]   (fixed order)
struct ReduceItem {
  const float* part;
  long long split_stride;
  float* out;
  const float* mul;        // device scalar or null (= 1)
  int n_split, rows, cols, part_ld, out_ld, out_col0;
  int transposed;          // partial element (r, c) at part[c * part_ld + r] (wgrad drains) instead of part[r * part_ld + c]
  int by_warp;             // many partials, few outputs: one warp per output, lanes stride over the partials
};
constexpr int kMaxReduceItems = 64;
struct ReduceTable {
  int n;
  ReduceItem it[kMaxReduceItems];
};

__device__ __forceinline__ void reduce_item(const ReduceItem& it) {
  const int total = it.rows * it.cols;
  const float mul = (it.mul != nullptr) ? *it.mul : 1.f;
  if (it.by_warp) {        // fixed order: lane l sums partials l, l + 32, ...; then a butterfly over the lanes
    const int lane = threadIdx.x & 31;
    for (int idx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; idx < total; idx += (gridDim.x * blockDim.x) >> 5) {
      const int r = idx / it.cols, c = idx - r * it.cols;
      const float* src = it.part + static_cast<long long>(r) * it.part_ld + c;
      float acc = 0.f;
      for (int s = lane; s < it.n_split; s += 32) acc += src[s * it.split_stride];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) it.out[static_cast<long long>(r) * it.out_ld + it.out_col0 + c] = acc * mul;
    }
    return;
  }
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    int r, c;
    const float* src;
    if (it.transposed) {       // r fastest: coalesced reads of the transposed partials
      c = idx / it.rows; r = idx - c * it.rows;
      src = it.part + static_cast<long long>(c) * it.part_ld + r;
    } else {
      r = idx / it.cols; c = idx - r * it.cols;
      src = it.part + static_cast<long long>(r) * it.part_ld + c;
    }
    float acc = 0.f;
    for (int s = 0; s < it.n_split; ++s) acc += src[s * it.split_stride];
    it.out[static_cast<long long>(r) * it.out_ld + it.out_col0 + c] = acc * mul;
  }
}
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const __grid_constant__ ReduceTable tab) {
  reduce_item(tab.it[blockIdx.y]);
}
// The same over a table planned on the device (its item count, the grid's y, does not depend on the plan).
__global__ void __launch_bounds__(256) wgrad_reduce_dev_kernel(const ReduceTable* __restrict__ tab) {
  reduce_item(tab->it[blockIdx.y]);
}

// Chain rule through the pack-time folding (layout.h): W' = Wd[:, :256] Wf, b' = Wd[:, :256] bf + bd
//   gWd[:, :256] = gW' Wf^T + gb' (x) bf     gWf = Wd[:, :256]^T gW'     gbf = Wd[:, :256]^T gb'     gbd = gb'
struct UnfoldParams {
  const float* gWp[2];     // (128, 256) gradient of the folded matrix
  const float* gbp[2];     // (128)
  const float* Wf[2];      // live xyz_encoding_final.weight (256,256)
  const float* bf[2];      // (256)
  const float* Wd[2];      // live dir_encoding.0.weight (128,283)
  float* gWd[2];           // (128,283): columns 0..255 written here
  float* gbd[2];           // (128)
  float* gWf[2];           // (256,256)
  float* gbf[2];           // (256)
};
__global__ void __launch_bounds__(256) unfold_kernel(const UnfoldParams p) {
  const int ps = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);       // global warp index
  if (gw < 128 * 256) {
    // gWd[m][j] = sum_n gW'[m][n] Wf[j][n] + gb'[m] bf[j]: one warp per output, both rows read coalesced
    const int m = gw >> 8, j = gw & 255;
    const float* a = p.gWp[ps] + m * 256;
    const float* w = p.Wf[ps] + j * 256;
    float acc = 0.f;
#pragma unroll
    for (int n = lane; n < 256; n += 32) acc = fmaf(a[n], w[n], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
      p.gWd[ps][m * 283 + j] = acc + p.gbp[ps][m] * p.bf[ps][j];
      if (j == 0) p.gbd[ps][m] = p.gbp[ps][m];
    }
    return;
  }
  const int idx = (gw - 128 * 256) * 32 + lane;
  if (idx < 256 * 256) {                              // gWf[j][n] = sum_m Wd[m][j] gW'[m][n]: coalesced over n
    const int j = idx >> 8, n = idx & 255;
    float acc = 0.f;
#pragma unroll 8
    for (int m = 0; m < 128; ++m) acc = fmaf(p.Wd[ps][m * 283 + j], p.gWp[ps][m * 256 + n], acc);
    p.gWf[ps][j * 256 + n] = acc;
  } else if (idx < 256 * 256 + 256) {                 // gbf[j] = sum_m Wd[m][j] gb'[m]
    const int j = idx - 256 * 256;
    float acc = 0.f;
    for (int m = 0; m < 128; ++m) acc = fmaf(p.Wd[ps][m * 283 + j], p.gbp[ps][m], acc);
    p.gbf[ps][j] = acc;
  }
}

// ------------------------------------------------------------------------------------- Adam
// torch.optim.Adam's update (the reference's default optimiser, utils/__init__.py:16-18:
// Adam(lr, eps, weight_decay), betas (0.9, 0.999), no amsgrad) for all parameter tensors of the two
// networks in ONE launch: torch's fused implementation costs two 80 us multi-tensor kernels for
// these 48 small tensors, a fifth of the remaining step.  Adam's update in fp32:
//   g = grad + weight_decay * p;  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2
//   p -= step_size * m / (sqrt(v) / bias2_sqrt + eps)
// step_size = lr / (1 - b1^t) and bias2_sqrt = sqrt(1 - b2^t) are computed on the host in double from the fp32
// hyper-parameters and rounded once (in fp32, 1 - b2^t cancels: ~50 ulps of the update at t = 2..3).  1 - b1 and
// 1 - b2 are exact in fp32.  torch.optim.Adam instead takes 1 - b2 of the unrounded double b2 (0.001 for 0.999,
// where 1 - fp32(0.999) = 0.00099998713), so the two differ by ~1e-5 relative in v; tests/adam_ref.py is the
// float64 model of this kernel that tests/test_gpu_train_loop.py holds it to.
constexpr int kAdamMaxTensors = 64;
struct AdamParams {
  int n_tensors;
  float* p[kAdamMaxTensors];
  const float* g[kAdamMaxTensors];
  float* m[kAdamMaxTensors];
  float* v[kAdamMaxTensors];
  int block0[kAdamMaxTensors + 1];     // first block of each tensor (1024 elements per block)
  int numel[kAdamMaxTensors];
  float beta1, beta2, eps, weight_decay, step_size, bias2_sqrt;    // step_size = lr / (1 - b1^t), bias2_sqrt = sqrt(1 - b2^t)
};
// The tensor block blockIdx.x belongs to.
__device__ __forceinline__ int adam_tensor_of_block(const AdamParams& a) {
  int lo = 0, hi = a.n_tensors;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (a.block0[mid] <= static_cast<int>(blockIdx.x)) lo = mid; else hi = mid;
  }
  return lo;
}

// Block blockIdx.x's 1024 elements of tensor t: the update shared by both kernels below.
__device__ __forceinline__ void adam_update_block(const AdamParams& a, int t, float step, float bias2_sqrt) {
  const int base = (static_cast<int>(blockIdx.x) - a.block0[t]) * 1024;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = base + q * 256 + threadIdx.x;
    if (i < a.numel[t]) {
      const float pv = a.p[t][i];
      const float g = a.g[t][i] + a.weight_decay * pv;
      const float m = a.beta1 * a.m[t][i] + (1.f - a.beta1) * g;
      const float v = a.beta2 * a.v[t][i] + (1.f - a.beta2) * g * g;
      a.m[t][i] = m;
      a.v[t][i] = v;
      a.p[t][i] = pv - step * m / (sqrtf(v) / bias2_sqrt + a.eps);
    }
  }
}

__global__ void __launch_bounds__(256) adam_kernel(const __grid_constant__ AdamParams a) {
  adam_update_block(a, adam_tensor_of_block(a), a.step_size, a.bias2_sqrt);
}

// The capturable form (nerfb200_adam_step_dev): lr and each tensor's step count are read from device memory, and the
// bias corrections are formed here in double from the same fp32 values the host path starts from (step_size and
// bias2_sqrt of AdamParams are unused).  Thread 0 forms them once per block.
struct AdamDevParams {
  AdamParams a;
  const float* lr;                           // device fp32 scalar
  const float* step[kAdamMaxTensors];        // device fp32 step count of each tensor before this update
};
__global__ void __launch_bounds__(256) adam_dev_kernel(const __grid_constant__ AdamDevParams d) {
  __shared__ float corr[2];
  const int t = adam_tensor_of_block(d.a);
  if (threadIdx.x == 0) {
    const double k = static_cast<double>(*d.step[t]) + 1.0;
    corr[0] = static_cast<float>(static_cast<double>(*d.lr) / (1.0 - pow(static_cast<double>(d.a.beta1), k)));
    corr[1] = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(d.a.beta2), k)));
  }
  __syncthreads();
  adam_update_block(d.a, t, corr[0], corr[1]);
}

}  // namespace nerfb200
