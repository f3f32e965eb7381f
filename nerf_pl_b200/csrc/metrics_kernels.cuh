// Image metrics of the reference's eval / validation loop on the device: SSIM as metrics.ssim defines it (kornia
// 0.2.0's published SSIM loss, 3 x 3 Gaussian window) and visualize_depth's JET colouring, bit for bit.
// Definitions, provenance and the BGR channel order: DESIGN.md "Image metrics".
#pragma once
#include <cfloat>
#include <cstdint>
#include <cuda_runtime.h>

#include "jet_lut.h"

namespace nerfb200 {

// ---- 1. SSIM -------------------------------------------------------------------------------------------------
// Pixel i of the (B, C, H, W) map is flat index ((b * C + c) * H + h) * W + w.  Tile t holds pixels
// [t * kSsimTile, (t + 1) * kSsimTile): its sum is formed in a fixed order by one block, so the reduction does not
// depend on how many blocks the grid has.
constexpr int kSsimTile = 256;     // pixels per tile = threads per block
constexpr int kSsimFinishThreads = 1024;

struct SsimParams {
  const float* x;          // image_pred
  const float* y;          // image_gt
  long long xs[4], ys[4];  // element strides along (b, c, h, w)
  long long C, H, W, n;    // n = B * C * H * W
  double g[2];             // the normalised 1-D Gaussian: g[0] off centre, g[1] at the centre
  float* map;              // 'none': the (B, C, H, W) map of 1 - 2 * loss, contiguous; else nullptr
  double* partial;         // 'mean' / 'sum': the loss sum of every tile; else nullptr
};

// kornia 0.2.0's per-pixel loss clamp(1 - ssim_map, 0, 1) / 2, in double.  The window is zero padded: taps outside
// the image add nothing.  A NaN input stays NaN (torch.clamp propagates it).
__device__ __forceinline__ double ssim_loss(const SsimParams& p, long long i) {
  const long long row = i / p.W, plane = row / p.H, b = plane / p.C;
  const long long w = i - row * p.W, h = row - plane * p.H, c = plane - b * p.C;
  const float* xb = p.x + b * p.xs[0] + c * p.xs[1];
  const float* yb = p.y + b * p.ys[0] + c * p.ys[1];
  double m1 = 0.0, m2 = 0.0, s11 = 0.0, s22 = 0.0, s12 = 0.0;
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy) {
    const long long hh = h + dy;
    const bool row_in = hh >= 0 && hh < p.H;
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx) {
      const long long ww = w + dx;
      if (row_in && ww >= 0 && ww < p.W) {
        const double k = (dy == 0 ? p.g[1] : p.g[0]) * (dx == 0 ? p.g[1] : p.g[0]);
        const double a = __ldg(xb + hh * p.xs[2] + ww * p.xs[3]);
        const double v = __ldg(yb + hh * p.ys[2] + ww * p.ys[3]);
        m1 += k * a;
        m2 += k * v;
        s11 += k * (a * a);
        s22 += k * (v * v);
        s12 += k * (a * v);
      }
    }
  }
  constexpr double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03;
  const double mu1_sq = m1 * m1, mu2_sq = m2 * m2, mu1_mu2 = m1 * m2;
  const double sigma1_sq = s11 - mu1_sq, sigma2_sq = s22 - mu2_sq, sigma12 = s12 - mu1_mu2;
  const double ssim_map = ((2.0 * mu1_mu2 + C1) * (2.0 * sigma12 + C2)) /
                          ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2));
  double d = 1.0 - ssim_map;
  d = d < 0.0 ? 0.0 : (d > 1.0 ? 1.0 : d);
  return d / 2.0;
}

// Sum of one value per thread over the block, in a fixed order (blockDim.x a multiple of 32, at most 1024).
__device__ __forceinline__ double block_sum(double v) {
  __shared__ double warp_sums[32];
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int k = 0; k < (blockDim.x >> 5); ++k) s += warp_sums[k];
  __syncthreads();
  return s;       // meaningful in thread 0
}

// At most 64 registers (4 blocks per SM): with the default target ptxas spills around the 64-bit division calls.
__global__ void __launch_bounds__(kSsimTile, 4) ssim_kernel(SsimParams p) {
  const long long tiles = (p.n + kSsimTile - 1) / kSsimTile;
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    const long long i = t * kSsimTile + threadIdx.x;
    const double loss = i < p.n ? ssim_loss(p, i) : 0.0;
    if (p.map != nullptr && i < p.n) p.map[i] = static_cast<float>(1.0 - 2.0 * loss);
    if (p.partial != nullptr) {
      const double s = block_sum(loss);
      if (threadIdx.x == 0) p.partial[t] = s;
    }
  }
}

// metrics.ssim's 'mean' (denom = n) or 'sum' (denom = 1): 1 - 2 * (sum of the tile sums) / denom, one block.
__global__ void __launch_bounds__(kSsimFinishThreads) ssim_finish_kernel(const double* __restrict__ partial,
                                                                         long long tiles, double denom,
                                                                         float* __restrict__ out) {
  double s = 0.0;
  for (long long t = threadIdx.x; t < tiles; t += blockDim.x) s += partial[t];
  s = block_sum(s);
  if (threadIdx.x == 0) *out = static_cast<float>(1.0 - 2.0 * (s / denom));
}

// ---- 2. visualize_depth --------------------------------------------------------------------------------------
// Every step in float32 as numpy takes it (correctly rounded, no contraction): nan_to_num, the min and max of the
// map, y = (x - mi) / (ma - mi + 1e-8f), u = uint8(255 * y) by truncation, then JET[u] / 255 per channel in cv2's
// (B, G, R) order, which ToTensor keeps.
constexpr int kDepthThreads = 256;
constexpr int kDepthItemsPerThread = 8;           // pixels per thread of the min/max pass, before the cap
constexpr int kDepthMinMaxCtas = 148 * 2;         // at most this many partial (min, max) pairs

struct DepthVizParams {
  const float* depth;
  long long H, W, sh, sw;   // element strides of the (H, W) map
  float2* partial;          // (min, max) of each block of the first pass
  int n_partial;
  float* out;               // (3, H, W)
};

__device__ __forceinline__ float nan_to_num(float x) {
  if (x != x) return 0.f;
  if (isinf(x)) return x > 0.f ? FLT_MAX : -FLT_MAX;
  return x;
}

__device__ __forceinline__ float depth_at(const DepthVizParams& p, long long i) {
  return nan_to_num(__ldg(p.depth + (i / p.W) * p.sh + (i % p.W) * p.sw));
}

// (min, max) over the block; min and max are exact, so the order does not matter.
__device__ __forceinline__ float2 block_minmax(float2 v) {
  __shared__ float2 warp_mm[32];
  for (int o = 16; o > 0; o >>= 1) {
    v.x = fminf(v.x, __shfl_xor_sync(0xffffffffu, v.x, o));
    v.y = fmaxf(v.y, __shfl_xor_sync(0xffffffffu, v.y, o));
  }
  if ((threadIdx.x & 31) == 0) warp_mm[threadIdx.x >> 5] = v;
  __syncthreads();
  v = warp_mm[0];
  for (int k = 1; k < (blockDim.x >> 5); ++k) {
    v.x = fminf(v.x, warp_mm[k].x);
    v.y = fmaxf(v.y, warp_mm[k].y);
  }
  __syncthreads();
  return v;       // in every thread
}

__global__ void __launch_bounds__(kDepthThreads) depth_minmax_kernel(DepthVizParams p) {
  const long long n = p.H * p.W;
  float2 v = make_float2(FLT_MAX, -FLT_MAX);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float x = depth_at(p, i);
    v.x = fminf(v.x, x);
    v.y = fmaxf(v.y, x);
  }
  v = block_minmax(v);
  if (threadIdx.x == 0) p.partial[blockIdx.x] = v;
}

__global__ void __launch_bounds__(kDepthThreads) depth_color_kernel(DepthVizParams p) {
  float2 v = make_float2(FLT_MAX, -FLT_MAX);
  for (int k = threadIdx.x; k < p.n_partial; k += blockDim.x) {
    v.x = fminf(v.x, p.partial[k].x);
    v.y = fmaxf(v.y, p.partial[k].y);
  }
  v = block_minmax(v);
  const float mi = v.x, den = __fadd_rn(__fsub_rn(v.y, v.x), 1e-8f);
  const long long n = p.H * p.W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float y = __fdiv_rn(__fsub_rn(depth_at(p, i), mi), den);
    // y is in [0, 1] (a NaN, from a map holding both infinities, is outside the contract and gives 0)
    const unsigned u = __float2uint_rz(__fmul_rn(255.f, y));
    const unsigned char* rgb = nb_jet_lut[u > 255u ? 255u : u];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) p.out[ch * n + i] = __fdiv_rn(static_cast<float>(rgb[ch]), 255.f);
  }
}

}  // namespace nerfb200
