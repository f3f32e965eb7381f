// Early ray termination for renders with empty samples skipped and N_importance = 0 (DESIGN.md §10f).  The coarse
// pass is evaluated front to back in rounds of one mask word (32 samples).  After round k a ray's float64
// transmittance is T_k = T_{k-1} * prod over word k of (1 - alpha_i + 1e-10); the ray is cut at the first k with
// T_k < eps and the samples of its later words are treated as empty (their mask words are cleared, so they are never
// emitted).  Never cut: a plain ray, a pass whose interval lengths are not all finite, and a NaN T.
//
// Per chunk of rays:  classify (skip_classify_kernel) -> start -> W x [scan -> emit word k -> coarse MLP -> round k]
// -> final stage.  The final stage gathers each ray's sigma / rgb from its rounds' rows and composites as
// skip_coarse_stage_kernel's K = 0 branch does.  composite_ray's weight of sample i depends on alpha_0..alpha_i only,
// so every sample up to the end of the cut word keeps its weight bit for bit and a ray never cut renders as the
// render without termination.  The per-ray kernels run one warp per ray in grid-stride order, as the other skip
// kernels, so no result depends on the launch shape.
#pragma once
#include "sample_skip_kernels.cuh"

namespace nerfb200 {

// Per-ray state of the rounds, carved from the coarse-only render's unused fine-pass workspace (zf).
struct EarlyStop {
  float eps;
  int words;            // S_c / 32
  double* T;            // (n) transmittance after the rounds so far
  int* state;           // (n) kMarching, kNeverCut, or the word the ray was cut after
  long long* base;      // (words, n) row of the ray's first evaluated sample of word k (written when k has rows)
  int* cut_out;         // nullable (n) the cut word, -1 where not cut
};
constexpr int kMarching = -1, kNeverCut = -2;

// Start: T = 1, the rays that are never cut (plain, or a non-finite interval: classify_ray's test), and the count of
// word 0.
__global__ void __launch_bounds__(kSkipWarps * 32) early_stop_start_kernel(SkipParams p, EarlyStop e) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.Sc;
  for (int r = blockIdx.x * kSkipWarps + warp; r < p.n; r += gridDim.x * kSkipWarps) {
    const SkipRay s = load_skip_ray(p, r);
    bool bad = false;
    for (int i = lane; i < S; i += 32) {
      const float delta =
          (i < S - 1) ? __fsub_rn(z_base(s.near, s.far, i + 1, S, p.use_disp != 0), z_base(s.near, s.far, i, S, p.use_disp != 0))
                      : 1e10f;
      bad |= !isfinite(__fmul_rn(delta, s.dnorm));
    }
    const bool never = s.plain || __any_sync(0xffffffffu, bad);
    if (lane == 0) {
      e.T[r] = 1.0;
      e.state[r] = never ? kNeverCut : kMarching;
      p.cnt[r] = __popc(p.mask[0][static_cast<long long>(r) * kSkipMaskWords]);
    }
  }
}

// Rows of word k: evaluated sample i of ray r goes to row row0 + ofs[r] + (evaluated samples of word k before i).
__global__ void __launch_bounds__(kSkipWarps * 32) early_stop_emit_kernel(SkipParams p, EarlyStop e, int k,
                                                                          long long row0) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = blockIdx.x * kSkipWarps + warp; r < p.n; r += gridDim.x * kSkipWarps) {
    const uint32_t b = p.mask[0][static_cast<long long>(r) * kSkipMaskWords + k];
    const long long pos = row0 + p.ofs[r];
    if (lane == 0) e.base[static_cast<long long>(k) * p.n + r] = pos;
    if ((b >> lane) & 1u) {
      const long long row = pos + __popc(b & ((1u << lane) - 1u));
      const float near = __ldg(p.rays + 8 * r + 6), far = __ldg(p.rays + 8 * r + 7);
      p.row_ray[row] = r;
      p.row_z[row] = z_base(near, far, 32 * k + lane, p.Sc, p.use_disp != 0);
    }
  }
}

// Round k of one ray per warp: the rule on word k (composite_ray's float32 delta |d| and fmaxf(sigma, 0), the product
// and exp in float64), a cut clears the later mask words; then the count of word k + 1 (0 once cut).
__global__ void __launch_bounds__(kSkipWarps * 32) early_stop_round_kernel(SkipParams p, EarlyStop e, int k,
                                                                           int sigma_only) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.Sc;
  for (int r = blockIdx.x * kSkipWarps + warp; r < p.n; r += gridDim.x * kSkipWarps) {
    uint32_t* m = p.mask[0] + static_cast<long long>(r) * kSkipMaskWords;
    int st = e.state[r];
    if (st == kMarching) {
      const uint32_t b = m[k];
      const SkipRay s = load_skip_ray(p, r);
      const int i = 32 * k + lane;
      float delta = (i < S - 1) ? __fsub_rn(z_base(s.near, s.far, i + 1, S, p.use_disp != 0),
                                            z_base(s.near, s.far, i, S, p.use_disp != 0))
                                : 1e10f;
      delta = __fmul_rn(delta, s.dnorm);
      float sg = 0.f;
      if ((b >> lane) & 1u) {
        const long long row = e.base[static_cast<long long>(k) * p.n + r] + __popc(b & ((1u << lane) - 1u));
        sg = sigma_only ? p.mlp_out[row] : p.mlp_out[row * 4 + 3];
      }
      const double a = 1.0 - exp(-(static_cast<double>(delta) * static_cast<double>(fmaxf(sg, 0.f))));
      double f = (1.0 - a) + 1e-10;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) f *= __shfl_xor_sync(0xffffffffu, f, o);
      const double T = e.T[r] * f;
      if (T < static_cast<double>(e.eps)) {
        st = k;
        for (int w = k + 1 + lane; w < e.words; w += 32) m[w] = 0u;
      }
      if (lane == 0) {
        e.T[r] = T;
        e.state[r] = st;
      }
    }
    if (k + 1 < e.words && lane == 0) p.cnt[r] = st >= 0 ? 0 : __popc(m[k + 1]);
  }
}

// Shared memory of one warp of the final stage.
struct alignas(16) EarlyStopScratch {
  float zc[kMaxSc];
  float sigma[kMaxSc];          // overwritten in place by the weights
  float rgb[3][kMaxSc];
};

// Final stage of one ray per warp: sigma / rgb from the rounds' rows (0 where skipped or dropped), then
// skip_coarse_stage_kernel's composite and results with K = 0.
__global__ void __launch_bounds__(kSkipWarps * 32) early_stop_final_kernel(SkipParams p, EarlyStop e) {
  __shared__ EarlyStopScratch scr[kSkipWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  EarlyStopScratch& w = scr[warp];
  const int Sc = p.Sc;
  const bool want_rgb = p.test_time == 0;
  for (long long r = static_cast<long long>(blockIdx.x) * kSkipWarps + warp; r < p.n;
       r += static_cast<long long>(gridDim.x) * kSkipWarps) {
    const uint32_t* m = p.mask[0] + r * kSkipMaskWords;
    const float near = __ldg(p.rays + r * 8 + 6), far = __ldg(p.rays + r * 8 + 7);
    for (int i = lane; i < Sc; i += 32) w.zc[i] = z_base(near, far, i, Sc, p.use_disp != 0);
    for (int k = 0; k < e.words; ++k) {
      const uint32_t b = m[k];
      const int i = 32 * k + lane;
      float sg = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f;
      if ((b >> lane) & 1u) {
        const long long row = e.base[k * p.n + r] + __popc(b & ((1u << lane) - 1u));
        if (want_rgb) {
          const float4 v = *reinterpret_cast<const float4*>(p.mlp_out + row * 4);
          c0 = v.x; c1 = v.y; c2 = v.z; sg = v.w;
        } else {
          sg = p.mlp_out[row];
        }
      }
      w.sigma[i] = sg;
      w.rgb[0][i] = c0; w.rgb[1][i] = c1; w.rgb[2][i] = c2;
      if (p.samples[0] != nullptr)
        *reinterpret_cast<float4*>(p.samples[0] + (r * Sc + i) * 4) = make_float4(c0, c1, c2, sg);
    }
    __syncwarp();
    const RayOut o = composite_ray(lane, Sc, w.zc, w.sigma, w.rgb[0], w.rgb[1], w.rgb[2], nullptr, 0.f,
                                   load_skip_ray(p, static_cast<int>(r)).dnorm, want_rgb, w.sigma);
    __syncwarp();
    store_pass(p, 0, r, lane, Sc, o, want_rgb, w.sigma);
    if (e.cut_out != nullptr && lane == 0) {
      const int st = e.state[r];
      e.cut_out[r] = st >= 0 ? st : -1;
    }
    __syncwarp();
  }
}

}  // namespace nerfb200
