// Stand-alone kernels for the individual reference functions on the hot path
// (SURVEY.md section 8a rows a2, a4, a7, a8, a9) and the weight packer.  The render kernel
// fuses all of them; these entries exist so each row has its own parity test and so callers
// that use the pieces directly (extract_color_mesh.py:127-140) have a drop-in.
#pragma once
#include "render_kernel.cuh"

namespace nerfb200 {

// ------------------------------------------------------------ weight packer
struct PackParams {
  const float* p[kNumParams];   // device pointers, order in layout.h
  uint8_t* out;
};

struct PackParams2 {
  PackParams net[2];            // blockIdx.y selects the network: a training step packs both images in one launch
};

// One thread per fp16 element of the slice region, then the fp32 tail.
__global__ void pack_weights_kernel(const __grid_constant__ PackParams2 pp2) {
  const PackParams& pp = pp2.net[blockIdx.y];
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long n_half = kHalfRegionBytes / 2;
  if (idx < n_half) {
    int slice, n, k, N;
    const long long n256 = static_cast<long long>(kNumSlices256) * 256 * 64;
    if (idx < n256) {
      slice = static_cast<int>(idx / (256 * 64));
      const int rem = static_cast<int>(idx % (256 * 64));
      n = rem / 64; k = rem % 64; N = 256;
    } else {
      const long long j = idx - n256;
      slice = kNumSlices256 + static_cast<int>(j / (128 * 64));
      const int rem = static_cast<int>(j % (128 * 64));
      n = rem / 64; k = rem % 64; N = 128;
    }
    // slice -> (weight tensor, input-feature offset, in_features, valid k)
    const float* W; int ld, koff, kvalid;
    if (slice == 0) { W = pp.p[0]; ld = 63; koff = 0; kvalid = 63; }
    else if (slice <= 12) { const int l = 1 + (slice - 1) / 4; W = pp.p[2 * l]; ld = 256; koff = ((slice - 1) % 4) * 64; kvalid = 64; }
    else if (slice == 13) { W = pp.p[8]; ld = 319; koff = 0; kvalid = 63; }
    else if (slice <= 17) { W = pp.p[8]; ld = 319; koff = 63 + (slice - 14) * 64; kvalid = 64; }
    else if (slice <= 29) { const int l = 5 + (slice - 18) / 4; W = pp.p[2 * l]; ld = 256; koff = ((slice - 18) % 4) * 64; kvalid = 64; }
    else if (slice <= 33) { W = nullptr; ld = 0; koff = (slice - 30) * 64; kvalid = 64; }   // fused W' (below)
    else { W = pp.p[18]; ld = 283; koff = 256; kvalid = 27; }
    float v = 0.f;
    if (W == nullptr) {
      // W'[n][koff+k] = sum_m W_dir[n][m] * W_final[m][koff+k]   (fp32, layout.h)
      const float* wd = pp.p[18] + static_cast<long long>(n) * 283;
      const float* wf = pp.p[16] + koff + k;
      float acc = 0.f;
#pragma unroll 16
      for (int m = 0; m < 256; ++m) acc = fmaf(wd[m], wf[static_cast<long long>(m) * 256], acc);
      v = acc;
    } else if (k < kvalid) {
      v = W[static_cast<long long>(n) * ld + koff + k];
    }
    const uint32_t base = (slice < kNumSlices256) ? slice * kSliceBytes256
                                                   : kOffDir + (slice - kNumSlices256) * kSliceBytes128;
    (void)N;
    *reinterpret_cast<__half*>(pp.out + base + sw128_off(n, k)) = __float2half_rn(v);
    return;
  }
  const long long f = idx - n_half;
  if (f >= kF32Count) {
    // ---- backward region (layout.h): transposed slices B[n][k] = W[k0 + k][n0 + n], 16-bit
    const long long e = f - kF32Count;
    if (e >= static_cast<long long>(kNumSlicesBwd) * 256 * 64) return;
    const int slice = static_cast<int>(e / (256 * 64));
    const int rem = static_cast<int>(e % (256 * 64));
    const int k = rem / 256, n = rem % 256;       // n fastest: the reads below are coalesced over n
    float v;
    if (slice < 2) {
      // W'[m][n] = sum_j W_dir[m][j] W_final[j][n], m = slice * 64 + k
      const float* wd = pp.p[18] + static_cast<long long>(slice * 64 + k) * 283;
      const float* wf = pp.p[16] + n;
      float acc = 0.f;
#pragma unroll 16
      for (int j = 0; j < 256; ++j) acc = fmaf(wd[j], wf[static_cast<long long>(j) * 256], acc);
      v = acc;
    } else {
      const int step = (slice - 2) / 4, kb = (slice - 2) % 4;
      const int L = 8 - step;                                   // xyz_encoding_L, L = 8 .. 2
      const int ld = (L == 5) ? 319 : 256, n0 = (L == 5) ? 63 : 0;
      v = pp.p[2 * (L - 1)][static_cast<long long>(kb * 64 + k) * ld + n0 + n];
    }
    *reinterpret_cast<__half*>(pp.out + kOffBwd + static_cast<uint32_t>(slice) * kSliceBytes256 + sw128_off(n, k)) =
        __float2half_rn(v);
    return;
  }
  float* o = reinterpret_cast<float*>(pp.out + kHalfRegionBytes);
  float v = 0.f;
  const int i = static_cast<int>(f);
  if (i < kF32WSigma) {
    const int l = i / 256, n = i % 256;
    if (l < 8) v = pp.p[2 * l + 1][n];
    else if (n < 128) {
      // b'[n] = b_dir[n] + sum_m W_dir[n][m] * b_final[m]
      float acc = pp.p[19][n];
      const float* wd = pp.p[18] + static_cast<long long>(n) * 283;
      for (int m = 0; m < 256; ++m) acc = fmaf(wd[m], pp.p[17][m], acc);
      v = acc;
    }
  } else if (i < kF32BSigma) v = pp.p[20][i - kF32WSigma];
  else if (i < kF32WRgb) v = (i == kF32BSigma) ? pp.p[21][0] : 0.f;
  else if (i < kF32BRgb) v = pp.p[22][i - kF32WRgb];
  else if (i < kF32WDirPart) v = (i - kF32BRgb < 3) ? pp.p[23][i - kF32BRgb] : 0.f;
  else {
    const int j = i - kF32WDirPart;
    const int k = j / 128, n = j % 128;          // transposed: coalesced over n
    v = (k < 27) ? pp.p[18][static_cast<long long>(n) * 283 + 256 + k] : 0.f;
  }
  o[i] = v;
}

// ------------------------------------------------ NeRF.forward (models/nerf.py:83-124)
// The row DirSrc reads in raw-position mode with stride 0: 63 unused xyz columns, then Embedding(3, 4) of the
// direction (0, 0, 0) (extract_mesh.ipynb's dir_ = zeros): [0 0 0, sin 0 x3, cos 0 x3, ...], exactly 0 and 1 in fp16.
struct ZeroDirRow {
  float v[kEncXyz + kEncDir];
};
constexpr ZeroDirRow make_zero_dir_row() {
  ZeroDirRow r{};
  for (int k = 0; k < (kEncDir - 3) / 6; ++k)
    for (int c = 0; c < 3; ++c) r.v[kEncXyz + 3 + 6 * k + 3 + c] = 1.f;
  return r;
}
__device__ const ZeroDirRow kZeroDirRow = make_zero_dir_row();

struct MlpParams {
  int raw_xyz;             // 1: x is (n, x_stride>=3) raw positions, encoded in-kernel; with sigma_only = 0 the
                           // direction is (0, 0, 0) (kZeroDirRow)
  const float* x;          // (n, x_stride): embedded xyz (63) [+ embedded dir (27)]
  long long x_stride;
  long long n;
  const uint8_t* net;
  int sigma_only;
  float* out;              // (n, 4) rgb,sigma  or (n, 1) sigma
  int* status;
  // training save mode (kSave; x embedded, not sigma_only): what nerfb200_nerf_backward reads, in the formats of
  // the render path's training workspace (PassBufs: enc, act, mask, d, sigma, rgb; one pass, one sample per row)
  PassBufs tr;
  uint8_t* xdir;           // tiled (n_pad, 64) fp16: the direction rows of the direction layer's extra K slice
  // compacted-sample mode (row_ray non-null, plain instantiation): row i is the sample at depth row_z[i] of ray
  // row_ray[i] of `rays`, encoded by encode_row as the render kernel encodes it; with sigma_only = 0 its direction
  // bias is the 128 floats at dirbias + row_ray[i] * kSkipDirStride (csrc/sample_skip_kernels.cuh), as the render
  // kernel's per-ray dirbias.  x is unused.
  const int* row_ray;
  const float* row_z;
  const float* rays;       // (., 8) [o, d, near, far]
  const float* dirbias;
  // compacted-sample training mode (kRowsSave): the fp16 direction row of each ray, (., 64) [Embedding(3, 4)(d), 0..]
  const __half* dirrow;
  // and the row count: *n_dev rows (the launch is sized for p.n, the carved worst case); tr.n_pad is derived from it
  const long long* n_dev;
  // SH mode (kSh; raw_xyz): the table of sh_table_kernel (kShTableFloats), out is (n, kShOut)
  const float* sh;
};
constexpr int kSkipDirStride = 2 * kDirW;   // per ray: the coarse network's direction bias, then the fine one's

// kSave: also stores per sample the encoded input rows, the 8 activations and their ReLU sign bits, the direction-layer
// output, the direction rows and raw sigma / rgb.  The returned values are those of the plain instantiation, bit for bit
// (the save mode only adds stores).
// kRowsSave (with kSave): the compacted-sample mode with the same stores, for training with empty samples skipped
// (csrc/train_skip_kernels.cuh).  The direction still enters through the per-ray fp32 bias, so the values are the
// compacted-sample mode's; xdir receives the row's ray's direction row, so that the direction-slice wgrad GEMM yields
// gW_dir[:, 256:283].  Padding rows of the last tile are stored as copies of row n - 1 (their gradient is 0), so every
// row below n_pad is written by this launch whatever an earlier, longer launch left in the workspace.  Its row count is
// read on the device (n_dev), so a CUDA graph can capture the launch; CTAs past the count's tiles write nothing.
// kSh (raw positions, not kSave): the SH mode of DESIGN.md §10k.  One trunk pass and the direction layer's MMAs per
// row, then per direction of the table its rgb and the projection (epi_sh); out receives kShOut floats per row.
template <bool kSave, bool kRowsSave = false, bool kSh = false>
__global__ void __launch_bounds__(kThreads, 1) mlp_forward_kernel(const MlpParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  Scratch* sc = reinterpret_cast<Scratch*>(smem + kSmemScratch);
  Barriers* bars = &sc->bars;
  if (!engine_setup(smem, bars)) {
    if (threadIdx.x == 0) report_fault(p.status, 101);
    return;
  }
  load_consts(smem, 0, p.net);
  if constexpr (kSh) {
    float4* dst = reinterpret_cast<float4*>(smem + kSmemSh);
    for (int i = threadIdx.x; i < kShTableFloats / 4; i += blockDim.x) dst[i] = __ldg(reinterpret_cast<const float4*>(p.sh) + i);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const long long n_rows = kRowsSave ? *p.n_dev : 0;     // (kRowsSave ? n_rows : p.n) is the row count
  const long long n_tiles = ((kRowsSave ? n_rows : p.n) + 127) / 128;
  const bool so = p.sigma_only != 0;
  const bool rows = kRowsSave || (!kSave && p.row_ray != nullptr);
  if (warp < kConsumerWarp0) {
    regs_dec<kRegsAux>();
    if (warp == kProducerWarp && lane == 0) {
      RingState rs;
      for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) produce_tile(rs, smem, bars, p.net, so, !so && !rows && !kSh);
    }
  } else {
    regs_inc<kRegsConsumer>();
    WgCtx c;
    wg_init(c, smem, bars);
    c.cst = consts_ptr(smem, 0);
    const float* b_dir = c.cst + kF32Bias + 8 * 256;      // b' (the direction part goes through the tensor core)
    const float* const dbias[2] = {b_dir, b_dir};
    uint8_t* enc = smem + kSmemEnc;
    const int t = c.wi * 32 + c.lane;
    if (kSave) {
      c.save_act = p.tr.act;
      c.save_mask = p.tr.mask;
      c.save_d = p.tr.d;
      c.save_n = kRowsSave ? n_tiles * 128 : p.tr.n_pad;
    }
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      // this warpgroup's 64 rows of the ENC tile: two threads per row (the previous tile's MMAs that read
      // them have completed: every layer ends with wgmma.wait_group 0)
      {
        const int row = 64 * c.wg + (t >> 1);
        const long long gi = min(tile * 128 + row, (kRowsSave ? n_rows : p.n) - 1);
        const float* xr = p.x + gi * p.x_stride;
        if (rows) {
          // a sample of a ray, as the render kernel encodes it (its helper warps' encode_row)
          const long long ri = __ldg(p.row_ray + gi);
          const float* ray = p.rays + ri * 8;
          const float o[3] = {__ldg(ray), __ldg(ray + 1), __ldg(ray + 2)};
          const float d[3] = {__ldg(ray + 3), __ldg(ray + 4), __ldg(ray + 5)};
          const float z = __ldg(p.row_z + gi);
          for (int part = (t & 1) * 2; part < (t & 1) * 2 + 2; ++part) encode_row(enc, row, part, o, d, z);
          if (kRowsSave) {
            // the row's two threads (adjacent lanes) wrote interleaved columns; each then stores its four 16-byte
            // chunks of the encoded row and of the ray's direction row, in the tile's swizzle
            __syncwarp();
            uint8_t* dst = p.tr.enc + tile * 16384;
            uint8_t* xd = p.xdir + tile * 16384;
            const uint4* dr = reinterpret_cast<const uint4*>(p.dirrow + ri * 64);
#pragma unroll
            for (int cc = 0; cc < 4; ++cc) {
              const uint32_t off = sw128_off(row, ((t & 1) * 4 + cc) * 8);
              *reinterpret_cast<uint4*>(dst + off) = *reinterpret_cast<const uint4*>(enc + off);
              *reinterpret_cast<uint4*>(xd + off) = __ldg(dr + (t & 1) * 4 + cc);
            }
          }
        } else if (p.raw_xyz) {
          // dense-grid sigma query (extract_color_mesh.py:127-140): encode the raw position here
          const float o[3] = {__ldg(xr), __ldg(xr + 1), __ldg(xr + 2)};
          const float zero[3] = {0.f, 0.f, 0.f};
          for (int part = (t & 1) * 2; part < (t & 1) * 2 + 2; ++part) encode_row(enc, row, part, o, zero, 0.f);
        } else {
          for (int k = (t & 1) * 32; k < (t & 1) * 32 + 32; ++k) {
            const float v = (k < kEncXyz) ? __ldg(xr + k) : 0.f;
            *reinterpret_cast<__half*>(enc + sw128_off(row, k)) = __float2half_rn(v);
          }
          if (kSave) {
            // the same copy-in-place of this thread's four 16-byte chunks as write_dir_rows (mlp_engine.cuh),
            // padding rows included
            uint8_t* dst = p.tr.enc + tile * 16384;
#pragma unroll
            for (int cc = 0; cc < 4; ++cc) {
              const uint32_t off = sw128_off(row, ((t & 1) * 4 + cc) * 8);
              *reinterpret_cast<uint4*>(dst + off) = *reinterpret_cast<const uint4*>(enc + off);
            }
          }
        }
        fence_proxy_async();
        wg_bar(c);
      }
      const DirSrc ds = p.raw_xyz ? DirSrc{kZeroDirRow.v, 0, tile * 128, p.n, nullptr}
                                  : DirSrc{p.x, p.x_stride, tile * 128, p.n, kSave ? p.xdir : nullptr};
      float sig[2], rgb[2][3];
      if constexpr (kSh) {
        float coef[2][kShLane];
        wg_tile<false, false, false, true>(c, kSmemEnc, dbias, nullptr, sig, rgb, coef);
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          const long long gi = tile * 128 + c.row[s];
          if (gi >= p.n) continue;
          const float sg = c.cst[kF32BSigma] + sig[s];
          float* o = p.out + gi * kShOut + kShLane * c.q;
#pragma unroll
          for (int i = 0; i < kShLane; ++i) o[i] = (kShLane * c.q + i == 3) ? sg : coef[s][i];
        }
        continue;
      }
      if (rows) {
        const float* rbias[2];
#pragma unroll
        for (int s = 0; s < 2; ++s)
          rbias[s] = p.dirbias + static_cast<long long>(__ldg(p.row_ray + min(tile * 128 + c.row[s],
                                                                             (kRowsSave ? n_rows : p.n) - 1))) *
                                     kSkipDirStride;
        if (kRowsSave) {
#pragma unroll
          for (int s = 0; s < 2; ++s) c.grow[s] = tile * 128 + c.row[s];
          wg_tile<false, false, true>(c, kSmemEnc, rbias, nullptr, sig, rgb);
        } else if (so) {
          wg_tile<true, false, false>(c, kSmemEnc, rbias, nullptr, sig, rgb);
        } else {
          wg_tile<false, false, false>(c, kSmemEnc, rbias, nullptr, sig, rgb);
        }
      } else if (kSave) {
#pragma unroll
        for (int s = 0; s < 2; ++s) c.grow[s] = (tile * 128 + c.row[s] < p.n) ? tile * 128 + c.row[s] : -1;
        wg_tile<false, true, true>(c, kSmemEnc, dbias, &ds, sig, rgb);
      } else if (so) {
        wg_tile<true, false, false>(c, kSmemEnc, dbias, nullptr, sig, rgb);
      } else {
        wg_tile<false, true, false>(c, kSmemEnc, dbias, &ds, sig, rgb);
      }
      if (c.q == 0) {
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          const long long gi = tile * 128 + c.row[s];
          if (gi >= (kRowsSave ? n_rows : p.n)) continue;
          const float sg = c.cst[kF32BSigma] + sig[s];
          if (so && !kSave) {
            p.out[gi] = sg;
          } else {
            float4 o;
            o.x = sigmoid_ref(c.cst[kF32BRgb + 0] + rgb[s][0]);
            o.y = sigmoid_ref(c.cst[kF32BRgb + 1] + rgb[s][1]);
            o.z = sigmoid_ref(c.cst[kF32BRgb + 2] + rgb[s][2]);
            o.w = sg;
            *reinterpret_cast<float4*>(p.out + gi * 4) = o;
            if (kSave) {
              p.tr.sigma[gi] = sg;
              p.tr.rgb[gi * 3 + 0] = o.x;
              p.tr.rgb[gi * 3 + 1] = o.y;
              p.tr.rgb[gi * 3 + 2] = o.z;
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------ the SH mode's table (DESIGN.md §10k)
// The fit's fixed directions (float32 unit vectors) and P = pinv(Y) (row m, column j), made on the host.
struct ShFit {
  float dirs[kShDirs * 3];
  float proj[kShBasis * kShDirs];
};
static_assert(sizeof(ShFit) <= 4000, "ShFit is passed as a kernel parameter");

// One block of kDirW threads per direction j: its bias row, the render path's dir_bias for a ray of direction d_j
// (skip_dir_bias_kernel), and its projection weight per output float (mlp_engine.cuh).
__global__ void __launch_bounds__(kDirW) sh_table_kernel(const __grid_constant__ ShFit fit, const uint8_t* net,
                                                          float* table) {
  __shared__ float direnc[28];
  const int j = blockIdx.x, t = threadIdx.x;
  if (t < 15) dir_embed_term(t, fit.dirs + 3 * j, direnc);
  __syncthreads();
  const float* f32 = reinterpret_cast<const float*>(net + kHalfRegionBytes);
  table[j * kDirW + t] = dir_bias(f32, __ldg(f32 + kF32Bias + 8 * 256 + t), t, direnc);
  if (t < kShOut) table[kShDirs * kDirW + j * kShOut + t] = t == 3 ? 0.f : fit.proj[(t < 3 ? 0 : (t - 1) / 3) * kShDirs + j];
}

// ------------------------------------------------ Embedding.forward (models/nerf.py:21-38)
// x: (n, 3) -> out: (n, 3 + 6*n_freqs), channel order [x, sin f0 x, cos f0 x, ...].
__global__ void embed_kernel(const float* __restrict__ x, long long n, int n_freqs,
                             float* __restrict__ out) {
  const int C = 3 + 6 * n_freqs;
  const long long total = n * C;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = idx / C;
    const int ch = static_cast<int>(idx - r * C);
    float v;
    if (ch < 3) {
      v = x[r * 3 + ch];
    } else {
      const int j = ch - 3;
      const int k = j / 6, fn = (j % 6) / 3, c = j % 3;
      const float a = __fmul_rn(exp2f(static_cast<float>(k)), x[r * 3 + c]);
      v = fn ? cosf(a) : sinf(a);
    }
    out[idx] = v;
  }
}

// ------------------------------------------------ searchsorted (torchsearchsorted)
// res[r, c] = #{k : a[r,k] <  v[r,c]} (side='left') or #{k : a[r,k] <= v[r,c]} ('right');
// a or v may have a single row that is broadcast (searchsorted.py:23-35, kernel.cu:83-107).
__global__ void searchsorted_kernel(const float* __restrict__ a, const float* __restrict__ v,
                                    long long* __restrict__ res, long long nrow_a, long long nrow_v,
                                    int ncol_a, int ncol_v, int side_right) {
  const long long nrow = nrow_a > nrow_v ? nrow_a : nrow_v;
  const long long total = nrow * ncol_v;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = idx / ncol_v;
    const int c = static_cast<int>(idx - r * ncol_v);
    const float* ar = a + (nrow_a == 1 ? 0 : r) * ncol_a;
    const float val = v[(nrow_v == 1 ? 0 : r) * ncol_v + c];
    int lo = 0, hi = ncol_a;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      const float x = __ldg(ar + mid);
      const bool go_right = side_right ? (x <= val) : (x < val);
      if (go_right) lo = mid + 1; else hi = mid;
    }
    res[idx] = lo;
  }
}

// ------------------------------------------------ sample_pdf (models/rendering.py:14-55)
// bins (R, nb = nw+1), weights (R, nw), u (R, K) sorted or not; out (R, K).  One warp per ray.
constexpr int kPdfWarps = 4;             // warps (rays in flight) per block
constexpr int kPdfMaxWeights = 4096;     // nw <= 4096: kPdfWarps cdfs of nw + 1 floats, 64 KB of shared memory
__global__ void sample_pdf_kernel(const float* __restrict__ bins, const float* __restrict__ weights,
                                  const float* __restrict__ u, long long n_rays, int nw, int K,
                                  float* __restrict__ out) {
  extern __shared__ float sh[];
  const int wpb = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* cdf = sh + warp * (nw + 1);
  for (long long r = static_cast<long long>(blockIdx.x) * wpb + warp; r < n_rays;
       r += static_cast<long long>(gridDim.x) * wpb) {
    const float* w = weights + r * nw;
    const float* b = bins + r * (nw + 1);
    float part = 0.f;
    for (int i = lane; i < nw; i += 32) part += __fadd_rn(w[i], 1e-5f);
    const float total = warp_sum(part);
    if (lane == 0) {
      float run = 0.f;
      cdf[0] = 0.f;
      for (int i = 0; i < nw; ++i) {
        run = __fadd_rn(run, __fdiv_rn(__fadd_rn(w[i], 1e-5f), total));
        cdf[i + 1] = run;
      }
    }
    __syncwarp();
    for (int j = lane; j < K; j += 32) {
      const float uj = u[r * K + j];
      int lo = 0, hi = nw + 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cdf[mid] <= uj) lo = mid + 1; else hi = mid;
      }
      const int below = max(lo - 1, 0), above = min(lo, nw);
      const float c0 = cdf[below], c1 = cdf[above];
      float denom = __fsub_rn(c1, c0);
      if (denom < 1e-5f) denom = 1.f;
      const float t = __fdiv_rn(__fsub_rn(uj, c0), denom);
      out[r * K + j] = __fadd_rn(b[below], __fmul_rn(t, __fsub_rn(b[above], b[below])));
    }
    __syncwarp();
  }
}

// ------------------------------------------------ volume rendering (models/rendering.py:143-170)
// sigmas (R,S), rgbs (R,S,3) nullable, z (R,S), dirs (R,3), noise (R,S) nullable.
// One warp per ray.  S % 32 == 0, S <= 192.
__global__ void composite_kernel(const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                                 const float* __restrict__ z, const float* __restrict__ dirs,
                                 const float* __restrict__ noise, float noise_std, int white_back,
                                 long long n_rays, int S, float* __restrict__ weights,
                                 float* __restrict__ rgb_out, float* __restrict__ depth_out,
                                 float* __restrict__ opac_out) {
  extern __shared__ float sh[];
  const int wpb = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* base = sh + warp * (6 * S);
  float *sz = base, *ss = base + S, *sr = base + 2 * S, *sg = base + 3 * S, *sb = base + 4 * S,
        *sw = base + 5 * S;
  for (long long r = static_cast<long long>(blockIdx.x) * wpb + warp; r < n_rays;
       r += static_cast<long long>(gridDim.x) * wpb) {
    for (int i = lane; i < S; i += 32) {
      sz[i] = z[r * S + i];
      ss[i] = sigmas[r * S + i];
      if (rgbs != nullptr) {
        sr[i] = rgbs[(r * S + i) * 3 + 0];
        sg[i] = rgbs[(r * S + i) * 3 + 1];
        sb[i] = rgbs[(r * S + i) * 3 + 2];
      }
    }
    __syncwarp();
    const float dx = dirs[r * 3], dy = dirs[r * 3 + 1], dz = dirs[r * 3 + 2];
    const float dn = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    const RayOut o = composite_ray(lane, S, sz, ss, sr, sg, sb, noise ? noise + r * S : nullptr,
                                   noise_std, dn, rgbs != nullptr, sw);
    __syncwarp();
    if (weights != nullptr)
      for (int i = lane; i < S; i += 32) weights[r * S + i] = sw[i];
    if (lane == 0) {
      opac_out[r] = o.opac;
      if (rgbs != nullptr) {
        const float add = white_back ? __fsub_rn(1.f, o.opac) : 0.f;
        rgb_out[r * 3 + 0] = o.r + add;
        rgb_out[r * 3 + 1] = o.g + add;
        rgb_out[r * 3 + 2] = o.b + add;
        depth_out[r] = o.depth;
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------ ray generation (datasets/ray_utils.py:5-94)
// One thread per pixel: get_ray_directions (:16-22, no +0.5 pixel centre), get_rays (:41-46:
// rotate by c2w[:, :3], normalise, origin = c2w[:, 3]) and optionally get_ndc_rays (:75-92, as
// datasets/llff.py:236-241 applies it: near plane 1.0, then near/far columns 0/1).
// Writes the (H*W, 8) ray rows [o, d, near, far] the renderer consumes, so rays never cross PCIe.
//
// pixel_ray is the per-pixel body, shared with view_batch_kernel (below): pixel (row j, column i) of an H x W view
// with pose c2w (row-major (3, 4)) -> its ray row, written as two float4 to `out` (16-byte aligned).
__device__ __forceinline__ void pixel_ray(int i, int j, int H, int W, float focal, const float* c2w, float near_in,
                                          float far_in, int ndc, float* out_row) {
  const float dx = __fdiv_rn(static_cast<float>(i) - 0.5f * W, focal);
  const float dy = -__fdiv_rn(static_cast<float>(j) - 0.5f * H, focal);
  const float dz = -1.f;
  float d[3], o[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    d[r] = __fadd_rn(__fadd_rn(__fmul_rn(dx, c2w[4 * r + 0]), __fmul_rn(dy, c2w[4 * r + 1])),
                     __fmul_rn(dz, c2w[4 * r + 2]));
    o[r] = c2w[4 * r + 3];
  }
  const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
#pragma unroll
  for (int r = 0; r < 3; ++r) d[r] = __fdiv_rn(d[r], nrm);
  float near = near_in, far = far_in;
  if (ndc) {
    const float n1 = 1.0f;                                   // llff.py:238 near plane at 1.0
    const float tt = -__fdiv_rn(__fadd_rn(n1, o[2]), d[2]);
#pragma unroll
    for (int r = 0; r < 3; ++r) o[r] = __fadd_rn(o[r], __fmul_rn(tt, d[r]));
    const float ox_oz = __fdiv_rn(o[0], o[2]), oy_oz = __fdiv_rn(o[1], o[2]);
    const float sx = -1.f / (W / (2.f * focal)), sy = -1.f / (H / (2.f * focal));
    const float o0 = sx * ox_oz, o1 = sy * oy_oz, o2 = 1.f + 2.f * n1 / o[2];
    const float d0 = sx * (__fdiv_rn(d[0], d[2]) - ox_oz), d1 = sy * (__fdiv_rn(d[1], d[2]) - oy_oz);
    const float d2 = 1.f - o2;
    o[0] = o0; o[1] = o1; o[2] = o2; d[0] = d0; d[1] = d1; d[2] = d2;
    near = 0.f; far = 1.f;
  }
  float4* out = reinterpret_cast<float4*>(out_row);
  out[0] = make_float4(o[0], o[1], o[2], d[0]);
  out[1] = make_float4(d[1], d[2], near, far);
}

struct RayGenParams {
  int H, W;
  float focal;
  float c2w[12];      // row-major (3, 4)
  float near, far;
  int ndc;
  float* rays;
};
__global__ void generate_rays_kernel(const RayGenParams p) {
  const long long total = static_cast<long long>(p.H) * p.W;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(idx / p.W), i = static_cast<int>(idx - static_cast<long long>(j) * p.W);
    pixel_ray(i, j, p.H, p.W, p.focal, p.c2w, p.near, p.far, p.ndc, p.rays + idx * 8);
  }
}

// ------------------------------------------------ training batches from the views (datasets/blender.py:47-69,
// datasets/llff.py:221-253)
// The reference concatenates every training view's rays and colours into all_rays / all_rgbs, view-major, pixels
// row-major.  Here pixel id p of that order is decoded (64-bit) into (view, row, column): the ray comes from the
// view's pose through pixel_ray, the colour from the view's uint8 pixel as T.ToTensor() makes it (a division by
// 255, not a multiplication by 1/255: torch's CPU div rounds the quotient once), blended onto white for RGBA
// (blender.py:58: rgb * a + (1 - a), three torch ops, three roundings).  An id outside [0, V*H*W) reads nothing
// and gives a NaN row.
struct ViewBatchParams {
  const uint8_t* images;   // (V, H, W, C) uint8
  long long V;
  int H, W, C;             // C: 3 (RGB) or 4 (RGBA)
  const float* c2w;        // (V, 3, 4)
  float focal, near, far;
  int ndc;
  const long long* ids;    // (n,)
  long long n;
  float* rays;             // (n, 8), 16-byte aligned
  float* rgbs;             // (n, 3)
};
__global__ void view_batch_kernel(const ViewBatchParams p) {
  const long long hw = static_cast<long long>(p.H) * p.W;
  const long long total = p.V * hw;
  for (long long k = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; k < p.n;
       k += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long id = __ldg(p.ids + k);
    float* ray = p.rays + k * 8;
    float* rgb = p.rgbs + k * 3;
    if (id < 0 || id >= total) {
      const float nan = __int_as_float(0x7fffffff);
      float4* out = reinterpret_cast<float4*>(ray);
      out[0] = make_float4(nan, nan, nan, nan);
      out[1] = out[0];
      rgb[0] = rgb[1] = rgb[2] = nan;
      continue;
    }
    const long long v = id / hw, rem = id - v * hw;
    const int j = static_cast<int>(rem / p.W), i = static_cast<int>(rem - static_cast<long long>(j) * p.W);
    float c2w[12];
    const float4* pose = reinterpret_cast<const float4*>(p.c2w + v * 12);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float4 row = __ldg(pose + r);
      c2w[4 * r + 0] = row.x; c2w[4 * r + 1] = row.y; c2w[4 * r + 2] = row.z; c2w[4 * r + 3] = row.w;
    }
    pixel_ray(i, j, p.H, p.W, p.focal, c2w, p.near, p.far, p.ndc, ray);
    const uint8_t* px = p.images + id * p.C;
    float c[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) c[ch] = __fdiv_rn(static_cast<float>(__ldg(px + ch)), 255.f);
    if (p.C == 4) {
      const float a = __fdiv_rn(static_cast<float>(__ldg(px + 3)), 255.f);
      const float bg = __fsub_rn(1.f, a);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) c[ch] = __fadd_rn(__fmul_rn(c[ch], a), bg);
    }
    rgb[0] = c[0]; rgb[1] = c[1]; rgb[2] = c[2];
  }
}

// ------------------------------------------------ float image -> uint8 (eval.py:126-128)
// img_pred_ = (clip(img_pred, 0, 1) * 255).astype(uint8)  (truncation, as numpy's astype does)
__global__ void to_uint8_kernel(const float* __restrict__ src, long long n, uint8_t* __restrict__ dst) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = fminf(fmaxf(src[i], 0.f), 1.f) * 255.f;
    dst[i] = static_cast<uint8_t>(v);
  }
}

// ------------------------------------------------ loss / metric epilogue (losses.py:9-14, metrics.py:4-13)
// out[0] = mean((rgb_coarse - t)^2), out[1] = mean((rgb_fine - t)^2) (0 if rgb_fine is null),
// out[2] = out[0] + out[1] (MSELoss.forward), out[3] = -10 log10(mse of the finest available)  (psnr).
// One block, fixed summation order (deterministic).
__global__ void __launch_bounds__(1024, 1) mse_psnr_kernel(const float* __restrict__ rgb_c,
                                                           const float* __restrict__ rgb_f,
                                                           const float* __restrict__ target, long long n_elem,
                                                           float* __restrict__ out) {
  __shared__ double red[2][32];
  double ac = 0.0, af = 0.0;
  for (long long i = threadIdx.x; i < n_elem; i += blockDim.x) {
    const float t = target[i];
    if (rgb_c != nullptr) { const float d = rgb_c[i] - t; ac += static_cast<double>(d) * d; }
    if (rgb_f != nullptr) { const float d = rgb_f[i] - t; af += static_cast<double>(d) * d; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    ac += __shfl_xor_sync(0xffffffffu, ac, o);
    af += __shfl_xor_sync(0xffffffffu, af, o);
  }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = ac; red[1][threadIdx.x >> 5] = af; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sc = 0.0, sf = 0.0;
    for (int w = 0; w < (blockDim.x >> 5); ++w) { sc += red[0][w]; sf += red[1][w]; }
    const float mc = static_cast<float>(sc / static_cast<double>(n_elem));
    const float mf = static_cast<float>(sf / static_cast<double>(n_elem));
    out[0] = mc; out[1] = mf; out[2] = mc + mf;
    out[3] = -10.f * log10f(rgb_f != nullptr ? mf : mc);
  }
}

}  // namespace nerfb200
