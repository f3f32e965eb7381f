// Packed weight image of one NeRF MLP (reference: models/nerf.py:61-81) as the
// fused kernels consume it.  One image per network (coarse / fine).
//
//  [fp16 region]  K-slices in consumption order.  A slice is a [N x 64] fp16 block in
//                 the UMMA K-major SWIZZLE_128B layout (row n at n*128 B, 16-byte chunk c
//                 at position c ^ (n & 7)), i.e. exactly the shared-memory image, so a
//                 plain 1-D bulk copy (cp.async.bulk) stages it.
//       slice 0        xyz_encoding_1  W[:, 0:63]           (col 63 zero)      N=256
//       slice 1..12    xyz_encoding_2..4, 4 K-blocks each                       N=256
//       slice 13       xyz_encoding_5  W[:, 0:63]  (skip: encoded-input part)   N=256
//       slice 14..17   xyz_encoding_5  W[:, 63:319] (hidden part)               N=256
//       slice 18..29   xyz_encoding_6..8                                        N=256
//       slice 30..33   W' = W_dir[:, 0:256] . W_final   (see below)             N=128
//       slice 34       dir_encoding    W[:, 256:283] (cols 27..63 zero)         N=128
//  [fp32 region]  biases (9 x 256), sigma head, rgb head, dir_encoding W[:, 256:283] transposed.
//
//  xyz_encoding_final has no activation (models/nerf.py:70,116), so it is folded into the
//  direction layer at pack time (fp32):  relu(W_dir . [W_f h + b_f, dir] + b_dir)
//    = relu(W' h + W_dir[:, 256:283] dir + b'),  W' = W_dir[:, 0:256] W_f,  b' = W_dir[:, 0:256] b_f + b_dir.
//  Same function, one 256->128 layer instead of 256->256->128 (65,536 fewer MACs per sample).
#pragma once
#include <cstdint>

namespace nerfb200 {

constexpr int kW = 256;            // hidden width            (models/nerf.py:43 W=256)
constexpr int kEncXyz = 63;        // in_channels_xyz         (models/nerf.py:44)
constexpr int kEncDir = 27;        // in_channels_dir
constexpr int kDirW = 128;         // W//2                    (models/nerf.py:74)

constexpr uint32_t kSliceBytes256 = 256 * 128;   // 32 KiB
constexpr uint32_t kSliceBytes128 = 128 * 128;   // 16 KiB
constexpr int kNumSlices256 = 30;                // layers 1..8
constexpr int kNumSlicesSigmaOnly = 30;          // layers 1..8 only
constexpr int kNumSlices128 = 5;                 // fused final.dir: 4 hidden + 1 direction-part slice

constexpr uint32_t kOffDir = kNumSlices256 * kSliceBytes256;                 //   983,040
constexpr uint32_t kHalfRegionBytes = kOffDir + kNumSlices128 * kSliceBytes128;  // 1,064,960

// fp32 region (offsets in floats from the start of the region)
constexpr int kNumBiasRows = 9;                  // b1..b8, b' (128 used)
constexpr int kF32Bias = 0;                      // [9][256]
constexpr int kF32WSigma = kF32Bias + kNumBiasRows * 256;   // [256]
constexpr int kF32BSigma = kF32WSigma + 256;     // [4]  (1 used)
constexpr int kF32WRgb = kF32BSigma + 4;         // [3][128]
constexpr int kF32BRgb = kF32WRgb + 3 * 128;     // [4]  (3 used)
constexpr int kF32WDirPart = kF32BRgb + 4;       // [28][128] transposed: [j][n] = W_dir[n][256+j] (27 used)
constexpr int kF32Count = kF32WDirPart + 28 * 128;
constexpr uint32_t kFwdBytes = kHalfRegionBytes + kF32Count * 4;

// [backward region]  the transposed ("dgrad") slices the backward chain kernel streams, fp16, in
// consumption order.  A slice is a [256 x 64] K-major
// SWIZZLE_128B block with B[n][k] = W[k0 + k][n0 + n]: n = INPUT feature of the layer (the output
// column of the dgrad GEMM), k = OUTPUT feature (its contraction index).
//       slice 0..1     W'        (128 x 256, the folded final.dir matrix above)  k blocks 0..1
//       slice 2..5     xyz_encoding_8 W      6..9 _7      10..13 _6
//       slice 14..17   xyz_encoding_5 W[:, 63:319]  (only the hidden part carries gradient on)
//       slice 18..21   xyz_encoding_4        22..25 _3    26..29 _2
// xyz_encoding_1 has no dgrad (its input is the encoding).
constexpr int kNumSlicesBwd = 30;
constexpr uint32_t kOffBwd = (kFwdBytes + 1023u) & ~1023u;
constexpr uint32_t kPackedBytes = kOffBwd + kNumSlicesBwd * kSliceBytes256;

// ---- activation / gradient arrays of the training path ("tiled" layout, 16-bit) ----------------
// A (rows, C) array, C a multiple of 64, is stored as 8 KiB blocks [64 rows x 64 columns]; block
// (chunk c = row / 64, column block fb = col / 64) starts at ((c * (C / 64)) + fb) * 8192 bytes and
// is a [64 x 128 B] SWIZZLE_128B image: element (rr, k) at rr * 128 + (((k >> 3) ^ (rr & 7)) << 4) +
// (k & 7) * 2.  This is at the same time
//   * the MN-major UMMA operand image (one 128-byte row per sample = K index, 64 features per
//     row; LBO = 8192 between column blocks, SBO = 1024 between 8-sample groups), which the wgrad
//     kernel reads with plain bulk copies (contraction over samples), and
//   * the K-major UMMA operand image of a [64 rows x 64 K] block, which the backward chain kernel
//     uses for its first A operand (contraction over features).
constexpr uint32_t kTileBlockBytes = 8192;
__host__ __device__ __forceinline__ constexpr unsigned long long tiled_block_off(unsigned long long chunk, uint32_t fb,
                                                                                uint32_t n_fb) {
  return (chunk * n_fb + fb) * static_cast<unsigned long long>(kTileBlockBytes);
}

// Parameter order of the 24 tensors handed to the pack routine
// (state_dict order of models/nerf.py NeRF):
//  0..15  xyz_encoding_{1..8}.0.{weight,bias}
//  16,17  xyz_encoding_final.{weight,bias}
//  18,19  dir_encoding.0.{weight,bias}
//  20,21  sigma.{weight,bias}
//  22,23  rgb.0.{weight,bias}
constexpr int kNumParams = 24;

}  // namespace nerfb200
