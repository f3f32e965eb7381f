// The NeRF MLP (models/nerf.py:83-124) as a warp-specialised wgmma tile engine (sm_90a).
//
// One CTA owns one 128-row tile of samples at a time, split between two consumer warpgroups of 64
// rows each.  The hidden activations never touch shared memory: each layer's fp32 accumulator lives
// in the consumer warpgroup's registers (wgmma m64n256k16), the epilogue applies bias / ReLU in
// place, converts to fp16 and keeps the result in registers as the A operand of the next layer's
// wgmma (the accumulator fragment of columns 16k..16k+15 is exactly the A fragment of K step k).
// Shared memory only holds the encoded-input tile and the weight ring, so its bandwidth is spent
// on weights alone.
//
//   warpgroup 0   warp 0: weight producer, streams the packed 32 KiB K-slices (layout.h) through a
//                 3-stage ring with cp.async.bulk + mbarriers; the other warps are free for the
//                 kernel's own helpers (render kernel) or idle
//   warpgroups 1, 2   consumers: rows 0..63 / 64..127 of the tile, wgmma M=64, N=256|128, K=16; A from
//                 registers for hidden K blocks, from the ENC shared-memory tile for the
//                 encoded-input slices.  Both consume every slice; a stage is refilled once all
//                 eight consumer warps have released it.
//   setmaxnreg moves registers from warpgroup 0 to the consumers (128 accumulator + 64 operand
//   registers per thread).
//   smem also keeps the fp32 biases and head weights of both networks resident (24 KiB), so the
//   epilogue reads them with broadcast LDS instead of L1/L2 loads
#pragma once
#include <cuda_fp16.h>

#include "layout.h"
#include "ptx.cuh"

namespace nerfb200 {

constexpr int kConsumerWGs = 2;
constexpr int kConsumerThreads = kConsumerWGs * 128;    // 256
constexpr int kConsumerWarp0 = 4;
constexpr int kProducerWarp = 0;
constexpr int kThreads = (1 + kConsumerWGs) * 128;     // 384
// 168 registers per thread at launch (one CTA of 384 threads per SM); warpgroup 0 gives up
// 168 - kRegsAux per thread, the consumers take it: kRegsAux + 2 kRegsConsumer <= 3 * 168.
constexpr int kRegsAux = 56;
constexpr int kRegsConsumer = 224;
static_assert(kRegsAux + 2 * kRegsConsumer <= 3 * 168, "setmaxnreg budget");
constexpr int kWgBar0 = 4;                  // named barriers 4, 5: consumer warpgroup 0 / 1 (128 threads each)
// Ring depth 3: the weights come from L2 and one slice of look-ahead per consumer is enough; the rest of
// shared memory holds the second ENC tile and the per-group state of the render kernel's helper warps.
#ifndef NERFB200_STAGES
#define NERFB200_STAGES 3
#endif
constexpr int kStages = NERFB200_STAGES;

constexpr uint32_t kSmemEnc = 0;                     // [128 x 64] fp16     16 KiB
constexpr uint32_t kSmemRing = 16384;                // kStages x 32 KiB
constexpr uint32_t kSmemEnc1 = kSmemRing + kStages * kSliceBytes256;      // second ENC tile (render kernel: double buffer)
constexpr uint32_t kSmemConsts = kSmemEnc1 + 16384;                       // fp32 biases + heads of two networks
constexpr uint32_t kConstFloats = kF32WDirPart;      // biases, sigma head, rgb head of one network
constexpr uint32_t kConstRegion = 24576;
constexpr uint32_t kSmemScratch = kSmemConsts + kConstRegion;
static_assert(2 * kConstFloats * 4 <= kConstRegion, "constants of two networks must fit");
static_assert(kSmemEnc1 % 1024 == 0 && kSmemConsts % 1024 == 0, "SWIZZLE_128B tiles need 1024-byte alignment");
constexpr uint32_t kSmemTotal = 232448;              // 227 KiB (max opt-in)
constexpr uint32_t kScratchBytes = kSmemTotal - kSmemScratch;

struct Barriers {
  uint64_t full[kStages];    // producer -> consumers: slice landed (transaction count)
  uint64_t empty[kStages];   // consumer warps -> producer: slice no longer read
};
static_assert(sizeof(Barriers) % 16 == 0, "Barriers must keep 16-byte alignment of what follows");

struct RingState {
  uint32_t stage = 0, phase = 0;
  __device__ __forceinline__ void advance() {
    if (++stage == kStages) { stage = 0; phase ^= 1; }
  }
};

// ----------------------------------------------------------------- set-up
// Called by all threads at kernel start.  Returns false (uniformly) on misaligned smem.
__device__ __forceinline__ bool engine_setup(uint8_t* smem, Barriers* bars) {
  if ((smem_u32(smem) & 1023u) != 0) return false;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(smem_u32(&bars->full[i]), 1);
      mbar_init(smem_u32(&bars->empty[i]), kConsumerWGs * 4);
    }
    fence_mbar_init();
  }
  __syncthreads();
  return true;
}

// Copy the fp32 constants (biases + heads) of a network image into shared-memory slot `slot`.
// Called by all threads before the first tile; followed by a __syncthreads().
__device__ __forceinline__ void load_consts(uint8_t* smem, int slot, const uint8_t* __restrict__ blob) {
  if (blob == nullptr) return;
  const float4* src = reinterpret_cast<const float4*>(blob + kHalfRegionBytes);
  float4* dst = reinterpret_cast<float4*>(smem + kSmemConsts) + slot * (kConstFloats / 4);
  for (uint32_t i = threadIdx.x; i < kConstFloats / 4; i += blockDim.x) dst[i] = __ldg(src + i);
}
__device__ __forceinline__ const float* consts_ptr(uint8_t* smem, int slot) {
  return reinterpret_cast<const float*>(smem + kSmemConsts) + slot * kConstFloats;
}

// --------------------------------------------------------------- producer
// One thread.  Streams the slices of one network for one tile, in consumption order.
__device__ __forceinline__ void produce_tile(RingState& rs, uint8_t* smem, Barriers* bars,
                                             const uint8_t* __restrict__ blob, bool sigma_only,
                                             bool dir_slice) {
  const int n256 = sigma_only ? kNumSlicesSigmaOnly : kNumSlices256;
  for (int i = 0; i < n256; ++i) {
    mbar_wait(smem_u32(&bars->empty[rs.stage]), rs.phase ^ 1, 1);
    const uint32_t full = smem_u32(&bars->full[rs.stage]);
    const uint32_t dst = smem_u32(smem + kSmemRing + rs.stage * kSliceBytes256);
    mbar_arrive_expect_tx(full, kSliceBytes256);
    const uint8_t* src = blob + static_cast<size_t>(i) * kSliceBytes256;
#pragma unroll
    for (int c = 0; c < 4; ++c) bulk_g2s(dst + c * 8192, src + c * 8192, 8192, full);
    rs.advance();
  }
  if (!sigma_only) {
    const int n128 = dir_slice ? 5 : 4;
    for (int i = 0; i < n128; ++i) {
      mbar_wait(smem_u32(&bars->empty[rs.stage]), rs.phase ^ 1, 2);
      const uint32_t full = smem_u32(&bars->full[rs.stage]);
      const uint32_t dst = smem_u32(smem + kSmemRing + rs.stage * kSliceBytes256);
      mbar_arrive_expect_tx(full, kSliceBytes128);
      const uint8_t* src = blob + kOffDir + static_cast<size_t>(i) * kSliceBytes128;
#pragma unroll
      for (int c = 0; c < 2; ++c) bulk_g2s(dst + c * 8192, src + c * 8192, 8192, full);
      rs.advance();
    }
  }
}

// ----------------------------------------------------------- consumer side
// Per consumer thread: warpgroup wg (0, 1) owns tile rows 64 wg .. 64 wg + 63; accumulator element i
// of the thread is row rows[(i >> 1) & 1], column 8 (i >> 2) + 2 q + (i & 1) (ptx.cuh).
struct WgCtx {
  uint8_t* smem;
  Barriers* bars;
  RingState rs;
  int wg, wi, lane, q;
  int row[2];                      // tile rows of the thread's two accumulator rows
  const float* cst;                // constants of the current network, resident in shared memory
  // training mode ("save"): post-activation outputs of layers 1..8 and of the direction layer are
  // also written to HBM for the backward pass
  uint8_t* save_act;               // 8 x tiled (save_n, 256) fp16 (layout.h), null = off
  uint2* save_mask;                // [8][save_n][4]: ReLU sign bits, 64 per (row, q): see epi_hidden
  uint8_t* save_d;                 // tiled (save_n, 128) fp16: output of dir_encoding
  long long save_n;                // padded rows per layer
  long long grow[2];               // global sample rows of row[0], row[1]; -1 = padding
};

__device__ __forceinline__ void wg_bar(const WgCtx& c) { named_bar_sync(kWgBar0 + c.wg, 128); }

__device__ __forceinline__ void release_stage(const WgCtx& c, uint32_t stage) {
  __syncwarp();
  if (c.lane == 0) mbar_arrive(smem_u32(&c.bars->empty[stage]));
}

// One layer's MMAs for this warpgroup.  kMode: 0 = layer 1 (one slice, A = ENC); 1 = hidden layer (4 slices,
// A = h); 2 = layer 5 (ENC slice, then 4 slices on h); 3 = fused final.dir (N = 128, 4 slices on h);
// 4 = the same plus the direction slice on ENC; 5 = two slices with A from shared memory (backward chain:
// K block kb at a_desc + kb * 16 KiB).
template <int kMode>
__device__ __forceinline__ void mma_layer(WgCtx& c, float (&acc)[128], const uint32_t (&h)[64], uint64_t a_desc,
                                          uint64_t ring_desc) {
  constexpr int n_slices = (kMode == 0) ? 1 : (kMode == 5) ? 2 : (kMode == 2 || kMode == 4) ? 5 : 4;
  constexpr bool kN128 = (kMode == 3 || kMode == 4);
  const uint32_t full0 = smem_u32(&c.bars->full[0]);
  wgmma_fence();
  uint32_t prev = 0;
#pragma unroll
  for (int s = 0; s < n_slices; ++s) {
    const bool from_smem = (kMode == 0) || (kMode == 5) || (kMode == 2 && s == 0) || (kMode == 4 && s == 4);
    const int kb = (kMode == 2) ? s - 1 : s;
    const uint32_t stage = c.rs.stage;
    mbar_wait(full0 + 8u * stage, c.rs.phase, 4);
    const uint64_t bdesc = ring_desc + static_cast<uint64_t>(stage * (kSliceBytes256 >> 4));
    const uint64_t adesc = a_desc + ((kMode == 5) ? static_cast<uint64_t>(kb * (16384 >> 4)) : 0ull);
#pragma unroll
    for (int j = 0; j < 4; ++j) {    // +32 B per K=16 step inside the 128-byte swizzle row
      const uint32_t sd = (s | j) != 0 ? 1u : 0u;
      if (from_smem) {
        if (kN128) wgmma_n128_ss(reinterpret_cast<float(&)[64]>(acc), adesc + 2 * j, bdesc + 2 * j, sd);
        else wgmma_n256_ss(acc, adesc + 2 * j, bdesc + 2 * j, sd);
      } else {
        const uint32_t(&a)[4] = *reinterpret_cast<const uint32_t(*)[4]>(&h[4 * (4 * kb + j)]);
        if (kN128) wgmma_n128_rs(reinterpret_cast<float(&)[64]>(acc), a, bdesc + 2 * j, sd);
        else wgmma_n256_rs(acc, a, bdesc + 2 * j, sd);
      }
    }
    wgmma_commit();
    if (s > 0) {
      wgmma_wait<1>();
      release_stage(c, prev);
    }
    prev = stage;
    c.rs.advance();
  }
  wgmma_wait<0>();
  reg_fence(acc);
  release_stage(c, prev);
}

__device__ __forceinline__ uint32_t cvt_f16x2_relu(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
// torch.relu in fp32: max(v, 0) that keeps a NaN (fmaxf returns 0 for it, which would hand a NaN point a finite
// sigma / rgb made of the biases alone).  Bitwise fmaxf(v, 0.f) for every other v.
__device__ __forceinline__ float relu_keep_nan(float v) {
  float d;
  asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(d) : "f"(v));
  return d;
}
__device__ __forceinline__ uint32_t cvt_f16x2(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}

// Byte offset of the 4-byte pair (row g, columns col, col + 1) in a tiled (n, 64 n_fb) 16-bit array (layout.h).
__device__ __forceinline__ long long tiled_pair_off(long long g, int col, uint32_t n_fb) {
  return static_cast<long long>(tiled_block_off(static_cast<unsigned long long>(g >> 6), static_cast<uint32_t>(col) >> 6, n_fb)) +
         (g & 63) * 128 + ((((static_cast<uint32_t>(col) >> 3) ^ static_cast<uint32_t>(g & 7)) & 7u) << 4) + (col & 7) * 2;
}

// Hidden-layer epilogue: h = relu(acc + bias) as fp16 pairs (h[2 j + s] = row s, columns 8 j + 2 q, +1).
//   kSigma: also the partial sigma head sum (this thread's 64 columns of each row).
//   kSave: HBM copies for the backward - the activations (tiled) and the ReLU sign bits: bit 2 (j & 15) + e of
//   word j >> 4 of the (row, q) entry is the sign of the pre-activation of column 8 j + 2 q + e.
template <bool kSigma, bool kSave>
__device__ __forceinline__ void epi_hidden(WgCtx& c, int l, const float (&acc)[128], uint32_t (&h)[64],
                                           const float* bias, const float* wsig, float (&sig)[2]) {
  uint32_t mk[2][2] = {{0u, 0u}, {0u, 0u}};
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float2 b = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * c.q);
    float2 w = make_float2(0.f, 0.f);
    if (kSigma) w = *reinterpret_cast<const float2*>(wsig + 8 * j + 2 * c.q);
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const float v0 = acc[4 * j + 2 * s] + b.x, v1 = acc[4 * j + 2 * s + 1] + b.y;
      if (kSigma) {
        sig[s] = fmaf(relu_keep_nan(v0), w.x, sig[s]);
        sig[s] = fmaf(relu_keep_nan(v1), w.y, sig[s]);
      }
      if (kSave)
        mk[s][j >> 4] |= ((__float_as_uint(v0) >> 31) << (2 * (j & 15))) | ((__float_as_uint(v1) >> 31) << (2 * (j & 15) + 1));
      h[2 * j + s] = cvt_f16x2_relu(v0, v1);
    }
  }
  if (kSave && c.save_act != nullptr) {
    uint8_t* base = c.save_act + static_cast<long long>(l) * c.save_n * 512;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const long long g = c.grow[s];
      if (g < 0) continue;
#pragma unroll
      for (int j = 0; j < 32; ++j) *reinterpret_cast<uint32_t*>(base + tiled_pair_off(g, 8 * j + 2 * c.q, 4)) = h[2 * j + s];
      c.save_mask[(static_cast<long long>(l) * c.save_n + g) * 4 + c.q] = make_uint2(mk[s][0], mk[s][1]);
    }
  }
}

// dir_encoding epilogue (N=128; accumulator elements 0..63) fused with the rgb head
// (models/nerf.py:119-120): d = relu(acc + dbias[n]); rgb[c] += d * w_rgb[c][n], per row.
// dbias[s] is the per-ray vector (bias + direction part) or b' of the image.
template <bool kSave>
__device__ __forceinline__ void epi_dir(WgCtx& c, const float (&acc)[128], const float* const (&dbias)[2],
                                        const float* wrgb, float (&rgb)[2][3]) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int n = 8 * j + 2 * c.q;
    const float2 wr = *reinterpret_cast<const float2*>(wrgb + n);
    const float2 wg = *reinterpret_cast<const float2*>(wrgb + 128 + n);
    const float2 wb = *reinterpret_cast<const float2*>(wrgb + 256 + n);
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const float2 b = *reinterpret_cast<const float2*>(dbias[s] + n);
      const float v0 = relu_keep_nan(acc[4 * j + 2 * s] + b.x);
      const float v1 = relu_keep_nan(acc[4 * j + 2 * s + 1] + b.y);
      rgb[s][0] = fmaf(v1, wr.y, fmaf(v0, wr.x, rgb[s][0]));
      rgb[s][1] = fmaf(v1, wg.y, fmaf(v0, wg.x, rgb[s][1]));
      rgb[s][2] = fmaf(v1, wb.y, fmaf(v0, wb.x, rgb[s][2]));
      if (kSave && c.save_d != nullptr && c.grow[s] >= 0)
        *reinterpret_cast<uint32_t*>(c.save_d + tiled_pair_off(c.grow[s], n, 2)) = cvt_f16x2(v0, v1);
    }
  }
}

// Where NeRF.forward finds the embedded direction of a row (27 values after the 63 xyz values).
struct DirSrc {
  const float* x;
  long long stride;
  long long row0;      // global row of tile row 0
  long long n;
  uint8_t* save;       // training save mode: tiled (n_pad, 64) fp16 copy of the rows written here, or null
};

// NeRF.forward mode: the ENC tile is dead after layer 5; this warpgroup rewrites its 64 rows with the
// embedded direction (27 values, columns 27..63 zero) for the extra K slice of the direction layer.
__device__ __forceinline__ void write_dir_rows(WgCtx& c, uint32_t enc_off, const DirSrc& ds) {
  uint8_t* enc = c.smem + enc_off;
  const int t = c.wi * 32 + c.lane;
  const int row = 64 * c.wg + (t >> 1);
  const long long gi = min(ds.row0 + row, ds.n - 1);
  const float* src = ds.x + gi * ds.stride + kEncXyz;
  for (int k = (t & 1) * 32; k < (t & 1) * 32 + 32; ++k) {
    const float v = (k < kEncDir) ? __ldg(src + k) : 0.f;
    *reinterpret_cast<__half*>(enc + sw128_off(row, k)) = __float2half_rn(v);
  }
  if (ds.save != nullptr) {
    // the tile's 128 rows are chunks 2 tile, 2 tile + 1 of the tiled array, whose 128-byte rows carry the same
    // swizzle as the shared-memory tile: copy this thread's four 16-byte chunks (its own stores above) in place.
    // Padding rows (copies of row n - 1) are stored too: the array is padded to whole tiles, and their gradient is 0
    uint8_t* dst = ds.save + ds.row0 * 128;
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const uint32_t off = sw128_off(row, ((t & 1) * 4 + cc) * 8);
      *reinterpret_cast<uint4*>(dst + off) = *reinterpret_cast<const uint4*>(enc + off);
    }
  }
  fence_proxy_async();
  wg_bar(c);
}

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

__device__ __forceinline__ float sigmoid_ref(float x) { return 1.f / (1.f + expf(-x)); }

// ---- view-dependent colour (DESIGN.md §10k): degree-2 spherical harmonics fitted over kShDirs fixed directions
constexpr int kShDirs = 64;
constexpr int kShBasis = 9;
constexpr int kShOut = 28;               // floats per point: (c_r0, c_g0, c_b0, sigma), then c_{r,g,b; m}, m = 1..8
constexpr int kShLane = kShOut / 4;      // output floats 7 q .. 7 q + 6 belong to lane q of a quad
// The table of the SH mode, in its workspace and resident in shared memory: [kShDirs][kDirW] direction biases
// (dir_bias of each direction), then [kShDirs][kShOut] the projection weight of each direction per output float
// (P[m, j] for the float holding channel ch of coefficient m; 0 for sigma).
constexpr int kShTableFloats = kShDirs * kDirW + kShDirs * kShOut;
constexpr uint32_t kSmemSh = kSmemScratch + 1024;       // after the Barriers, which is all mlp_forward_kernel keeps there
static_assert(sizeof(Barriers) <= 1024 && 1024 + kShTableFloats * 4 <= kScratchBytes, "SH table must fit the scratch");

// The SH epilogue: acc holds the direction layer's W' h8 without its bias (mma_layer<3>).  For each direction j in
// order its rgb is epi_dir's with the direction's bias row, quad-summed and passed through the sigmoid as in the
// rgb + sigma query (every lane holds it), and each lane accumulates its 7 output floats of both rows.
__device__ __forceinline__ void epi_sh(WgCtx& c, const float (&acc)[128], const float* table,
                                       float (*coef)[kShLane]) {
  const float* wrgb = c.cst + kF32WRgb;
  const float* proj = table + kShDirs * kDirW + kShLane * c.q;
  int ch[kShLane];
#pragma unroll
  for (int i = 0; i < kShLane; ++i) {
    const int o = kShLane * c.q + i;
    ch[i] = o < 3 ? o : (o - 1) % 3;          // o = 3 (sigma) has weight 0
    coef[0][i] = coef[1][i] = 0.f;
  }
#pragma unroll 1
  for (int j = 0; j < kShDirs; ++j) {
    const float* b = table + j * kDirW;
    const float* const db[2] = {b, b};
    float rgb[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    epi_dir<false>(c, acc, db, wrgb, rgb);
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int k = 0; k < 3; ++k) rgb[s][k] = sigmoid_ref(c.cst[kF32BRgb + k] + quad_sum(rgb[s][k]));
#pragma unroll
    for (int i = 0; i < kShLane; ++i) {
      const float w = proj[j * kShOut + i];
#pragma unroll
      for (int s = 0; s < 2; ++s)
        coef[s][i] = fmaf(w, ch[i] == 0 ? rgb[s][0] : ch[i] == 1 ? rgb[s][1] : rgb[s][2], coef[s][i]);
    }
  }
}

// The MLP of one tile for this warpgroup.  Pre-condition: the ENC tile (enc_off) holds the encoded input
// of the warpgroup's rows and is visible to the async proxy.  Returns per row (s = 0, 1) the complete
// sigma-head and rgb-head pre-activation sums without their biases (every lane of the quad holds them).
//   dbias[s]: direction bias vector of row s (smem, 128 floats); kDirSlice: b' from the image, the
//   direction part goes through the tensor core (NeRF.forward mode, ds says where the directions are).
//   kSh: the SH mode; instead of rgb, coef receives this lane's output floats of both rows (epi_sh).
template <bool kSigmaOnly, bool kDirSlice, bool kSave, bool kSh = false>
__device__ __forceinline__ void wg_tile(WgCtx& c, uint32_t enc_off, const float* const (&dbias)[2], const DirSrc* ds,
                                        float (&sig)[2], float (&rgb)[2][3], float (*coef)[kShLane] = nullptr) {
  float acc[128];
  uint32_t h[64];
  const float* bias = c.cst + kF32Bias;
  const float* wsig = c.cst + kF32WSigma;
  const uint64_t enc_desc = make_desc_sw128(smem_u32(c.smem + enc_off + c.wg * 8192));
  const uint64_t ring_desc = make_desc_sw128(smem_u32(c.smem + kSmemRing));
  float dummy[2] = {0.f, 0.f};
  sig[0] = sig[1] = 0.f;
#pragma unroll
  for (int s = 0; s < 2; ++s) rgb[s][0] = rgb[s][1] = rgb[s][2] = 0.f;
  mma_layer<0>(c, acc, h, enc_desc, ring_desc);
  epi_hidden<false, kSave>(c, 0, acc, h, bias, nullptr, dummy);
#pragma unroll 1
  for (int l = 1; l < 7; ++l) {
    if (l == 4) mma_layer<2>(c, acc, h, enc_desc, ring_desc);
    else mma_layer<1>(c, acc, h, enc_desc, ring_desc);
    epi_hidden<false, kSave>(c, l, acc, h, bias + l * 256, nullptr, dummy);
  }
  mma_layer<1>(c, acc, h, enc_desc, ring_desc);
  epi_hidden<true, kSave>(c, 7, acc, h, bias + 7 * 256, wsig, sig);
  if constexpr (kSh) {
    mma_layer<3>(c, acc, h, enc_desc, ring_desc);
    epi_sh(c, acc, reinterpret_cast<const float*>(c.smem + kSmemSh), coef);
  } else if (!kSigmaOnly) {
    if (kDirSlice) {
      write_dir_rows(c, enc_off, *ds);
      mma_layer<4>(c, acc, h, enc_desc, ring_desc);
    } else {
      mma_layer<3>(c, acc, h, enc_desc, ring_desc);
    }
    epi_dir<kSave>(c, acc, dbias, c.cst + kF32WRgb, rgb);
  }
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    sig[s] = quad_sum(sig[s]);
    if (!kSigmaOnly && !kSh) {
      rgb[s][0] = quad_sum(rgb[s][0]);
      rgb[s][1] = quad_sum(rgb[s][1]);
      rgb[s][2] = quad_sum(rgb[s][2]);
    }
  }
}

// Consumer set-up common to the kernels: thread -> (warpgroup, rows).
__device__ __forceinline__ void wg_init(WgCtx& c, uint8_t* smem, Barriers* bars) {
  const int ct = threadIdx.x - kConsumerWarp0 * 32;
  c.smem = smem;
  c.bars = bars;
  c.wg = ct >> 7;
  c.wi = (ct >> 5) & 3;
  c.lane = ct & 31;
  c.q = c.lane & 3;
  c.row[0] = 64 * c.wg + 16 * c.wi + (c.lane >> 2);
  c.row[1] = c.row[0] + 8;
  c.cst = nullptr;
  c.save_act = nullptr; c.save_mask = nullptr; c.save_d = nullptr; c.save_n = 0;
  c.grow[0] = c.grow[1] = -1;
}

}  // namespace nerfb200
