// C ABI of libnerf_pl_b200.so (declarations + reference citations: include/nerf_pl_b200.h).
#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <mutex>
#include <utility>
#include <vector>

#include "../../include/nerf_pl_b200.h"
#include "aux_kernels.cuh"
#include "bwd_kernels.cuh"
#include "mesh_kernels.cuh"
#include "occupancy_kernels.cuh"
#include "metrics_kernels.cuh"
#include "sample_skip_kernels.cuh"
#include "train_skip_kernels.cuh"
#include "density_kernels.cuh"
#include "masked_grid_kernels.cuh"
#include "early_stop_kernels.cuh"
#include "sparse_mc_kernels.cuh"
#include "baked_kernels.cuh"
#include "../../include/nerf_pl_b200_sparse_mc.h"
#include "../../include/nerf_pl_b200_baked.h"
#include "../../include/nerf_pl_b200_baked_sh.h"

#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

using namespace nerfb200;

namespace {

thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

__attribute__((format(printf, 2, 3))) int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  std::vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
int cuda_fail(cudaError_t e, const char* where) {
  return fail(static_cast<int>(e), "%s: %s (%s)", where, cudaGetErrorString(e), cudaGetErrorName(e));
}
#define CUDA_TRY(expr, where)                          \
  do {                                                 \
    cudaError_t e_ = (expr);                           \
    if (e_ != cudaSuccess) return cuda_fail(e_, where); \
  } while (0)
// return the non-zero code of a helper or entry that already recorded its message
#define TRY(expr)                                \
  do {                                           \
    if (const int rc_ = (expr)) return rc_;      \
  } while (0)

// Every kernel launch of the library: enqueue it, count it (nerfb200_launch_count) and report a launch error as
// `where`.  A failed launch returns before the caller enqueues the next one.
template <class... Params, class... Args>
int launch(const char* where, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, void* stream,
           Args&&... args) {
  kernel<<<grid, block, smem, static_cast<cudaStream_t>(stream)>>>(std::forward<Args>(args)...);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), where);
  return 0;
}
// A CUB device algorithm (`e`: its return value) counts as one launch.
int cub_launch(cudaError_t e, const char* where) {
  CUDA_TRY(e, where);
  g_launches++;
  return 0;
}

long long ceil_div(long long a, long long b) { return (a + b - 1) / b; }

struct DeviceInfo {
  int sm_count = 0;
  int cc_major = 0, cc_minor = 0;
  bool attrs_set = false;
  int* status = nullptr;        // device view of the mapped status word below
  volatile int* status_host = nullptr;   // pinned, mapped: the kernels write it, the host polls it without a sync
};

// Read ONCE per process.  NERFB200_MAX_CTAS caps the render kernel's persistent grid and every grid-stride launch
// (grid_blocks), so tests can show that results do not depend on the grid; unset in production.
struct EnvSwitches {
  int max_ctas = 0;
  EnvSwitches() {
    if (const char* mc = std::getenv("NERFB200_MAX_CTAS")) max_ctas = std::atoi(mc);
  }
};
const EnvSwitches& env_switches() {
  static const EnvSwitches e;
  return e;
}

// Grid-stride launches: one block per `per_block` items, at most one wave of 8 CTAs per SM of an H100 (`cap`), at
// most NERFB200_MAX_CTAS, at least one.
constexpr long long kGridStrideCtas = 148 * 8;
int grid_blocks(long long items, int per_block, long long cap = kGridStrideCtas) {
  long long b = ceil_div(items, per_block);
  if (b > cap) b = cap;
  const int env = env_switches().max_ctas;
  if (env > 0 && b > env) b = env;
  return static_cast<int>(b < 1 ? 1 : b);
}

// Lays out a workspace: consecutive buffers from `base`, each rounded up to `align` bytes.  With base == nullptr it
// only sizes the workspace (take returns nullptr); `off` is then the bytes it needs.
struct Carver {
  uint8_t* base;
  size_t off;
  size_t align;
  template <class T = uint8_t>
  T* take(size_t count) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += (count * sizeof(T) + align - 1) / align * align;
    return p;
  }
};

std::mutex g_mu;
DeviceInfo g_dev[64];

int device_info(DeviceInfo** out) {
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev), "cudaGetDevice");
  if (dev < 0 || dev >= 64) return fail(NERFB200_EDEVICE, "device ordinal out of range");
  std::lock_guard<std::mutex> lk(g_mu);
  DeviceInfo& d = g_dev[dev];
  if (d.sm_count == 0) {
    CUDA_TRY(cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev), "attr sm");
    CUDA_TRY(cudaDeviceGetAttribute(&d.cc_major, cudaDevAttrComputeCapabilityMajor, dev), "attr cc");
    CUDA_TRY(cudaDeviceGetAttribute(&d.cc_minor, cudaDevAttrComputeCapabilityMinor, dev), "attr cc minor");
  }
  // the kernels are built for sm_90a (wgmma, setmaxnreg), which only compute capability 9.0 executes
  if (d.cc_major != 9 || d.cc_minor != 0) return fail(NERFB200_EDEVICE, "nerf_pl_b200 needs an sm_90 (H100) device");
  if (!d.attrs_set) {
    CUDA_TRY(cudaFuncSetAttribute(render_rays_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kSmemTotal)), "smem attr render");
    CUDA_TRY(cudaFuncSetAttribute(render_rays_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kSmemTotal)), "smem attr render(save)");
    CUDA_TRY(cudaFuncSetAttribute(mlp_forward_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kSmemTotal)), "smem attr mlp");
    CUDA_TRY(cudaFuncSetAttribute(mlp_forward_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kSmemTotal)), "smem attr mlp(save)");
    CUDA_TRY(cudaFuncSetAttribute(mlp_forward_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kSmemTotal)), "smem attr mlp(save rows)");
    CUDA_TRY(cudaFuncSetAttribute(mlp_forward_kernel<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kSmemTotal)), "smem attr mlp(sh)");
    CUDA_TRY(cudaFuncSetAttribute(chain_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kChSmemTotal)), "smem attr chain");
    CUDA_TRY(cudaFuncSetAttribute(chain_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kChSmemTotal)), "smem attr chain (probe)");
    CUDA_TRY(cudaFuncSetAttribute(chain_bwd_dev_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kChSmemTotal)), "smem attr chain (planned)");
    CUDA_TRY(cudaFuncSetAttribute(chain_bwd_dev_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kChSmemTotal)), "smem attr chain (planned probe)");
    CUDA_TRY(cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kWgSmemTotal)), "smem attr wgrad");
    // one cdf of n_weights + 1 floats per warp: above the 48 KB default from n_weights = 3072
    CUDA_TRY(cudaFuncSetAttribute(sample_pdf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kPdfWarps * (kPdfMaxWeights + 1) * sizeof(float))), "smem attr sample_pdf");
    int* hs = nullptr;
    CUDA_TRY(cudaHostAlloc(&hs, sizeof(int), cudaHostAllocMapped), "status alloc");
    *hs = 0;
    CUDA_TRY(cudaHostGetDevicePointer(&d.status, hs, 0), "status device pointer");
    d.status_host = hs;
    d.attrs_set = true;
  }
  *out = &d;
  return 0;
}

// A kernel of an EARLIER call on this device reported a device-side fault (misaligned shared
// memory, code 101; a training backward whose per-sample gradients overflowed fp16, code 102; one whose per-sample
// gradients were not finite, code 103)
// through the internal status word: surface it on this call and clear it.
// (The word lives in mapped pinned host memory, so this is a plain host read, no synchronisation;
// callers that want the fault of THIS call pass their own `status` word or call
// nerfb200_check_status() after synchronising.)
int check_sticky_status(DeviceInfo* d) {
  if (d->status_host == nullptr) return 0;
  const int st = *d->status_host;
  if (st == 0) return 0;
  *d->status_host = 0;
  if (st == 102)
    return fail(NERFB200_EDEVICE, "an earlier training backward reported device status 102: a per-sample "
                "gradient exceeded the fp16 range of its layer's scale, its weight gradients are wrong");
  if (st == 103)
    return fail(NERFB200_EDEVICE, "an earlier training backward reported device status 103: a per-sample gradient "
                "was not finite (a non-finite ray, input, output or upstream gradient), its weight gradients are wrong");
  return fail(NERFB200_EDEVICE, "an earlier nerf_pl_b200 kernel reported device status %d", st);
}

int check_render_shapes(const nerfb200_render_args* a) {
  if (a == nullptr) return fail(NERFB200_EINVAL, "args is NULL");
  if (a->n_rays < 0) return fail(NERFB200_EINVAL, "n_rays < 0");
  if (a->n_samples != 32 && a->n_samples != 64 && a->n_samples != 128)
    return fail(NERFB200_EUNSUPPORTED, "N_samples must be 32, 64 or 128");
  if (a->n_importance < 0 || (a->n_importance % 32) != 0)
    return fail(NERFB200_EUNSUPPORTED, "N_importance must be a multiple of 32");
  if (a->n_samples + a->n_importance > kMaxSf)
    return fail(NERFB200_EUNSUPPORTED, "N_samples + N_importance must be <= 192");
  if (a->n_rays == 0) return 0;
  if (!a->rays || !a->packed_coarse) return fail(NERFB200_EINVAL, "rays / packed_coarse is NULL");
  if (a->ray_stride < 8) return fail(NERFB200_EINVAL, "ray_stride < 8");
  if (!a->opacity_coarse) return fail(NERFB200_EINVAL, "opacity_coarse is NULL");
  if (!a->test_time && (!a->rgb_coarse || !a->depth_coarse))
    return fail(NERFB200_EINVAL, "rgb_coarse / depth_coarse is NULL with test_time=0");
  if (a->n_importance > 0) {
    if (!a->packed_fine) return fail(NERFB200_EINVAL, "packed_fine is NULL with N_importance>0");
    if (!a->rgb_fine || !a->depth_fine || !a->opacity_fine)
      return fail(NERFB200_EINVAL, "fine outputs are NULL with N_importance>0");
  }
  if (a->rng_in_kernel == 2 && !a->rng_seed_dev) return fail(NERFB200_EINVAL, "rng_in_kernel = 2 needs rng_seed_dev");
  if (a->perturb > 0.f && !a->rng_in_kernel) {
    if (!a->perturb_rand) return fail(NERFB200_EINVAL, "perturb>0 needs perturb_rand");
    if (a->n_importance > 0 && !a->u_rand) return fail(NERFB200_EINVAL, "perturb>0 needs u_rand");
  }
  if (a->noise_std > 0.f) {
    if (!a->noise_coarse) return fail(NERFB200_EINVAL, "noise_std>0 needs noise_coarse");
    if (a->n_importance > 0 && !a->noise_fine) return fail(NERFB200_EINVAL, "noise_std>0 needs noise_fine");
  }
  if ((reinterpret_cast<uintptr_t>(a->packed_coarse) & 15) ||
      (reinterpret_cast<uintptr_t>(a->packed_fine) & 15))
    return fail(NERFB200_EINVAL, "packed images must be 16-byte aligned");
  return 0;
}


// ------------------------------------------------------------------ training workspace layout
// One device buffer per (n_rays, N_samples, N_importance); the layout is a pure function of those
// numbers and the SM count, recomputed on every call (no state kept in the library).
// kJDir (NeRF.forward backward only): the direction slice gW_dir[:, 256:283] = dd^T xdir over the direction rows
// the forward fed the tensor core (the render path sums dd per ray instead: dir_grad_kernel)
enum { kJ1 = 0, kJ2, kJ3, kJ4, kJ5a, kJ5b, kJ6, kJ7, kJ8, kJ9, kNumJobKinds, kJDir = kNumJobKinds, kNumJobKindsMlp };
constexpr int kWgSlotFloats = 256 * 256 + 256;           // partial of one CTA: out (transposed), bias
constexpr int kMaxWgJobs = 1024;
constexpr int kMaxWgCtas = 512;
constexpr int kWgPieceChunks = 512;                      // 32,768 samples per wgmma accumulator (plan_wgrad)
struct TrainLayout {
  PassBufs pass[2];
  int n_pass, n_rays;
  int n_kinds;                    // wgrad GEMMs per pass: kNumJobKinds (render path) or kNumJobKindsMlp
  uint8_t* xdir;                  // NeRF.forward path: tiled (n_pad, 64) fp16 direction rows (else null)
  WgradJob* jobs_dev;             // pieces, in (pass, layer, chunk) order
  int* cta_first_dev;             // [n_cta + 1]: CTA b works on pieces [cta_first[b], cta_first[b + 1])
  int n_jobs, n_cta;
  int n_split[2][kNumJobKindsMlp];   // CTAs, hence partials, of each (pass, layer)
  int first_cta[2][kNumJobKindsMlp];
  float* wg_part;                 // [n_cta][kWgSlotFloats]
  int head_grid;                  // blocks of head_bwd_kernel (both passes in one launch)
  float* head_part[2];            // [head_grid][kHeadPartFloats] per pass
  float* raysum[2];               // (n_rays, 128) per-ray sums of dd
  float* direnc;                  // (n_rays, 28) embedded directions
  float* dir_part[2];             // [kDirSlices][128][27]
  float* gWp[2];                  // (128,256)
  float* gbp[2];                  // (128)
  float* lscale;                  // [2][kLevels] per-pass, per-level gradient scales
  float* linv;                    // [2][kLevels] their inverses
  unsigned* lamax;                // [2][kLevels] probe statistics
  unsigned* amax;                 // [2][2] max |d sigma|, |d rgb_pre| per pass
  float* loss_part;               // [max CTAs][2]
  unsigned* loss_counter;
  size_t bytes;
};

__host__ __device__ void plan_wgrad(TrainLayout* L, int n_cta, WgradJob* jobs, int* cta_first);

__host__ __device__ void job_shape(int kind, int* a_fb, int* b_fb) {
  *a_fb = (kind == kJ9 || kind == kJDir) ? 2 : 4;
  *b_fb = (kind == kJ1 || kind == kJ5a || kind == kJDir) ? 1 : 4;
}

// The per-pass buffers of a training workspace, in PassBufs order.
void take_pass_bufs(PassBufs& b, Carver& c) {
  const size_t np = static_cast<size_t>(b.n_pad);
  b.enc = c.take(np * 128);
  b.act = c.take(np * 512 * 8);
  b.mask = c.take<uint2>(np * 32);
  b.d = c.take(np * 256);
  b.sigma = c.take<float>(np);
  b.rgb = c.take<float>(np * 3);
  b.z = c.take<float>(static_cast<size_t>(b.n));
  b.dsigma = c.take<float>(np);
  b.dprergb = c.take<float>(np * 3);
  b.dd = c.take(np * 256);
  b.dpre = c.take(np * 512 * 8);
}

// Both training workspaces.  The render path (nerfb200_render_rays in training mode, nerfb200_render_backward):
// n rays, a coarse pass of n_samples per ray and, when n_importance > 0, a fine pass of n_samples + n_importance.
// A direct NeRF.forward call over n samples (`mlp`: nerfb200_nerf_forward_train, nerfb200_nerf_backward): one pass
// with one sample per row, the per-pass buffers of the render path in the same order (so one reader serves both),
// then the direction rows the forward fed the tensor core, the wgrad plan (with the direction-slice GEMM kJDir) and
// the head partials.  Its head kernel views the batch as n_pad / 64 pseudo-rays of 64 samples; nothing per ray
// (direnc, raysum, dir_part) and no fused loss exists there.
constexpr int kMlpPseudoRay = 64;
void make_train_layout(TrainLayout* L, uint8_t* base, bool mlp, int64_t n, int n_samples, int n_importance,
                       int sm_count) {
  Carver c{base, 0, 1024};
  std::memset(L, 0, sizeof(*L));
  L->n_pass = n_importance > 0 ? 2 : 1;
  L->n_kinds = mlp ? kNumJobKindsMlp : kNumJobKinds;
  for (int ps = 0; ps < L->n_pass; ++ps) {
    PassBufs& b = L->pass[ps];
    b.S = ps ? n_samples + n_importance : n_samples;
    b.n = n * b.S;
    b.n_pad = (b.n + 127) / 128 * 128;
    take_pass_bufs(b, c);
  }
  if (mlp) L->xdir = c.take(static_cast<size_t>(L->pass[0].n_pad) * 128);
  const int64_t head_rays = mlp ? L->pass[0].n_pad / kMlpPseudoRay : n;
  L->n_rays = static_cast<int>(head_rays);
  plan_wgrad(L, sm_count > 0 ? sm_count : 148, nullptr, nullptr);
  L->jobs_dev = c.take<WgradJob>(kMaxWgJobs);
  L->cta_first_dev = c.take<int>(kMaxWgCtas + 1);
  L->wg_part = c.take<float>(static_cast<size_t>(L->n_cta) * kWgSlotFloats);
  L->head_grid = static_cast<int>((L->n_pass * head_rays + kHeadWarps - 1) / kHeadWarps);
  if (!mlp) L->direnc = c.take<float>(static_cast<size_t>(n) * 28);
  for (int ps = 0; ps < (mlp ? 1 : 2); ++ps) {
    L->head_part[ps] = c.take<float>(static_cast<size_t>(L->head_grid) * kHeadPartFloats);
    if (!mlp) {
      L->raysum[ps] = c.take<float>(static_cast<size_t>(n) * 128);
      L->dir_part[ps] = c.take<float>(static_cast<size_t>(kDirSlices) * 128 * 27);
    }
    L->gWp[ps] = c.take<float>(128 * 256);
    L->gbp[ps] = c.take<float>(128);
  }
  L->lscale = c.take<float>(2 * kLevels);
  L->linv = c.take<float>(2 * kLevels);
  L->lamax = c.take<unsigned>(2 * kLevels);
  L->amax = c.take<unsigned>(4);
  if (!mlp) {
    L->loss_part = c.take<float>(1024 * 2);
    L->loss_counter = c.take<unsigned>(4);
  }
  L->bytes = c.off;
}

// The wgrad plan of a layout: CTA counts per (pass, layer) (always), and when `jobs` / `cta_first` are
// given the image of the piece table and of the per-CTA piece ranges (host memory for the plain paths, the
// workspace's tables for train_skip_plan_kernel).
__host__ __device__ void job_operands(const TrainLayout& L, int ps, int k, const uint8_t** A, const uint8_t** B) {
  const PassBufs& b = L.pass[ps];
  const size_t lay = static_cast<size_t>(b.n_pad) * 512;
  switch (k) {
    case kJ1: *A = b.dpre; *B = b.enc; break;
    case kJ5a: *A = b.dpre + 4 * lay; *B = b.enc; break;
    case kJ5b: *A = b.dpre + 4 * lay; *B = b.act + 3 * lay; break;
    case kJ9: *A = b.dd; *B = b.act + 7 * lay; break;
    case kJDir: *A = b.dd; *B = L.xdir; break;
    default: {
      const int l = (k <= kJ4) ? k + 1 : k;            // kJ2..kJ4 -> layers 2..4, kJ6..kJ8 -> layers 6..8
      *A = b.dpre + static_cast<size_t>(l - 1) * lay;
      *B = b.act + static_cast<size_t>(l - 2) * lay;
    }
  }
}

__host__ __device__ void fill_piece(TrainLayout* L, WgradJob* jobs, int piece, int cta, int ps, int k, long long c0, long long c1,
                int step, bool add) {
  if (!jobs) return;
  int a_fb, b_fb;
  job_shape(k, &a_fb, &b_fb);
  const uint8_t *A = nullptr, *B = nullptr;
  job_operands(*L, ps, k, &A, &B);
  WgradJob& j = jobs[piece];
  float* slot = L->wg_part + static_cast<size_t>(cta) * kWgSlotFloats;
  j.a = A; j.b = B; j.a_fb = a_fb; j.b_fb = b_fb;
  j.chunk0 = static_cast<int>(c0);
  j.chunk1 = static_cast<int>(c1);
  j.chunk_step = step;
  j.add = add ? 1 : 0;
  j.out = slot;
  j.bias_out = (k == kJ5b || k == kJDir) ? nullptr : slot + 256 * 256;
}

__host__ __device__ void plan_wgrad(TrainLayout* L, int n_cta, WgradJob* jobs, int* cta_first) {
  if (n_cta > kMaxWgCtas) n_cta = kMaxWgCtas;
  const int kinds = L->n_kinds;
  long long total = 0;
  long long work[2][kNumJobKindsMlp];
  for (int ps = 0; ps < L->n_pass; ++ps)
    for (int k = 0; k < kinds; ++k) {
      int a_fb, b_fb;
      job_shape(k, &a_fb, &b_fb);
      work[ps][k] = (L->pass[ps].n_pad / 64) * (a_fb + b_fb);
      total += work[ps][k];
    }
  // whole CTAs per GEMM: a share of the SMs by bytes streamed, at least one (with fewer SMs than GEMMs the grid runs
  // in more than one wave); the CTAs of one GEMM take its chunks round-robin, so together they read ONE moving window
  // of each operand
  int n_of[2][kNumJobKindsMlp];
  int used = 0;
  for (int ps = 0; ps < L->n_pass; ++ps)
    for (int k = 0; k < kinds; ++k) {
      const double share = total > 0 ? static_cast<double>(work[ps][k]) * n_cta / static_cast<double>(total) : 0.0;
      int n = static_cast<int>(share);
      if (n < 1) n = 1;
      n_of[ps][k] = n;
      used += n;
    }
  while (used < n_cta) {          // hand the remaining SMs to the GEMMs with the most work per CTA
    int bp = 0, bk = 0;
    double best = -1;
    for (int ps = 0; ps < L->n_pass; ++ps)
      for (int k = 0; k < kinds; ++k) {
        const double load = static_cast<double>(work[ps][k]) / n_of[ps][k];
        if (load > best) { best = load; bp = ps; bk = k; }
      }
    ++n_of[bp][bk];
    ++used;
  }
  // CTA j of a GEMM with g CTAs takes chunks j, j + g, ..; it sums them in pieces of at most kWgPieceChunks chunks
  // (more only if the piece table would overflow), each piece in the tensor core's accumulators, the pieces added
  // in fp32 into the CTA's partial.  The tensor core's fp32 accumulation error grows with the number of K steps one
  // accumulator sums instead of averaging out: one accumulator per CTA gave weight gradients with relative L2
  // errors of 3.1e-5, 1.2e-4 and 3.0e-4 for 1,024, 4,096 and 8,192-ray batches (64 + 64, 64 + 64 and 64 + 128
  // samples) on an H100 80GB HBM3 at 700 W; with pieces the last two are 5.7e-5 and 5.8e-5.
  int n_cta_used = 0;
  for (int ps = 0; ps < L->n_pass; ++ps)
    for (int k = 0; k < kinds; ++k)
      n_cta_used += static_cast<int>(n_of[ps][k] < L->pass[ps].n_pad / 64 ? n_of[ps][k] : L->pass[ps].n_pad / 64);
  const int max_pieces = n_cta_used > 0 ? kMaxWgJobs / n_cta_used : kMaxWgJobs;        // per CTA
  int piece = 0, cta = 0;
  for (int ps = 0; ps < L->n_pass; ++ps)
    for (int k = 0; k < kinds; ++k) {
      const long long chunks = L->pass[ps].n_pad / 64;
      int g = n_of[ps][k];
      if (g > chunks) g = static_cast<int>(chunks);
      L->first_cta[ps][k] = cta;
      // CTA j's share, ceil((chunks - j) / g) chunks, is q + 1 for j < r and q for the others (chunks = q g + r): the
      // divisions are per GEMM, not per CTA (train_skip_plan_kernel runs this on one device thread)
      const long long q = g > 0 ? chunks / g : 0, r = g > 0 ? chunks - q * g : 0;
      long long len_of[2];
      for (int e = 0; e < 2; ++e) {
        const long long want = (q + 1 - e + max_pieces - 1) / max_pieces;
        len_of[e] = want > kWgPieceChunks ? want : kWgPieceChunks;
      }
      for (int j = 0; j < g; ++j, ++cta) {
        const int e = j < r ? 0 : 1;
        const long long mine = q + 1 - e, len = len_of[e];
        if (cta_first) cta_first[cta] = piece;
        for (long long s = 0; s < mine; s += len, ++piece)
          fill_piece(L, jobs, piece, cta, ps, k, j + s * g, chunks < j + (s + len) * g ? chunks : j + (s + len) * g, g,
                     s > 0);
      }
      L->n_split[ps][k] = g;
    }
  if (cta_first) cta_first[cta] = piece;
  L->n_jobs = piece;
  L->n_cta = cta;
}

// grow-only device arena for the *_host entry
struct Arena {
  uint8_t* base = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes) {
    if (bytes <= cap) return 0;
    if (base) cudaFree(base);
    base = nullptr; cap = 0;
    cudaError_t e = cudaMalloc(&base, bytes);
    if (e != cudaSuccess) return cuda_fail(e, "arena cudaMalloc");
    cap = bytes;
    return 0;
  }
};
Arena g_arena[64];
std::mutex g_host_call_mu;
std::mutex g_arena_mu;   // separate from g_mu: the host entry calls nerfb200_render_rays (device_info locks g_mu)

// Step 3 of a training backward: the chain kernel's probe pass over pt0 + pt1 tiles spread evenly over each pass, then
// (after the phase-1 scales) the real pass over all t0 + t1 tiles, the probe's first.  The parameters of both launches
// from a layout, on the host for the plain paths and on the device for train_skip_plan_kernel.
__host__ __device__ void chain_plan(const TrainLayout& L, const uint8_t* const net[2], int* status, int sm_count,
                                    ChainParams* probe, ChainParams* real) {
  ChainParams& cp = *probe;
  const int q1 = L.n_pass > 1 ? 1 : 0;
  cp.n_pass = L.n_pass;
  cp.pass[0] = L.pass[0]; cp.pass[1] = L.pass[1];
  cp.net[0] = net[0]; cp.net[1] = net[1];
  cp.lscale = L.lscale;
  cp.lamax = L.lamax;
  cp.status = status;
  const long long t0 = L.pass[0].n_pad / 128, t1 = q1 ? L.pass[1].n_pad / 128 : 0;
  const long long n_probe = q1 ? (sm_count + 1) / 2 : sm_count;      // probe tiles per pass, at most
  const long long span[2] = {t0, t1}, pt[2] = {t0 < n_probe ? t0 : n_probe, t1 < n_probe ? t1 : n_probe};
  for (int ps = 0; ps < 2; ++ps) {
    long long s = (pt[ps] > 0 && span[ps] > pt[ps]) ? span[ps] / pt[ps] : 1;
    for (;;) {                    // the smallest stride from span / probe tiles up that is coprime to the span
      long long x = s, y = span[ps];
      while (y != 0) { const long long r = x % y; x = y; y = r; }
      if (span[ps] <= 1 || x == 1) break;
      ++s;
    }
    cp.span[ps] = span[ps] > 0 ? span[ps] : 1;
    cp.stride[ps] = s;
    cp.tiles[ps] = cp.head[ps] = pt[ps];
  }
  *real = cp;
  real->tiles[0] = t0;
  real->tiles[1] = t1;
}

// Step 2: the head kernel's parameters (host and device, as chain_plan).
__host__ __device__ void head_plan(const TrainLayout& L, const float* w_rgb0, const float* w_rgb1, const float* rays,
                                   long long ray_stride, HeadBwdParams* hp) {
  hp->n_rays = L.n_rays; hp->n_pass = L.n_pass;
  hp->pass[0] = L.pass[0]; hp->pass[1] = L.pass[1];
  if (!rays) {
    hp->pass[0].S = kMlpPseudoRay;
    hp->pass[1] = hp->pass[0];
  }
  hp->w_rgb[0] = w_rgb0; hp->w_rgb[1] = w_rgb1;
  hp->lscale = L.lscale;
  hp->rays = rays; hp->ray_stride = ray_stride;
  hp->raysum[0] = L.raysum[0]; hp->raysum[1] = L.raysum[1];
  hp->direnc = L.direnc;
  hp->part[0] = L.head_part[0]; hp->part[1] = L.head_part[1];
}

// Step 5: the reduction items of pass ps that both training backwards share (wgrad GEMMs of layers 1..8 and of the
// folded W', the head partials), appended to `tab`.  g: the pass's 24 gradient tensors.
__host__ __device__ void add_reduce_items(ReduceTable& tab, const TrainLayout& L, int ps, float* const* g) {
  auto add = [&](const float* part, long long stride, int n_split, float* out, const float* mul, int rows, int cols,
                 int part_ld, int out_ld, int out_col0, int transposed = 0) {
    ReduceItem& it = tab.it[tab.n++];
    it.part = part; it.split_stride = stride; it.n_split = n_split; it.out = out; it.mul = mul;
    it.rows = rows; it.cols = cols; it.part_ld = part_ld; it.out_ld = out_ld; it.out_col0 = out_col0;
    it.transposed = transposed;
    it.by_warp = (n_split >= 128 && rows * cols <= 4096) ? 1 : 0;
  };
  const float* linv = L.linv + ps * kLevels;       // level v: 0 = dd, v = 1..8 = dpre_{9-v}
  auto slot = [&](int kind) { return L.wg_part + static_cast<size_t>(L.first_cta[ps][kind]) * kWgSlotFloats; };
  auto ns = [&](int kind) { return L.n_split[ps][kind]; };
  add(slot(kJ1), kWgSlotFloats, ns(kJ1), g[0], linv + 8, 256, 63, 256, 63, 0, 1);
  add(slot(kJ1) + 65536, kWgSlotFloats, ns(kJ1), g[1], linv + 8, 1, 256, 256, 256, 0);
  const int hidden[6] = {kJ2, kJ3, kJ4, kJ6, kJ7, kJ8};
  const int layer[6] = {2, 3, 4, 6, 7, 8};
  for (int i = 0; i < 6; ++i) {
    const float* inv = linv + (9 - layer[i]);
    add(slot(hidden[i]), kWgSlotFloats, ns(hidden[i]), g[2 * (layer[i] - 1)], inv, 256, 256, 256, 256, 0, 1);
    add(slot(hidden[i]) + 65536, kWgSlotFloats, ns(hidden[i]), g[2 * (layer[i] - 1) + 1], inv, 1, 256, 256, 256, 0);
  }
  add(slot(kJ5a), kWgSlotFloats, ns(kJ5a), g[8], linv + 4, 256, 63, 256, 319, 0, 1);
  add(slot(kJ5b), kWgSlotFloats, ns(kJ5b), g[8], linv + 4, 256, 256, 256, 319, 63, 1);
  add(slot(kJ5a) + 65536, kWgSlotFloats, ns(kJ5a), g[9], linv + 4, 1, 256, 256, 256, 0);
  add(slot(kJ9), kWgSlotFloats, ns(kJ9), L.gWp[ps], linv, 128, 256, 128, 256, 0, 1);
  add(slot(kJ9) + 65536, kWgSlotFloats, ns(kJ9), L.gbp[ps], linv, 1, 128, 128, 128, 0);
  add(L.head_part[ps] + kHeadPartSigW, kHeadPartFloats, L.head_grid, g[20], nullptr, 1, 256, 256, 256, 0);
  add(L.head_part[ps] + kHeadPartSigB, kHeadPartFloats, L.head_grid, g[21], nullptr, 1, 1, 1, 1, 0);
  add(L.head_part[ps] + kHeadPartRgbW, kHeadPartFloats, L.head_grid, g[22], nullptr, 1, 384, 384, 384, 0);
  add(L.head_part[ps] + kHeadPartRgbB, kHeadPartFloats, L.head_grid, g[23], nullptr, 1, 3, 3, 3, 0);
  if (L.n_kinds == kNumJobKindsMlp)      // direction slice: gW_dir[:, 256:283] = dd^T xdir / s_0 (columns 0..26 of 64)
    add(slot(kJDir), kWgSlotFloats, ns(kJDir), g[18], linv, 128, 27, 128, 283, 256, 1);
  else                                   // per-ray direction sums (dir_grad_kernel)
    add(L.dir_part[ps], 128 * 27, kDirSlices, g[18], nullptr, 128, 27, 27, 283, 256);
}

// Both *_workspace_init entries, after their own checks: zero the workspace (padding rows of the operand arrays are
// never written afterwards, counters start at zero), upload the wgrad plan, and return once both are on the device.
int init_train_workspace(TrainLayout& L, void* ws, int sm_count, cudaStream_t stream) {
  CUDA_TRY(cudaMemsetAsync(ws, 0, L.bytes, stream), "workspace memset");
  std::vector<WgradJob> jobs(kMaxWgJobs);
  std::vector<int> cta_first(kMaxWgCtas + 1, 0);
  std::memset(jobs.data(), 0, sizeof(WgradJob) * kMaxWgJobs);
  plan_wgrad(&L, sm_count, jobs.data(), cta_first.data());
  CUDA_TRY(cudaMemcpyAsync(L.jobs_dev, jobs.data(), sizeof(WgradJob) * kMaxWgJobs, cudaMemcpyHostToDevice, stream),
           "job table upload");
  CUDA_TRY(cudaMemcpyAsync(L.cta_first_dev, cta_first.data(), sizeof(int) * (kMaxWgCtas + 1), cudaMemcpyHostToDevice, stream),
           "cta table upload");
  CUDA_TRY(cudaStreamSynchronize(stream), "workspace init sync");
  return 0;
}

// The count-dependent launch parameters of one network's backward tail when training with empty samples skipped,
// written into the workspace by train_skip_plan_kernel from the device's sample count.
struct TrainSkipPlan {
  HeadBwdParams head;
  int head_grid;
  ChainParams probe, chain;
  ReduceTable tab;
};

// Steps 2-6 of both training backwards, once step 1 has left each pass's per-sample d sigma / d rgb_pre and their
// maxima in the workspace.  params / grads / net: per pass.  rays: the render path's rays, whose directions the head
// kernel embeds for the per-ray direction part of gW_dir; null for a direct NeRF.forward call, whose head kernel walks
// pseudo-rays of 64 samples and whose direction part is the wgrad GEMM kJDir.  plan: null, or the device plan of a
// layout carved for more rows (training with empty samples skipped): every launch then has the grid of L, the carved
// worst case, and the count-dependent kernels read their parameters from the plan.
int backward_tail(const TrainLayout& L, const float* const* const params[2], float* const* const grads[2],
                  const uint8_t* const net[2], const float* rays, long long ray_stride, const DeviceInfo* d,
                  cudaStream_t stream, const char* what, const TrainSkipPlan* plan = nullptr) {
  const int q1 = L.n_pass > 1 ? 1 : 0;        // table entry of the second pass: a single pass fills both slots
  ScaleParams sp;
  sp.n_pass = L.n_pass; sp.phase = 0;
  sp.amax = L.amax; sp.lamax = L.lamax; sp.lscale = L.lscale; sp.linv = L.linv;
  sp.w_rgb[0] = params[0][22]; sp.w_rgb[1] = params[q1][22];
  sp.w_sigma[0] = params[0][20]; sp.w_sigma[1] = params[q1][20];
  TRY(launch(what, bwd_scale_kernel, 1, 128, 0, stream, sp));
  // 2. rgb head, ReLU of the direction layer (both passes in one launch), direction part of gW_dir
  HeadBwdParams hp;
  head_plan(L, params[0][22], params[q1][22], rays, ray_stride, &hp);
  if (plan)
    TRY(launch(what, head_bwd_dev_kernel, L.head_grid, kHeadWarps * 32, 0, stream, &plan->head, &plan->head_grid));
  else
    TRY(launch(what, head_bwd_kernel, L.head_grid, kHeadWarps * 32, 0, stream, hp));
  if (rays) {
    DirGradParams dp;
    dp.n_rays = L.n_rays;
    dp.raysum[0] = L.raysum[0]; dp.raysum[1] = L.raysum[1];
    dp.direnc = L.direnc;
    dp.part[0] = L.dir_part[0]; dp.part[1] = L.dir_part[1];
    TRY(launch(what, dir_grad_kernel, dim3(kDirSlices, L.n_pass), 128, 0, stream, dp));
  }
  // 3. dgrad chain (wgmma): a probe pass over one tile per SM picks the per-layer scales, then the real pass.
  // The probe's tiles are spread evenly over each pass: gradients are not uniform over a batch (rays whose
  // colour is already right carry almost none), and scales taken from the first tiles alone saturate the rest.
  // Both launches visit the tiles of a pass in the order j -> j * stride mod span (stride coprime to span, about
  // span / probe tiles), the real pass the probe's tiles first, so its first wave finds them in L2.  A tile the
  // probe did not see can still exceed its level's range: the wgrad kernel reports that (status 102).
  ChainParams probe, cp;
  chain_plan(L, net, d->status, d->sm_count, &probe, &cp);
  const int probe_ctas = static_cast<int>(probe.tiles[0] + probe.tiles[1]);
  const long long total = cp.tiles[0] + cp.tiles[1];
  const int ctas = static_cast<int>(total < d->sm_count ? total : d->sm_count);
  if (plan)
    TRY(launch(what, chain_bwd_dev_kernel<true>, probe_ctas, kThreads, kChSmemTotal, stream, &plan->probe));
  else
    TRY(launch(what, chain_bwd_kernel<true>, probe_ctas, kThreads, kChSmemTotal, stream, probe));
  sp.phase = 1;
  TRY(launch(what, bwd_scale_kernel, 1, 128, 0, stream, sp));
  if (plan)
    TRY(launch(what, chain_bwd_dev_kernel<false>, ctas, kThreads, kChSmemTotal, stream, &plan->chain));
  else
    TRY(launch(what, chain_bwd_kernel<false>, ctas, kThreads, kChSmemTotal, stream, cp));
  // 4. split-K wgrad (wgmma)
  TRY(launch(what, wgrad_kernel, L.n_cta, kWgThreads, kWgSmemTotal, stream, L.jobs_dev, L.cta_first_dev, d->status));
  // 5. partial sums -> gradient tensors (fixed order), 6. unfold W'
  ReduceTable tab;
  tab.n = 0;
  for (int ps = 0; ps < L.n_pass; ++ps) add_reduce_items(tab, L, ps, grads[ps]);
  // latency-bound: 64 blocks per item (16 measured 40 us)
  if (plan)
    TRY(launch(what, wgrad_reduce_dev_kernel, dim3(64, tab.n), 256, 0, stream, &plan->tab));
  else
    TRY(launch(what, wgrad_reduce_kernel, dim3(64, tab.n), 256, 0, stream, tab));
  UnfoldParams up;
  for (int ps = 0; ps < 2; ++ps) {
    const int q = ps ? q1 : 0;
    up.gWp[ps] = L.gWp[q]; up.gbp[ps] = L.gbp[q];
    up.Wf[ps] = params[q][16]; up.bf[ps] = params[q][17]; up.Wd[ps] = params[q][18];
    up.gWd[ps] = grads[q][18]; up.gbd[ps] = grads[q][19]; up.gWf[ps] = grads[q][16]; up.gbf[ps] = grads[q][17];
  }
  // warps: one per gWd output (128 x 256), then one thread per gWf / gbf output
  return launch(what, unfold_kernel, dim3((128 * 256 + (256 * 256 + 256 + 31) / 32 + 7) / 8, L.n_pass), 256, 0, stream,
                up);
}

// The four entries of mlp_forward_kernel, after their own checks: one CTA per 128-row tile, at most one per SM.  With
// a NeRF.forward training workspace `ws` the save-mode instantiation also stores what nerfb200_nerf_backward reads;
// with p.sh the SH mode runs.
int launch_mlp(MlpParams p, void* ws, void* stream, const char* what) {
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  TRY(check_sticky_status(d));
  p.status = d->status;
  const long long tiles = (p.n + 127) / 128;
  const int ctas = static_cast<int>(tiles < d->sm_count ? tiles : d->sm_count);
  if (ws) {
    TrainLayout L;
    make_train_layout(&L, static_cast<uint8_t*>(ws), true, p.n, 1, 0, d->sm_count);
    p.tr = L.pass[0];
    p.xdir = L.xdir;
  }
  return launch(what, p.sh ? mlp_forward_kernel<false, false, true> : ws ? mlp_forward_kernel<true> : mlp_forward_kernel<false>,
                ctas, kThreads, kSmemTotal, stream, p);
}

// The tensor table of both Adam entries: each tensor checked (steps: the device step counts, or null) and given its
// run of 1024-element blocks.  *blocks: the total.
int fill_adam_table(AdamParams& a, int32_t n_tensors, float* const* params, const float* const* grads,
                    float* const* exp_avg, float* const* exp_avg_sq, const int64_t* numel, const float* const* steps,
                    float beta1, float beta2, float eps, float weight_decay, const char* who, int* blocks) {
  a.n_tensors = n_tensors;
  int b = 0;
  for (int i = 0; i < n_tensors; ++i) {
    if (numel[i] < 0 || numel[i] > 0x7fffffff ||
        (numel[i] > 0 && (!params[i] || !grads[i] || !exp_avg[i] || !exp_avg_sq[i] || (steps && !steps[i]))))
      return fail(NERFB200_EINVAL, "%s: NULL tensor / bad size", who);
    a.p[i] = params[i]; a.g[i] = grads[i]; a.m[i] = exp_avg[i]; a.v[i] = exp_avg_sq[i];
    a.numel[i] = static_cast<int>(numel[i]);
    a.block0[i] = b;
    b += static_cast<int>((numel[i] + 1023) / 1024);
  }
  a.block0[n_tensors] = b;
  a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.weight_decay = weight_decay;
  *blocks = b;
  return 0;
}

int fill_pack_params(PackParams* pp, const float* const params[24], void* packed) {
  if (!params || !packed) return fail(NERFB200_EINVAL, "pack_weights: NULL argument");
  if (reinterpret_cast<uintptr_t>(packed) & 15) return fail(NERFB200_EINVAL, "packed must be 16-byte aligned");
  for (int i = 0; i < kNumParams; ++i) {
    if (!params[i]) return fail(NERFB200_EINVAL, "pack_weights: NULL parameter tensor");
    pp->p[i] = params[i];
  }
  pp->out = static_cast<uint8_t*>(packed);
  return 0;
}

int launch_pack(const PackParams2& pp2, int n_nets, void* stream) {
  const long long total = kHalfRegionBytes / 2 + kF32Count + static_cast<long long>(kNumSlicesBwd) * 256 * 64;
  const int threads = 256;
  const int blocks = static_cast<int>((total + threads - 1) / threads);
  return launch("pack_weights launch", pack_weights_kernel, dim3(blocks, n_nets), threads, 0, stream, pp2);
}

// ------------------------------------------------------------------ coloured mesh extraction
// (extract_color_mesh.py; kernels: mesh_kernels.cuh)

// Both dense grid queries: the N^3 points `chunk` at a time, their positions into the workspace, then
// query(xyz, first point, points).
template <class Query>
int grid_chunks(int64_t N, const double ranges_host[6], int64_t chunk, void* ws, void* stream, Query&& query) {
  float* xyz = static_cast<float*>(ws);
  const long long total = N * N * N;
  for (long long s = 0; s < total; s += chunk) {
    const long long n = total - s < chunk ? total - s : chunk;
    TRY(nerfb200_grid_positions(N, ranges_host, s, n, xyz, stream));
    TRY(query(xyz, s, n));
  }
  return 0;
}

struct U8ToInt {
  __host__ __device__ __forceinline__ int operator()(uint8_t v) const { return v; }
};
using U8It = thrust::transform_iterator<U8ToInt, const uint8_t*, int>;

// What a workspace holds for CUB besides the kernels' buffers: the alternate buffers of a radix sort and the
// temporary storage of its algorithms (temp_bytes: the largest size CUB asks for).
struct CubScratch {
  void* keys_alt = nullptr;
  void* vals_alt = nullptr;
  void* temp = nullptr;
  size_t temp_bytes = 0;
};

int bits_for(long long v) {
  int b = 1;
  while ((1LL << b) < v) ++b;
  return b;
}

constexpr long long kMcMaxPoints = 400LL * 1000 * 1000;   // keeps 3 P vertices and 5 C triangles in int32

// The marching-cubes workspace of P points and C cells at `base` (nullptr: sizing only): its buffers in p, CUB's in
// s.  Returns its bytes.
size_t mc_carve(long long P, long long C, void* base, McParams* p, CubScratch* s) {
  size_t t1 = 0, t2 = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, t1, U8It(nullptr, U8ToInt()), static_cast<int*>(nullptr), static_cast<int>(P + 1));
  cub::DeviceScan::ExclusiveSum(nullptr, t2, U8It(nullptr, U8ToInt()), static_cast<int*>(nullptr), static_cast<int>(C + 1));
  s->temp_bytes = t1 > t2 ? t1 : t2;
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  p->vcnt = c.take(P + 1);
  p->vofs = c.take<int>(P + 1);
  p->ccnt = c.take(C + 1);
  p->cofs = c.take<int>(C + 1);
  s->temp = c.take(s->temp_bytes);
  return c.off;
}

int mc_prepare(const float* sigma, int64_t n0, int64_t n1, int64_t n2, double thr, void* ws, size_t bytes, McParams* p,
               CubScratch* s, const char* who) {
  if (n0 < 2 || n1 < 2 || n2 < 2) return fail(NERFB200_EINVAL, "%s: every grid dimension must be >= 2", who);
  if (n0 * n1 * n2 > kMcMaxPoints) return fail(NERFB200_EUNSUPPORTED, "%s: grid larger than 4e8 points", who);
  if (!sigma || !ws) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  const long long P = n0 * n1 * n2, C = (n0 - 1) * (n1 - 1) * (n2 - 1);
  if (bytes < mc_carve(P, C, ws, p, s))
    return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_mc_workspace_bytes", who);
  p->sigma = sigma; p->n0 = n0; p->n1 = n1; p->n2 = n2; p->thr = thr;
  p->vertices = nullptr; p->triangles = nullptr;
  return 0;
}

// The cluster workspace of V vertices and T triangles, as mc_carve.
size_t cluster_carve(long long V, long long T, void* base, ClusterParams* p, CubScratch* s) {
  const long long E = 3 * T;
  size_t t1 = 0, t2 = 0, t3 = 0;
  cub::DoubleBuffer<unsigned long long> kb(nullptr, nullptr);
  cub::DoubleBuffer<int> vb(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, t1, kb, vb, static_cast<int>(E), 0, 2 * bits_for(V));
  cub::DeviceScan::ExclusiveSum(nullptr, t2, U8It(nullptr, U8ToInt()), static_cast<int*>(nullptr), static_cast<int>(T + 1));
  cub::DeviceScan::ExclusiveSum(nullptr, t3, U8It(nullptr, U8ToInt()), static_cast<int*>(nullptr), static_cast<int>(V + 1));
  s->temp_bytes = std::max({t1, t2, t3});
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  p->keys = c.take<unsigned long long>(E);
  s->keys_alt = c.take<unsigned long long>(E);
  p->vals = c.take<int>(E);
  s->vals_alt = c.take<int>(E);
  p->parent = c.take<int>(T);
  p->count = c.take<int>(T);
  p->best = c.take<unsigned long long>(1);
  p->tflag = c.take(T + 1);
  p->tofs = c.take<int>(T + 1);
  p->vflag = c.take(V + 1);
  p->vofs = c.take<int>(V + 1);
  s->temp = c.take(s->temp_bytes);
  return c.off;
}

int cluster_prepare(const int32_t* tris, int64_t n_tris, int64_t n_verts, void* ws, size_t bytes, ClusterParams* p,
                    CubScratch* s, const char* who) {
  if (n_tris < 0 || n_verts < 0 || n_tris > 0x7fffffffLL / 3 || n_verts > 0x7fffffffLL)
    return fail(NERFB200_EINVAL, "%s: bad mesh size", who);
  if (n_tris > 0 && (!tris || !ws)) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  const size_t need = cluster_carve(n_verts, n_tris, ws, p, s);
  if (n_tris > 0 && bytes < need)
    return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_mesh_cluster_workspace_bytes", who);
  p->tris = tris; p->n_tris = n_tris; p->n_verts = n_verts;
  p->vin = nullptr; p->vout = nullptr; p->tout = nullptr;
  return 0;
}

__global__ void cluster_pack_keys_kernel(unsigned long long* keys, long long n, int bits) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[t];
    keys[t] = ((k >> 32) << bits) | (k & 0xffffffffull);
  }
}

int read_two_counts(const int* a, const int* b, int64_t counts_host[2], cudaStream_t s, const char* who) {
  int h[2] = {0, 0};
  CUDA_TRY(cudaMemcpyAsync(&h[0], a, sizeof(int), cudaMemcpyDeviceToHost, s), who);
  CUDA_TRY(cudaMemcpyAsync(&h[1], b, sizeof(int), cudaMemcpyDeviceToHost, s), who);
  CUDA_TRY(cudaStreamSynchronize(s), who);
  counts_host[0] = h[0];
  counts_host[1] = h[1];
  return 0;
}

// The .vol indices are uint32 (extract_mesh.ipynb casts them): N^3 < 2^32 up to N = 1625.
constexpr long long kVolMaxN = 1625;

// The volume workspace of an N^3 grid (kVolTile points per tile), as mc_carve.
size_t volume_carve(long long N, void* base, VolumeParams* p, CubScratch* s) {
  const long long tiles = ceil_div(N * N * N, kVolTile);
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, static_cast<const unsigned long long*>(nullptr),
                                static_cast<unsigned long long*>(nullptr), static_cast<int>(tiles + 1));
  s->temp_bytes = tb;
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  p->tcnt = c.take<unsigned long long>(tiles + 1);
  p->tofs = c.take<unsigned long long>(tiles + 1);
  s->temp = c.take(s->temp_bytes);
  return c.off;
}

int volume_prepare(const float* rgbsigma, int64_t N, double xmin, double xmax, void* ws, size_t bytes, VolumeParams* p,
                   CubScratch* s, const char* who) {
  if (N < 2 || N > kVolMaxN) return fail(NERFB200_EINVAL, "%s: N must be in [2, 1625] (uint32 indices)", who);
  if (!rgbsigma || !ws) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  if (reinterpret_cast<uintptr_t>(rgbsigma) & 15) return fail(NERFB200_EINVAL, "%s: rgbsigma must be 16-byte aligned", who);
  if (bytes < volume_carve(N, ws, p, s))
    return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_volume_workspace_bytes", who);
  p->rgbsigma = reinterpret_cast<const float4*>(rgbsigma);
  p->P = N * N * N;
  // -(xmax - xmin) / N is a Python float; numpy rounds it to float32 before the multiply
  p->c = static_cast<float>(-(xmax - xmin) / static_cast<double>(N));
  p->out = nullptr;
  return 0;
}

// The vertex-normals workspace, as mc_carve: corner keys / triangle ids (and their sort buffers), triangle normals,
// the index flag.
size_t normals_carve(long long V, long long T, void* base, NormalsParams* p, CubScratch* s) {
  const long long E = 3 * T;
  size_t tb = 0;
  cub::DoubleBuffer<int> kb(nullptr, nullptr), vb(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, tb, kb, vb, static_cast<int>(E), 0, bits_for(V + 1));
  s->temp_bytes = tb;
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  p->keys = c.take<int>(E);
  s->keys_alt = c.take<int>(E);
  p->vals = c.take<int>(E);
  s->vals_alt = c.take<int>(E);
  p->tri_n = c.take<double>(T * 3);
  p->bad = c.take<int>(1);
  s->temp = c.take(s->temp_bytes);
  return c.off;
}

// V + 1 (the key of an out-of-range corner) and 3T stay in int32
bool normals_size_ok(long long V, long long T) {
  return V >= 0 && T >= 0 && V < 0x7fffffffLL && T <= 0x7fffffffLL / 3;
}

// ------------------------------------------------------------------ empty-space skipping
// (kernels: occupancy_kernels.cuh)

// The occupancy workspace of C cells: two byte-per-cell buffers the dilation passes alternate between.  A cascade
// reuses them level by level.
size_t occupancy_carve(long long C, void* base, uint8_t* buf[2]) {
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  buf[0] = c.take(C);
  buf[1] = c.take(C);
  return c.off;
}

// Dilate one level's occupancy bytes a by `dilate` cells (Chebyshev, within the level; b is the other buffer) and
// pack them into that level's words, the inner cells [ia, ib)^3 cleared.
int occupancy_finish(uint8_t* a, uint8_t* b, long long M, long long ia, long long ib, int32_t dilate, uint32_t* bits,
                     cudaStream_t s, const char* dilate_what, const char* pack_what) {
  const long long C = M * M * M;
  // a radius of M - 1 cells already reaches across the grid
  const int radius = static_cast<int>(dilate < M - 1 ? dilate : M - 1);
  if (radius > 0) {
    const long long stride[3] = {1, M, M * M};
    for (int ax = 0; ax < 3; ++ax) {
      TRY(launch(dilate_what, occ_dilate_axis_kernel, grid_blocks(C, 256), 256, 0, s, a, b, M, stride[ax], radius));
      std::swap(a, b);
    }
  }
  return launch(pack_what, occ_pack_kernel, grid_blocks(C, 256), 256, 0, s, a, M, ia, ib, bits);
}

// The cull workspace of n rays (kCullTile rays per tile): live rays per tile and their exclusive scan.
size_t cull_carve(long long n, void* base, CullParams* p) {
  const long long tiles = ceil_div(n, kCullTile);
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  p->tcnt = c.take<int>(tiles + 1);
  p->tofs = c.take<long long>(tiles + 1);
  return c.off;
}

int cull_prepare(const float* rays, int64_t n, void* ws, size_t bytes, CullParams* p, const char* who) {
  if (n < 0) return fail(NERFB200_EINVAL, "%s: n_rays < 0", who);
  if (n == 0) return 0;
  if (!rays || !ws) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  if (reinterpret_cast<uintptr_t>(rays) & 15) return fail(NERFB200_EINVAL, "%s: rays must be 16-byte aligned", who);
  if (bytes < cull_carve(n, ws, p)) return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_cull_workspace_bytes", who);
  p->rays = rays; p->n = n;
  p->grid.bits = nullptr; p->flag = nullptr; p->live_idx = nullptr; p->live_rays = nullptr;
  return 0;
}

// ------------------------------------------------------------------ the density grid (kernels: density_kernels.cuh)

// The workspace of an update of C cells, `chunk` (<= C) at a time: the chunk's points and sigma, then the two
// byte-per-cell buffers of occupancy_carve.
size_t density_carve(long long C, long long chunk, void* base, float** xyz, float** sigma, uint8_t* buf[2]) {
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  *xyz = c.take<float>(chunk * 3);
  *sigma = c.take<float>(chunk);
  c.off += occupancy_carve(C, base ? static_cast<uint8_t*>(base) + c.off : nullptr, buf);
  return c.off;
}

// The lattice of the density grid and of the per-sample skipping entries' occupancy grid: N in [2, 1625] points per
// axis and every range finite with min != max.
int grid_box_ok(int64_t N, const double* ranges, const char* who) {
  if (N < 2 || N > kVolMaxN) return fail(NERFB200_EINVAL, "%s: N must be in [2, 1625]", who);
  if (!ranges) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  for (int a = 0; a < 6; a += 2)
    if (!std::isfinite(ranges[a]) || !std::isfinite(ranges[a + 1]) || ranges[a] == ranges[a + 1])
      return fail(NERFB200_EINVAL, "%s: every range must be finite with min != max", who);
  return 0;
}

// Axis a of cascade level k's box (DESIGN.md §10h): the range as given at level 0; for k >= 1, with
// c = 0.5 (lo + hi) and h = 0.5 (hi - lo) in double, c -+ 2^k h (2^k h is exact, so each end is rounded once).
void level_range(const double* ranges, int k, int a, double* lo, double* hi) {
  if (k == 0) {
    *lo = ranges[2 * a];
    *hi = ranges[2 * a + 1];
    return;
  }
  const double c = 0.5 * (ranges[2 * a] + ranges[2 * a + 1]), h = 0.5 * (ranges[2 * a + 1] - ranges[2 * a]);
  const double e = std::ldexp(h, k);
  *lo = c - e;
  *hi = c + e;
}

// The grid size argument of the occupancy, culling, density and masked-grid entries (NERFB200_GRID_N): N points per
// axis in its low 32 bits and levels - 1 above them, so every value the one-level entries accepted means what it
// meant.  A negative value stays an N, which the N check rejects.
void grid_n(int64_t v, int64_t* N, int32_t* levels) {
  if (v < 0) {
    *N = v;
    *levels = 1;
    return;
  }
  const int64_t hi = v >> 32;
  *N = v & 0xffffffffLL;
  *levels = hi < kMaxLevels ? static_cast<int32_t>(hi + 1) : kMaxLevels + 1;
}

// grid_box_ok, and 1 <= levels <= kMaxLevels with every level's box finite with min != max.
int levels_ok(int64_t N, int32_t levels, const double* ranges, const char* who) {
  TRY(grid_box_ok(N, ranges, who));
  if (levels < 1 || levels > kMaxLevels) return fail(NERFB200_EINVAL, "%s: levels must be in [1, 8]", who);
  for (int k = 1; k < levels; ++k)
    for (int a = 0; a < 3; ++a) {
      double lo, hi;
      level_range(ranges, k, a, &lo, &hi);
      if (!std::isfinite(lo) || !std::isfinite(hi) || lo == hi)
        return fail(NERFB200_EINVAL, "%s: level %d's box is not finite with min != max", who, k);
    }
  return 0;
}

int density_box(int64_t N, int32_t levels, const double* ranges, int level, DensityBox* b, const char* who) {
  TRY(levels_ok(N, levels, ranges, who));
  for (int a = 0; a < 3; ++a) level_range(ranges, level, a, &b->lo[a], &b->hi[a]);
  b->M = N - 1;
  b->level = level;
  b->ia = level ? inner_lo(b->M) : 0;
  b->ib = level ? std::max(inner_hi(b->M), b->ia) : 0;
  return 0;
}

// The cells of level k an update evaluates: all of level 0, the non-inner ones of a level k >= 1.
long long level_cells(const DensityBox& b) {
  const long long n = b.ib - b.ia;
  return b.M * b.M * b.M - n * n * n;
}


// ------------------------------------------------------------------ per-sample skipping (kernels: sample_skip_kernels.cuh)
constexpr long long kSkipMaxRays = 1LL << 22;   // rows (n * S_f) and ray indices stay in int32

bool samples_shape_ok(long long n, int Sc, int K) {
  return n >= 0 && n <= kSkipMaxRays && (Sc == 32 || Sc == 64 || Sc == 128) && K >= 0 && K % 32 == 0 &&
         Sc + K <= kMaxSf;
}

// The workspace of n rays: per-ray masks, counts, offsets, fine depths and direction biases, and the compacted rows
// of the larger pass with their MLP outputs (16 bytes per row).
size_t samples_carve(long long n, int Sc, int K, void* base, SkipParams* p) {
  const long long Sf = Sc + K, rows = n * Sf;
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  p->mask[0] = c.take<uint32_t>(n * kSkipMaskWords);
  p->mask[1] = c.take<uint32_t>(n * kSkipMaskWords);
  p->cnt = c.take<int>(n + 1);
  p->ofs = c.take<long long>(n + 1);
  p->zf = c.take<float>(n * Sf);
  p->dirbias = c.take<float>(n * kSkipDirStride);
  p->row_ray = c.take<int>(rows);
  p->row_z = c.take<float>(rows);
  p->mlp_out = c.take<float>(rows * 4);
  p->zc = c.take<float>(n * Sc);    // the perturbed coarse depths (nerfb200_render_samples uses it with perturb > 0)
  return c.off;
}

// The compacted-row MLP of one pass over `rows` rows (mlp_forward_kernel's compacted-sample mode).
int samples_mlp(const SkipParams& sp, int pass, long long rows, bool sigma_only, void* stream) {
  MlpParams m{};
  m.n = rows;
  m.net = sp.net[pass];
  m.sigma_only = sigma_only;
  m.out = const_cast<float*>(sp.mlp_out);
  m.row_ray = sp.row_ray;
  m.row_z = sp.row_z;
  m.rays = sp.rays;
  m.dirbias = sp.dirbias + pass * kDirW;
  return launch_mlp(m, nullptr, stream, pass ? "render_samples fine mlp launch" : "render_samples coarse mlp launch");
}

// Scan the per-ray counts of the current pass and read the total back.
int samples_scan(const SkipParams& sp, cudaStream_t s, long long* total) {
  TRY(launch("render_samples scan launch", cull_scan_kernel, 1, 1024, 0, s, sp.cnt, sp.ofs, static_cast<long long>(sp.n)));
  CUDA_TRY(cudaMemcpyAsync(total, sp.ofs + sp.n, sizeof(*total), cudaMemcpyDeviceToHost, s), "render_samples readback");
  CUDA_TRY(cudaStreamSynchronize(s), "render_samples readback");
  return 0;
}

// The coarse pass of a coarse-only render with early ray termination (early_stop_kernels.cuh), after the
// classification: one round per mask word, then the final stage.  The per-ray state lives in the fine depths' part
// of the workspace, which a coarse-only render does not use: T and the state (12 bytes per ray) and the row bases
// (8 bytes per ray and word), S_c / 4 + 12 bytes per ray against zf's 4 S_c.  The rounds' rows together are the
// evaluated samples, at most the n S_c rows carved.
int samples_early_stop(const SkipParams& p, float eps, int32_t* cut_out, int ray_blocks, cudaStream_t s,
                       long long* live) {
  EarlyStop e{};
  e.eps = eps;
  e.words = p.Sc / 32;
  e.base = reinterpret_cast<long long*>(p.zf);
  e.T = reinterpret_cast<double*>(e.base + static_cast<long long>(e.words) * p.n);
  e.state = reinterpret_cast<int*>(e.T + p.n);
  e.cut_out = cut_out;
  const bool coarse_rgb = p.test_time == 0;
  TRY(launch("render_samples early_stop start launch", early_stop_start_kernel, ray_blocks, kSkipWarps * 32, 0, s, p, e));
  long long rows = 0;
  bool have_bias = false;
  for (int k = 0; k < e.words; ++k) {
    long long n_k = 0;
    TRY(samples_scan(p, s, &n_k));
    if (n_k > 0) {
      TRY(launch("render_samples early_stop emit launch", early_stop_emit_kernel, ray_blocks, kSkipWarps * 32, 0, s, p, e,
                 k, rows));
      if (coarse_rgb && !have_bias) {
        TRY(launch("render_samples dir_bias launch", skip_dir_bias_kernel, grid_blocks(p.n, 1), kDirW, 0, s, p, 0, 1));
        have_bias = true;
      }
      SkipParams q = p;          // the MLP writes this round's rows only
      q.row_ray += rows;
      q.row_z += rows;
      q.mlp_out += rows * (coarse_rgb ? 4 : 1);
      TRY(samples_mlp(q, 0, n_k, !coarse_rgb, s));
    }
    TRY(launch("render_samples early_stop round launch", early_stop_round_kernel, ray_blocks, kSkipWarps * 32, 0, s, p, e,
               k, coarse_rgb ? 0 : 1));
    rows += n_k;
  }
  TRY(launch("render_samples early_stop final launch", early_stop_final_kernel, ray_blocks, kSkipWarps * 32, 0, s, p, e));
  *live = rows;
  return 0;
}

// The random inputs of both per-sample skipping entries (the fields nerfb200_samples_args and
// nerfb200_train_samples_args share), checked and copied into p.
template <class A>
int skip_randoms(const A* a, const char* who, SkipParams* p) {
  const bool fine = a->n_importance > 0;
  if (a->rng_in_kernel < 0 || a->rng_in_kernel > 2) return fail(NERFB200_EINVAL, "%s: rng_in_kernel must be 0, 1 or 2", who);
  if (a->rng_in_kernel == 2 && !a->rng_seed) return fail(NERFB200_EINVAL, "%s: rng_in_kernel = 2 needs rng_seed", who);
  if (!(a->perturb >= 0.f) || !(a->noise_std >= 0.f)) return fail(NERFB200_EINVAL, "%s: perturb / noise_std < 0", who);
  if (a->perturb > 0.f && !a->rng_in_kernel && (!a->perturb_rand || (fine && !a->u_rand)))
    return fail(NERFB200_EINVAL, "%s: perturb>0 needs perturb_rand and u_rand", who);
  if (a->noise_std > 0.f && (!a->noise_coarse || (fine && !a->noise_fine)))
    return fail(NERFB200_EINVAL, "%s: noise_std>0 needs noise_coarse and noise_fine", who);
  p->perturb = a->perturb; p->noise_std = a->noise_std;
  p->perturb_rand = a->perturb_rand; p->u_rand = a->u_rand;
  p->noise[0] = a->noise_coarse; p->noise[1] = a->noise_fine;
  p->rng_seed = a->rng_seed; p->rng_in_kernel = a->rng_in_kernel;
  return 0;
}

// The occupancy grid of the cell walk, the per-sample skipping entries and the masked grids: every level's box.
int skip_grid(const uint32_t* bits, int64_t N, int32_t levels, const double* ranges, SkipGrid* g, const char* who) {
  TRY(levels_ok(N, levels, ranges, who));
  for (int k = 0; k < levels; ++k)
    for (int ax = 0; ax < 3; ++ax) {
      double lo, hi;
      level_range(ranges, k, ax, &lo, &hi);
      g->lo[k][ax] = lo;
      g->scale[k][ax] = static_cast<double>(N - 1) / (hi - lo);
    }
  g->bits = bits;
  g->M = N - 1;
  g->words = ceil_div(g->M * g->M * g->M, 32);
  g->levels = levels;
  return 0;
}

// ------------------------------------------------------------------ grids through an occupancy grid
// (kernels: masked_grid_kernels.cuh)

// The workspace of one chunk of `chunk` points: the tile counts, their scan and CUB's scratch, then the compacted
// positions, indices and query outputs.  The outputs are sized for four channels, so one size serves both entries.
size_t masked_grid_carve(long long chunk, void* base, MaskedGridParams* p, CubScratch* s) {
  const long long tiles = ceil_div(chunk, kMaskTile);
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, static_cast<const unsigned long long*>(nullptr),
                                static_cast<unsigned long long*>(nullptr), static_cast<int>(tiles + 1));
  s->temp_bytes = tb;
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  p->tcnt = c.take<unsigned long long>(tiles + 1);
  p->tofs = c.take<unsigned long long>(tiles + 1);
  s->temp = c.take(s->temp_bytes);
  p->xyz = c.take<float>(chunk * 3);
  p->idx = c.take<long long>(chunk);
  p->vals = c.take<float>(chunk * 4);
  return c.off;
}

// Both masked grids (channels 1 or 4), after the entry's own checks of N and the output.  Per chunk: classify, scan,
// one read-back of the evaluated count; with points to evaluate, emit, the point query and the scatter.
int masked_grid(const void* packed, int64_t N, const double* ranges, const uint32_t* bits, int64_t occ_grid_N,
                const double* occ_ranges, int64_t chunk, void* ws, size_t bytes, float* out, int64_t* evaluated_host,
                int channels, void* stream, const char* who) {
  if (chunk < 1) return fail(NERFB200_EINVAL, "%s: chunk < 1", who);
  if (!packed || !ranges || !bits || !occ_ranges || !ws || !out || !evaluated_host)
    return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  MaskedGridParams p{};
  int64_t occ_N;
  int32_t occ_levels;
  grid_n(occ_grid_N, &occ_N, &occ_levels);
  TRY(skip_grid(bits, occ_N, occ_levels, occ_ranges, &p.occ, who));
  CubScratch sc;
  if (bytes < masked_grid_carve(chunk, ws, &p, &sc))
    return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_masked_grid_workspace_bytes(chunk)", who);
  for (int a = 0; a < 3; ++a) { p.lo[a] = ranges[2 * a]; p.hi[a] = ranges[2 * a + 1]; }
  p.N = N;
  p.channels = channels;
  p.out = out;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long total = N * N * N;
  long long evaluated = 0;
  for (long long s0 = 0; s0 < total; s0 += chunk) {
    p.start = s0;
    p.count = total - s0 < chunk ? total - s0 : chunk;
    const long long tiles = ceil_div(p.count, kMaskTile);
    CUDA_TRY(cudaMemsetAsync(p.tcnt + tiles, 0, sizeof(unsigned long long), s), "masked grid memset");
    TRY(launch("masked grid classify launch", masked_grid_classify_kernel, grid_blocks(tiles * kMaskThreads, 256),
               kMaskThreads, 0, s, p));
    size_t tb = sc.temp_bytes;
    TRY(cub_launch(cub::DeviceScan::ExclusiveSum(sc.temp, tb, p.tcnt, p.tofs, static_cast<int>(tiles + 1), s),
                   "masked grid scan"));
    unsigned long long h = 0;
    CUDA_TRY(cudaMemcpyAsync(&h, p.tofs + tiles, sizeof(h), cudaMemcpyDeviceToHost, s), "masked grid readback");
    CUDA_TRY(cudaStreamSynchronize(s), "masked grid readback");
    if (h == 0) continue;
    const long long n = static_cast<long long>(h);
    TRY(launch("masked grid emit launch", masked_grid_emit_kernel, grid_blocks(tiles * kMaskThreads, 256), kMaskThreads,
               0, s, p));
    TRY(channels == 4 ? nerfb200_query_rgb_sigma(p.xyz, n, 3, packed, p.vals, stream)
                      : nerfb200_query_sigma(p.xyz, n, 3, packed, p.vals, stream));
    TRY(launch("masked grid scatter launch", masked_grid_scatter_kernel, grid_blocks(n, 256), 256, 0, s, p, n));
    evaluated += n;
  }
  *evaluated_host = evaluated;
  return 0;
}

// ------------------------------------------------------------------ sparse marching cubes
// (kernels: sparse_mc_kernels.cuh, entries: include/nerf_pl_b200_sparse_mc.h)
constexpr long long kSmcMaxN = 2048;
constexpr long long kSmcChunkBricks = 4096;   // active bricks per point query: at most 2^21 rows
constexpr long long kSmcMaxCount = 0x7fffffffLL;

long long smc_bricks(long long N) { return ceil_div(N, kBrick); }

using SmcVertIt = thrust::transform_iterator<SmcVerts, const unsigned*, unsigned long long>;
using SmcTriIt = thrust::transform_iterator<SmcTris, const unsigned*, unsigned long long>;
using SmcIndexIt = thrust::counting_iterator<int>;

// The plan workspace: per brick its map slot, flag, evaluated count and three lists; the selection counts.
size_t smc_plan_carve(long long N, void* base, SparseMcParams* p, CubScratch* s) {
  const long long nb = smc_bricks(N), B = nb * nb * nb;
  size_t tb = 0;
  cub::DeviceSelect::Flagged(nullptr, tb, SmcIndexIt(0), static_cast<const uint8_t*>(nullptr), static_cast<int*>(nullptr),
                             static_cast<int*>(nullptr), static_cast<int>(B));
  s->temp_bytes = tb;
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  p->nsel = c.take<int>(4);
  p->map = c.take<int>(B);
  p->flag = c.take(B);
  p->cnt = c.take<int>(B);
  p->cand = c.take<int>(B);
  p->active = c.take<int>(B);
  p->march = c.take<int>(B);
  s->temp = c.take(s->temp_bytes);
  return c.off;
}

// The count / emit workspace of A active and Mb march bricks: V and T, the row counts and offsets, the active
// bricks' values, one query's rows, the march bricks' counts and offsets, and the scans' scratch.
size_t smc_carve(long long A, long long Mb, void* base, SparseMcParams* p, unsigned long long** rcnt,
                 unsigned long long** vt, CubScratch* s) {
  const long long rows = std::min(A, kSmcChunkBricks) * kBrickPoints;
  size_t t1 = 0, t2 = 0, t3 = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, t1, static_cast<const unsigned long long*>(nullptr),
                                static_cast<unsigned long long*>(nullptr), static_cast<int>(A + 1));
  cub::DeviceScan::ExclusiveSum(nullptr, t2, SmcVertIt(nullptr, SmcVerts()), static_cast<unsigned long long*>(nullptr),
                                static_cast<int>(Mb + 1));
  cub::DeviceScan::ExclusiveSum(nullptr, t3, SmcTriIt(nullptr, SmcTris()), static_cast<unsigned long long*>(nullptr),
                                static_cast<int>(Mb + 1));
  s->temp_bytes = std::max({t1, t2, t3});
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  *vt = c.take<unsigned long long>(2);
  *rcnt = c.take<unsigned long long>(A + 1);
  p->rofs = c.take<unsigned long long>(A + 1);
  p->vals = c.take<float>(A * kBrickPoints);
  p->xyz = c.take<float>(rows * 3);
  p->dst = c.take<long long>(rows);
  p->out = c.take<float>(rows);
  p->bcnt = c.take<unsigned>(Mb + 1);
  p->vofs = c.take<unsigned long long>(Mb + 1);
  p->tofs = c.take<unsigned long long>(Mb + 1);
  s->temp = c.take(s->temp_bytes);
  return c.off;
}

// The emit workspace of V vertex and T triangle keys: both sort buffers of each and the sorts' scratch.
size_t smc_emit_carve(long long V, long long T, void* base, unsigned long long* vk[2], unsigned long long* tk[2],
                      CubScratch* s) {
  size_t t1 = 0, t2 = 0;
  cub::DoubleBuffer<unsigned long long> kb(nullptr, nullptr);
  cub::DeviceRadixSort::SortKeys(nullptr, t1, kb, static_cast<int>(V), 0, 64);
  cub::DeviceRadixSort::SortKeys(nullptr, t2, kb, static_cast<int>(T), 0, 64);
  s->temp_bytes = std::max(t1, t2);
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  vk[0] = c.take<unsigned long long>(V);
  vk[1] = c.take<unsigned long long>(V);
  tk[0] = c.take<unsigned long long>(T);
  tk[1] = c.take<unsigned long long>(T);
  s->temp = c.take(s->temp_bytes);
  return c.off;
}

bool smc_counts_ok(long long N, long long A, long long Mb) {
  const long long nb = smc_bricks(N);
  return N >= 2 && N <= kSmcMaxN && A >= 0 && Mb >= A && Mb <= nb * nb * nb && (A > 0 || Mb == 0);
}

// The mesh grid, N and (with bits) the occupancy grid into p.
int smc_grids(int64_t N, const double* ranges, const uint32_t* bits, int64_t occ_grid_N, const double* occ_ranges,
              SparseMcParams* p, const char* who) {
  if (N < 2 || N > kSmcMaxN) return fail(NERFB200_EINVAL, "%s: N must be in [2, 2048]", who);
  if (!ranges || !bits || !occ_ranges) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  int64_t occ_N;
  int32_t occ_levels;
  grid_n(occ_grid_N, &occ_N, &occ_levels);
  TRY(skip_grid(bits, occ_N, occ_levels, occ_ranges, &p->m.occ, who));
  for (int a = 0; a < 3; ++a) { p->m.lo[a] = ranges[2 * a]; p->m.hi[a] = ranges[2 * a + 1]; }
  p->m.N = N;
  p->m.start = 0;
  p->nb = smc_bricks(N);
  return 0;
}

int smc_select(const SparseMcParams& p, CubScratch& sc, int* out, int* count, cudaStream_t s, const char* what) {
  size_t tb = sc.temp_bytes;
  const long long B = p.nb * p.nb * p.nb;
  return cub_launch(cub::DeviceSelect::Flagged(sc.temp, tb, SmcIndexIt(0), p.flag, out, count, static_cast<int>(B), s),
                    what);
}

// The evaluated points of the A > 0 active bricks through the point query on compacted rows: their row counts (rcnt)
// and first rows (p.rofs), then per kSmcChunkBricks bricks the rows (smc_sigma_emit_kernel), the query into p.out
// (`channels`: 1 for sigma, 4 for nerfb200_query_rgb_sigma, 28 for nerfb200_query_rgb_sh with its workspace sh_ws)
// and `scatter(rows)`, which enqueues the chunk's scatter.  Reads the chunks' row bounds back, so it synchronises.
template <class Scatter>
int smc_query(SparseMcParams& p, const CubScratch& sc, unsigned long long* rcnt, long long A, const void* packed,
              int channels, void* sh_ws, cudaStream_t s, Scatter&& scatter) {
  TRY(launch("sparse_mc row counts launch", smc_row_counts_kernel, grid_blocks(A + 1, 256), 256, 0, s, p, rcnt));
  size_t tb = sc.temp_bytes;
  TRY(cub_launch(cub::DeviceScan::ExclusiveSum(sc.temp, tb, rcnt, p.rofs, static_cast<int>(A + 1), s), "sparse_mc row scan"));
  const long long chunks = ceil_div(A, kSmcChunkBricks);
  std::vector<unsigned long long> bound(chunks + 1);
  CUDA_TRY(cudaMemcpy2DAsync(bound.data(), sizeof(unsigned long long), p.rofs, kSmcChunkBricks * sizeof(unsigned long long),
                             sizeof(unsigned long long), chunks, cudaMemcpyDeviceToHost, s), "sparse_mc row readback");
  CUDA_TRY(cudaMemcpyAsync(bound.data() + chunks, p.rofs + A, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s),
           "sparse_mc row readback");
  CUDA_TRY(cudaStreamSynchronize(s), "sparse_mc row readback");
  for (long long c = 0; c < chunks; ++c) {
    const long long rows = static_cast<long long>(bound[c + 1] - bound[c]);
    if (rows == 0) continue;
    p.slot0 = c * kSmcChunkBricks;
    p.slots = std::min(kSmcChunkBricks, A - p.slot0);
    TRY(launch("sparse_mc sigma emit launch", smc_sigma_emit_kernel, grid_blocks(p.slots, 1), kBrickPoints, 0, s, p));
    TRY(channels == 28 ? nerfb200_query_rgb_sh(p.xyz, rows, 3, packed, sh_ws, nerfb200_query_rgb_sh_workspace_bytes(),
                                               p.out, s)
        : channels == 4 ? nerfb200_query_rgb_sigma(p.xyz, rows, 3, packed, p.out, s)
                        : nerfb200_query_sigma(p.xyz, rows, 3, packed, p.out, s));
    TRY(scatter(rows));
  }
  return 0;
}

// ------------------------------------------------------------------ baked volumes
// (kernels: baked_kernels.cuh, entries: include/nerf_pl_b200_baked.h, and include/nerf_pl_b200_baked_sh.h for the
// view-dependent kind of kW = 7 float4 per point).  The brick plan and its workspace are the sparse marching cubes'
// (nerfb200_sparse_mc_plan); a volume stores the plan's march bricks.
constexpr long long kBakedShMaxN = 1024;
long long baked_max_n(int W) { return W == 1 ? kSmcMaxN : kBakedShMaxN; }          // bake, render
long long baked_dense_max_n(int W) { return W == 1 ? kVolMaxN : kBakedShMaxN; }    // from_grid, to_dense
const char* baked_api(int W) { return W == 1 ? "nerfb200_baked" : "nerfb200_baked_sh"; }

size_t baked_bytes(long long N, long long bricks, int W = 1) {
  const long long nb = smc_bricks(N);
  return static_cast<size_t>(bricks) * kBakedPoints * W * sizeof(float4) + static_cast<size_t>(nb * nb * nb) * sizeof(int);
}

bool baked_bricks_ok(long long N, long long bricks, int W = 1) {
  const long long nb = smc_bricks(N);
  return N >= 2 && N <= baked_max_n(W) && bricks >= 0 && bricks <= nb * nb * nb;
}

// The bake's workspace for A active bricks: the row counts and offsets, one query's rows (positions, destinations and
// 4 W outputs each), the scan's scratch and, for W > 1, the SH query's table (sh_ws).
size_t baked_carve(long long A, void* base, SparseMcParams* p, unsigned long long** rcnt, CubScratch* s, int W = 1,
                   void** sh_ws = nullptr) {
  const long long rows = std::min(A, kSmcChunkBricks) * kBrickPoints;
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, static_cast<const unsigned long long*>(nullptr),
                                static_cast<unsigned long long*>(nullptr), static_cast<int>(A + 1));
  s->temp_bytes = tb;
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  *rcnt = c.take<unsigned long long>(A + 1);
  p->rofs = c.take<unsigned long long>(A + 1);
  p->xyz = c.take<float>(rows * 3);
  p->dst = c.take<long long>(rows);
  p->out = c.take<float>(rows * 4 * W);
  s->temp = c.take(s->temp_bytes);
  if (W > 1) *sh_ws = c.take<float>(kShTableFloats);
  return c.off;
}

// A volume buffer of `bricks` stored bricks at N, W float4 per point: its data and map.
int baked_volume(const void* volume, size_t volume_bytes, int64_t N, int64_t bricks, float4** data, int** map,
                 const char* who, int W = 1) {
  if (N < 2 || N > baked_max_n(W)) return fail(NERFB200_EINVAL, "%s: N must be in [2, %lld]", who, baked_max_n(W));
  if (!baked_bricks_ok(N, bricks, W)) return fail(NERFB200_EINVAL, "%s: bricks must be in [0, ceil(N / 8)^3]", who);
  if (!volume) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  if (volume_bytes != baked_bytes(N, bricks, W))
    return fail(NERFB200_EINVAL, "%s: volume_bytes differs from %s_bytes(N, bricks)", who, baked_api(W));
  *data = static_cast<float4*>(const_cast<void*>(volume));
  *map = reinterpret_cast<int*>(static_cast<uint8_t*>(const_cast<void*>(volume)) +
                                static_cast<size_t>(bricks) * kBakedPoints * W * sizeof(float4));
  return 0;
}

// The map of the `count` bricks of `list` (device values) and zeroed data.
int baked_map(const int* list, const int* count, long long nb, long long bricks, float4* data, int* map, cudaStream_t s,
              int W = 1) {
  CUDA_TRY(cudaMemsetAsync(map, 0xff, static_cast<size_t>(nb * nb * nb) * sizeof(int), s), "baked memset");
  if (bricks == 0) return 0;
  CUDA_TRY(cudaMemsetAsync(data, 0, static_cast<size_t>(bricks) * kBakedPoints * W * sizeof(float4), s), "baked memset");
  return launch("baked map launch", baked_map_kernel, grid_blocks(bricks, 256), 256, 0, s, list, count, map);
}

// The entries of both kinds, kW float4 per point (`who`: the entry's name in messages).
template <int kW>
int baked_bake(const char* who, const void* packed, int64_t N, const double ranges_host[6], const uint32_t* bits,
               int64_t occ_N, const double occ_ranges_host[6], void* plan_ws, size_t plan_bytes,
               const int64_t bricks_host[2], void* ws, size_t bytes, void* volume, size_t volume_bytes, void* stream) {
  if (N < 2 || N > baked_max_n(kW)) return fail(NERFB200_EINVAL, "%s: N must be in [2, %lld]", who, baked_max_n(kW));
  SparseMcParams p{};
  TRY(smc_grids(N, ranges_host, bits, occ_N, occ_ranges_host, &p, who));
  if (!packed || !plan_ws || !bricks_host || !ws || !volume) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  const long long A = bricks_host[0], Mb = bricks_host[1];
  if (!smc_counts_ok(N, A, Mb)) return fail(NERFB200_EINVAL, "%s: bricks_host is not a plan's {active, march}", who);
  CubScratch sc, sq;
  if (plan_bytes < smc_plan_carve(N, plan_ws, &p, &sc))
    return fail(NERFB200_EINVAL, "%s: plan workspace smaller than nerfb200_sparse_mc_plan_workspace_bytes(N)", who);
  unsigned long long* rcnt;
  void* sh_ws = nullptr;
  if (bytes < baked_carve(A, ws, &p, &rcnt, &sq, kW, &sh_ws))
    return fail(NERFB200_EINVAL, "%s: workspace smaller than %s_workspace_bytes(N, active, march)", who, baked_api(kW));
  float4* data;
  int* map;
  TRY(baked_volume(volume, volume_bytes, N, Mb, &data, &map, who, kW));
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int h[2] = {0, 0};
  CUDA_TRY(cudaMemcpyAsync(h, p.nsel + 1, sizeof(h), cudaMemcpyDeviceToHost, s), "baked bake readback");
  CUDA_TRY(cudaStreamSynchronize(s), "baked bake readback");
  if (h[0] != A || h[1] != Mb) return fail(NERFB200_EINVAL, "%s: bricks_host differs from the plan's", who);
  TRY(baked_map(p.march, p.nsel + 2, p.nb, Mb, data, map, s, kW));
  if (A == 0) return 0;
  TRY(smc_query(p, sq, rcnt, A, packed, 4 * kW, sh_ws, s, [&](long long rows) {
    return launch("baked scatter launch", baked_scatter_kernel<kW>, grid_blocks(rows, 256), 256, 0, s, p, map, data, rows);
  }));
  return launch("baked apron launch", baked_apron_kernel<kW>, grid_blocks(Mb * kBakedPoints, 256), 256, 0, s, p.march,
                p.nsel + 2, map, p.nb, data);
}

template <int kW>
int baked_from_grid_count(const char* who, const float* grid, int64_t N, void* plan_ws, size_t plan_bytes,
                          int64_t bricks_host[1], void* stream) {
  const long long top = baked_dense_max_n(kW);
  if (N < 2 || N > top) return fail(NERFB200_EINVAL, "%s: N must be in [2, %lld]", who, top);
  if (!grid || !plan_ws || !bricks_host) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  SparseMcParams p{};
  p.nb = smc_bricks(N);
  CubScratch sc;
  if (plan_bytes < smc_plan_carve(N, plan_ws, &p, &sc))
    return fail(NERFB200_EINVAL, "%s: plan workspace smaller than nerfb200_sparse_mc_plan_workspace_bytes(N)", who);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long B = p.nb * p.nb * p.nb;
  TRY(launch("baked grid flag launch", baked_grid_flag_kernel<kW>, grid_blocks(B, 1), 256, 0, s,
             reinterpret_cast<const float4*>(grid), static_cast<long long>(N), p.nb, p.flag));
  TRY(smc_select(p, sc, p.march, p.nsel + 2, s, "baked grid select"));
  int h = 0;
  CUDA_TRY(cudaMemcpyAsync(&h, p.nsel + 2, sizeof(h), cudaMemcpyDeviceToHost, s), "baked from_grid readback");
  CUDA_TRY(cudaStreamSynchronize(s), "baked from_grid readback");
  bricks_host[0] = h;
  return 0;
}

template <int kW>
int baked_from_grid(const char* who, const float* grid, int64_t N, void* plan_ws, size_t plan_bytes, int64_t bricks,
                    void* volume, size_t volume_bytes, void* stream) {
  const long long top = baked_dense_max_n(kW);
  if (N < 2 || N > top) return fail(NERFB200_EINVAL, "%s: N must be in [2, %lld]", who, top);
  if (!grid || !plan_ws) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  float4* data;
  int* map;
  TRY(baked_volume(volume, volume_bytes, N, bricks, &data, &map, who, kW));
  SparseMcParams p{};
  p.nb = smc_bricks(N);
  CubScratch sc;
  if (plan_bytes < smc_plan_carve(N, plan_ws, &p, &sc))
    return fail(NERFB200_EINVAL, "%s: plan workspace smaller than nerfb200_sparse_mc_plan_workspace_bytes(N)", who);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int h = 0;
  CUDA_TRY(cudaMemcpyAsync(&h, p.nsel + 2, sizeof(h), cudaMemcpyDeviceToHost, s), "baked from_grid readback");
  CUDA_TRY(cudaStreamSynchronize(s), "baked from_grid readback");
  if (h != bricks) return fail(NERFB200_EINVAL, "%s: bricks differs from %s_from_grid_count's", who, baked_api(kW));
  TRY(baked_map(p.march, p.nsel + 2, p.nb, bricks, data, map, s, kW));
  if (bricks == 0) return 0;
  return launch("baked grid copy launch", baked_grid_copy_kernel<kW>, grid_blocks(bricks * kBakedPoints, 256), 256, 0, s,
                reinterpret_cast<const float4*>(grid), static_cast<long long>(N), p.march, p.nsel + 2, p.nb, data);
}

template <int kW>
int baked_to_dense(const char* who, const void* volume, size_t volume_bytes, int64_t N, int64_t bricks, float* grid,
                   void* stream) {
  const long long top = baked_dense_max_n(kW);
  if (N < 2 || N > top) return fail(NERFB200_EINVAL, "%s: N must be in [2, %lld]", who, top);
  float4* data;
  int* map;
  TRY(baked_volume(volume, volume_bytes, N, bricks, &data, &map, who, kW));
  if (!grid) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  return launch("baked to_dense launch", baked_to_dense_kernel<kW>, grid_blocks(N * N * N, 256), 256, 0, stream, data,
                map, static_cast<long long>(N), smc_bricks(N), reinterpret_cast<float4*>(grid));
}

template <int kW>
int baked_render(const char* who, const void* volume, size_t volume_bytes, int64_t N, const double ranges_host[6],
                 int64_t bricks, const float* rays, int64_t n_rays, double step, int32_t white_back, double early_stop,
                 float* rgb, float* depth, float* opacity, void* stream) {
  BakedRenderParams r{};
  float4* data;
  int* map;
  TRY(baked_volume(volume, volume_bytes, N, bricks, &data, &map, who, kW));
  if (!ranges_host) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  for (int a = 0; a < 3; ++a) {
    const float lo = static_cast<float>(ranges_host[2 * a]), hi = static_cast<float>(ranges_host[2 * a + 1]);
    const float scale = static_cast<float>(static_cast<double>(N - 1) / (ranges_host[2 * a + 1] - ranges_host[2 * a]));
    if (!std::isfinite(lo) || !std::isfinite(hi) || lo == hi || !std::isfinite(scale) || scale == 0.f)
      return fail(NERFB200_EINVAL, "%s: every range must be finite with min != max in float32", who);
    r.lo[a] = lo;
    r.scale[a] = scale;
  }
  const float s32 = static_cast<float>(step);
  if (!(step > 0.0) || !std::isfinite(s32) || !(s32 > 0.f))
    return fail(NERFB200_EINVAL, "%s: step must be > 0 and finite in float32", who);
  if (!(early_stop >= 0.0 && early_stop <= 1.0)) return fail(NERFB200_EINVAL, "%s: early_stop must be in [0, 1]", who);
  if (white_back != 0 && white_back != 1) return fail(NERFB200_EINVAL, "%s: white_back must be 0 or 1", who);
  if (n_rays < 0) return fail(NERFB200_EINVAL, "%s: n_rays < 0", who);
  if (n_rays > 0 && (!rays || !rgb || !depth || !opacity)) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  if (n_rays == 0) return 0;
  r.data = data;
  r.map = map;
  r.N = static_cast<int>(N);
  r.nb = static_cast<int>(smc_bricks(N));
  r.step = s32;
  r.eps = static_cast<float>(early_stop);
  r.white_back = static_cast<float>(white_back);
  r.rays = rays;
  r.n = n_rays;
  r.rgb = rgb;
  r.depth = depth;
  r.opacity = opacity;
  return launch("baked render launch", baked_render_kernel<kW>, grid_blocks(n_rays, kBakedThreads, 0x7fffffffLL),
                kBakedThreads, 0, stream, r);
}

// The SH fit of DESIGN.md §10k, made once in float64 and rounded to float32: the Fibonacci-sphere directions and
// P = pinv(Y) = (Y^T Y)^-1 Y^T, Y the 64 x 9 basis matrix at the float32 directions (cond(Y) = 1.014, so the normal
// equations lose nothing that float32 keeps).
struct ShFitHost {
  ShFit f;
  ShFitHost() {
    const double C0 = 0.28209479177387814, C1 = 0.4886025119029199;
    const double C2[5] = {1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792,
                          0.5462742152960396};
    double Y[kShDirs][kShBasis];
    for (int j = 0; j < kShDirs; ++j) {
      const double z = 1.0 - (2.0 * j + 1.0) / kShDirs, phi = j * M_PI * (3.0 - std::sqrt(5.0));
      const double rr = std::sqrt(1.0 - z * z);
      const double d[3] = {rr * std::cos(phi), rr * std::sin(phi), z};
      for (int a = 0; a < 3; ++a) f.dirs[3 * j + a] = static_cast<float>(d[a]);
      const double x = f.dirs[3 * j], y = f.dirs[3 * j + 1], zz = f.dirs[3 * j + 2];
      const double b[kShBasis] = {C0, -C1 * y, C1 * zz, -C1 * x, C2[0] * x * y, C2[1] * y * zz,
                                  C2[2] * (2.0 * zz * zz - x * x - y * y), C2[3] * x * zz, C2[4] * (x * x - y * y)};
      for (int m = 0; m < kShBasis; ++m) Y[j][m] = b[m];
    }
    // [Y^T Y | Y^T], reduced by Gauss-Jordan with partial pivoting to [I | P]
    double M[kShBasis][kShBasis + kShDirs];
    for (int a = 0; a < kShBasis; ++a) {
      for (int b = 0; b < kShBasis; ++b) {
        double acc = 0.0;
        for (int j = 0; j < kShDirs; ++j) acc += Y[j][a] * Y[j][b];
        M[a][b] = acc;
      }
      for (int j = 0; j < kShDirs; ++j) M[a][kShBasis + j] = Y[j][a];
    }
    for (int c = 0; c < kShBasis; ++c) {
      int piv = c;
      for (int r = c + 1; r < kShBasis; ++r)
        if (std::fabs(M[r][c]) > std::fabs(M[piv][c])) piv = r;
      for (int k = 0; k < kShBasis + kShDirs; ++k) std::swap(M[c][k], M[piv][k]);
      const double inv = 1.0 / M[c][c];
      for (int k = 0; k < kShBasis + kShDirs; ++k) M[c][k] *= inv;
      for (int r = 0; r < kShBasis; ++r) {
        if (r == c) continue;
        const double g = M[r][c];
        for (int k = 0; k < kShBasis + kShDirs; ++k) M[r][k] -= g * M[c][k];
      }
    }
    for (int m = 0; m < kShBasis; ++m)
      for (int j = 0; j < kShDirs; ++j) f.proj[m * kShDirs + j] = static_cast<float>(M[m][kShBasis + j]);
  }
};
const ShFit& sh_fit() {
  static const ShFitHost h;
  return h.f;
}

// ------------------------------------------------------------------ training with empty samples skipped
// (kernels: sample_skip_kernels.cuh, train_skip_kernels.cuh).  One workspace per batch shape, sized for every sample
// evaluated: the per-ray buffers, the compacted rows of the larger pass, then per network a NeRF.forward training
// workspace carved for that worst case and the device plan of its backward.  Nothing is reallocated or re-zeroed
// between steps, and no launch is sized on the host from a step's sample count: each pass's count stays on the device
// (the total of its scan), the compacted-row MLP reads it, and train_skip_plan_kernel turns it into the backward's
// layout, wgrad tables, head / chain parameters and reduction table.  Every launch has the grid of the carved worst
// case, so the step can be captured in a CUDA graph.
struct TrainSkipWs {
  SkipParams p;                 // p.ofs: the offsets of the pass a launch works on (ofs[pass] below)
  long long* ofs[2];            // (n + 1) exclusive scans of the evaluated samples of each pass
  uint8_t* net_ws[2];
  TrainSkipPlan* plan[2];
  long long* live;              // [2] the eager forward's counts, read back once
  long long cap[2];             // rows of each network with every sample evaluated
};

size_t train_skip_carve(long long n, int Sc, int K, void* base, int sm_count, TrainSkipWs* w) {
  const long long Sf = Sc + K, rows = n * Sf;
  Carver c{static_cast<uint8_t*>(base), 0, 1024};
  SkipParams& p = w->p;
  p.mask[0] = c.take<uint32_t>(n * kSkipMaskWords);
  p.mask[1] = c.take<uint32_t>(n * kSkipMaskWords);
  p.cnt = c.take<int>(n + 1);
  w->ofs[0] = c.take<long long>(n + 1);
  w->ofs[1] = c.take<long long>(n + 1);
  p.zc = c.take<float>(n * Sc);
  p.zf = c.take<float>(n * Sf);
  p.dirbias = c.take<float>(n * kSkipDirStride);
  p.dirrow = c.take<__half>(n * 64);
  p.row_ray = c.take<int>(rows);
  p.row_z = c.take<float>(rows);
  p.mlp_out = c.take<float>(rows * 4);
  w->live = c.take<long long>(2);
  w->net_ws[0] = w->net_ws[1] = nullptr;
  w->plan[0] = w->plan[1] = nullptr;
  w->cap[0] = w->cap[1] = 0;
  for (int ps = 0; ps < (K > 0 ? 2 : 1); ++ps) {
    w->cap[ps] = n * (ps ? Sf : Sc);
    TrainLayout L;
    make_train_layout(&L, nullptr, true, w->cap[ps], 1, 0, sm_count);
    w->net_ws[ps] = c.take(L.bytes);
    w->plan[ps] = c.take<TrainSkipPlan>(1);
  }
  return c.off;
}

// The NeRF.forward training layout of `rows` rows inside a layout carved for more: every buffer keeps its worst-case
// address; the row count, the padded row count (the stride of the activation layers) and the head kernel's
// pseudo-rays and blocks are the step's.  With the wgrad plan (plan_wgrad) this plan of fewer rows needs no more
// CTAs, pieces or head blocks than the carved one.
__host__ __device__ void train_skip_rows(TrainLayout* L, long long rows) {
  PassBufs& b = L->pass[0];
  b.n = rows;
  b.n_pad = (rows + 127) / 128 * 128;
  L->n_rays = static_cast<int>(b.n_pad / kMlpPseudoRay);
  L->head_grid = (L->n_rays + kHeadWarps - 1) / kHeadWarps;
}

// The backward plans of the networks from their evaluated rows, block ps for network ps (one thread each): the step's
// layout, its wgrad piece table and CTA ranges in the workspace's tables (the CTAs past the step's own up to the carved
// count get empty ranges), the head and chain parameters and the reduction table, each from the planner the host uses
// for the plain paths.  The plan is built in local memory and stored once.
struct TrainSkipPlanArgs {
  TrainLayout L[2];             // carved for each network's worst case
  const long long* rows[2];     // device: the pass's evaluated rows (null: no plan for that network)
  const float* params[2][24];
  float* grads[2][24];
  const uint8_t* net[2];
  TrainSkipPlan* out[2];
  int sm_count;
  int* status;
};

__global__ void __launch_bounds__(32) train_skip_plan_kernel(const TrainSkipPlanArgs a) {
  __shared__ TrainSkipPlan o;
  const int ps = blockIdx.x;
  if (a.rows[ps] == nullptr) return;
  if (threadIdx.x == 0) {
    TrainLayout L = a.L[ps];
    const int cap_ctas = L.n_cta;
    train_skip_rows(&L, *a.rows[ps]);
    plan_wgrad(&L, a.sm_count, L.jobs_dev, L.cta_first_dev);
    for (int b = L.n_cta + 1; b <= cap_ctas; ++b) L.cta_first_dev[b] = L.n_jobs;
    head_plan(L, a.params[ps][22], a.params[ps][22], nullptr, 0, &o.head);
    o.head_grid = L.head_grid;
    const uint8_t* const net[2] = {a.net[ps], a.net[ps]};
    chain_plan(L, net, a.status, a.sm_count, &o.probe, &o.chain);
    o.tab.n = 0;
    add_reduce_items(o.tab, L, 0, a.grads[ps]);
  }
  __syncwarp();
  // the warp stores the plan
  static_assert(sizeof(TrainSkipPlan) % 8 == 0, "plan words");
  const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&o);
  unsigned long long* dst = reinterpret_cast<unsigned long long*>(a.out[ps]);
  for (int i = threadIdx.x; i < static_cast<int>(sizeof(TrainSkipPlan) / 8); i += 32) dst[i] = src[i];
}

// The argument checks of both entries, and the step's parameters and workspace carve.
int train_skip_setup(const nerfb200_train_samples_args* a, void* ws, size_t bytes, int sm_count, TrainSkipWs* w,
                     const char* who) {
  if (!a) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  if (!samples_shape_ok(a->n_rays, a->n_samples, a->n_importance) || a->n_rays < 1)
    return fail(NERFB200_EUNSUPPORTED, "%s: needs N_samples in {32, 64, 128}, N_importance a multiple of 32, "
                "N_samples + N_importance <= 192 and 1 <= n_rays <= 2^22", who);
  std::memset(w, 0, sizeof(*w));
  SkipParams& p = w->p;
  TRY(skip_grid(a->bits, a->N, a->levels ? a->levels : 1, a->ranges, &p.grid, who));
  const bool fine = a->n_importance > 0;
  // target and loss_out: both (the fused loss) or neither (the upstream gradients alone)
  if (!a->rays || !a->packed_coarse || !a->bits || !a->target != !a->loss_out || !a->rgb_coarse || !a->depth_coarse ||
      !a->opacity_coarse || !ws)
    return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  if (fine && (!a->packed_fine || !a->rgb_fine || !a->depth_fine || !a->opacity_fine))
    return fail(NERFB200_EINVAL, "%s: packed_fine / fine outputs are NULL with N_importance>0", who);
  TRY(skip_randoms(a, who, &p));
  if ((reinterpret_cast<uintptr_t>(a->rays) | reinterpret_cast<uintptr_t>(a->packed_coarse) |
       reinterpret_cast<uintptr_t>(a->packed_fine) | reinterpret_cast<uintptr_t>(a->samples_coarse) |
       reinterpret_cast<uintptr_t>(a->samples_fine)) & 15)
    return fail(NERFB200_EINVAL, "%s: rays, packed images and samples must be 16-byte aligned", who);
  if (reinterpret_cast<uintptr_t>(ws) & 1023) return fail(NERFB200_EINVAL, "%s: workspace must be 1024-byte aligned", who);
  if (bytes < train_skip_carve(a->n_rays, a->n_samples, a->n_importance, ws, sm_count, w))
    return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_train_samples_workspace_bytes", who);
  p.rays = a->rays; p.n = static_cast<int>(a->n_rays);
  p.Sc = a->n_samples; p.K = a->n_importance; p.use_disp = a->use_disp; p.white_back = a->white_back;
  p.net[0] = static_cast<const uint8_t*>(a->packed_coarse);
  p.net[1] = static_cast<const uint8_t*>(a->packed_fine);
  p.rgb_coarse = a->rgb_coarse; p.depth_coarse = a->depth_coarse; p.opacity_coarse = a->opacity_coarse;
  p.rgb_fine = a->rgb_fine; p.depth_fine = a->depth_fine; p.opacity_fine = a->opacity_fine;
  p.z_fine = a->z_fine; p.weights_coarse = a->weights_coarse; p.weights_fine = a->weights_fine;
  p.samples[0] = a->samples_coarse; p.samples[1] = a->samples_fine;
  p.z_coarse = a->z_coarse;
  return 0;
}

// The training MLP of one network over the pass's compacted rows (mlp_forward_kernel<true, true>), at the grid of
// the carved worst case; the kernel reads the row count from the pass's scan.
int train_skip_mlp(const TrainSkipWs& w, int pass, const DeviceInfo* d, cudaStream_t s) {
  const SkipParams& p = w.p;
  TrainLayout L;
  make_train_layout(&L, w.net_ws[pass], true, w.cap[pass], 1, 0, d->sm_count);
  MlpParams m{};
  m.n = w.cap[pass];
  m.n_dev = w.ofs[pass] + p.n;
  m.net = p.net[pass];
  m.out = const_cast<float*>(p.mlp_out);
  m.status = d->status;
  m.tr = L.pass[0];
  m.xdir = L.xdir;
  m.row_ray = p.row_ray;
  m.row_z = p.row_z;
  m.rays = p.rays;
  m.dirbias = p.dirbias + pass * kDirW;
  m.dirrow = p.dirrow;
  const long long tiles = ceil_div(m.n, 128);
  return launch(pass ? "train_samples fine mlp launch" : "train_samples coarse mlp launch", mlp_forward_kernel<true, true>,
                static_cast<int>(tiles < d->sm_count ? tiles : d->sm_count), kThreads, kSmemTotal, s, m);
}

// The forward of both entries, every launch at the grid of the carved worst case.  live_dev[2] receives the
// evaluated coarse and fine sample counts as soon as the last scan has them; with live_host (the eager entry) they
// are also read back there, once.  That read-back is not left to the end: the host then enqueues the rest of the
// forward and returns to queue the backward while the GPU runs the last MLP, as it did when it read each count before
// sizing the launches after it.
int train_skip_forward(const nerfb200_train_samples_args* a, const TrainSkipWs& w, long long* live_dev,
                       int64_t* live_host, const DeviceInfo* d, cudaStream_t s) {
  SkipParams p = w.p;
  const bool fine = p.K > 0;
  const long long n = p.n;
  const int ray_blocks = grid_blocks(ceil_div(n, kSkipWarps), 1);
  const char* what = "train_samples_forward launches";
  auto counts = [&]() -> int {
    TRY(launch(what, train_skip_counts_kernel, 1, 32, 0, s, w.ofs[0] + n, fine ? w.ofs[1] + n : nullptr, live_dev));
    if (!live_host) return 0;
    long long live[2];
    CUDA_TRY(cudaMemcpyAsync(live, live_dev, sizeof(live), cudaMemcpyDeviceToHost, s), "train_samples readback");
    CUDA_TRY(cudaStreamSynchronize(s), "train_samples readback");
    live_host[0] = live[0];
    live_host[1] = live[1];
    return 0;
  };
  // coarse pass
  TRY(launch(what, skip_classify_kernel, ray_blocks, kSkipWarps * 32, 0, s, p));
  TRY(launch(what, skip_dir_bias_kernel, grid_blocks(n, 1), kDirW, 0, s, p, 0, fine ? 2 : 1));
  p.ofs = w.ofs[0];
  TRY(launch(what, cull_scan_kernel, 1, 1024, 0, s, p.cnt, p.ofs, n));
  if (!fine) TRY(counts());
  TRY(launch(what, skip_emit_kernel, ray_blocks, kSkipWarps * 32, 0, s, p, 0));
  TRY(train_skip_mlp(w, 0, d, s));
  TRY(launch(what, skip_coarse_stage_kernel, ray_blocks, kSkipWarps * 32, 0, s, p));
  if (fine) {
    p.ofs = w.ofs[1];
    TRY(launch(what, cull_scan_kernel, 1, 1024, 0, s, p.cnt, p.ofs, n));
    TRY(counts());
    TRY(launch(what, skip_emit_kernel, ray_blocks, kSkipWarps * 32, 0, s, p, 1));
    TRY(train_skip_mlp(w, 1, d, s));
    TRY(launch(what, skip_fine_stage_kernel, ray_blocks, kSkipWarps * 32, 0, s, p));
  }
  // losses.py / metrics.py on the results, one block in a fixed order
  if (a->target)
    TRY(launch(what, mse_psnr_kernel, 1, 1024, 0, s, p.rgb_coarse, fine ? p.rgb_fine : nullptr, a->target, n * 3,
               a->loss_out));
  uint32_t* const mask_out[2] = {a->mask_coarse, a->mask_fine};
  for (int ps = 0; ps < (fine ? 2 : 1); ++ps)
    if (mask_out[ps])
      CUDA_TRY(cudaMemcpyAsync(mask_out[ps], p.mask[ps], sizeof(uint32_t) * n * kSkipMaskWords,
                               cudaMemcpyDeviceToDevice, s), "train_samples mask copy");
  return 0;
}

// The backward of the networks with run[ps]: one plan launch for all of them from the device counts, then per network
// the sparse compositing backward, the optional per-row copies and the tail, every launch at the grid of the carved
// worst case.
int train_skip_backward(const nerfb200_train_samples_args* a, const TrainSkipWs& w, const bool run[2],
                        const float* loss_grad, const float* const* const params[2], float* const* const grads[2],
                        const DeviceInfo* d, cudaStream_t s) {
  const SkipParams& p = w.p;
  const char* what = "train_samples_backward launches";
  const int n_net = p.K > 0 ? 2 : 1;
  TrainLayout L[2];
  TrainSkipPlanArgs pa;
  std::memset(&pa, 0, sizeof(pa));
  for (int ps = 0; ps < n_net; ++ps) {
    if (!run[ps]) continue;
    make_train_layout(&L[ps], w.net_ws[ps], true, w.cap[ps], 1, 0, d->sm_count);
    pa.L[ps] = L[ps];
    pa.rows[ps] = w.ofs[ps] + p.n;
    for (int i = 0; i < kNumParams; ++i) {
      pa.params[ps][i] = params[ps][i];
      pa.grads[ps][i] = grads[ps][i];
    }
    pa.net[ps] = p.net[ps];
    pa.out[ps] = w.plan[ps];
  }
  pa.sm_count = d->sm_count;
  pa.status = d->status;
  TRY(launch(what, train_skip_plan_kernel, n_net, 32, 0, s, pa));
  for (int ps = 0; ps < n_net; ++ps) {
    if (!run[ps]) continue;
    const long long* rows = pa.rows[ps];
    const PassBufs& pb = L[ps].pass[0];
    TrainSkipBwdParams bp;
    bp.n_rays = p.n; bp.S = ps ? p.Sc + p.K : p.Sc;
    bp.n_rows = rows;
    bp.rays = p.rays; bp.z = ps ? p.zf : p.zc;
    bp.mask = p.mask[ps]; bp.ofs = w.ofs[ps];
    bp.sigma = pb.sigma; bp.rgb = pb.rgb;
    bp.noise = p.noise_std > 0.f ? p.noise[ps] : nullptr;
    bp.noise_std = p.noise_std; bp.white_back = p.white_back;
    bp.g_rgb = ps ? a->g_rgb_fine : a->g_rgb_coarse;
    bp.g_depth = ps ? a->g_depth_fine : a->g_depth_coarse;
    bp.g_opac = ps ? a->g_opacity_fine : a->g_opacity_coarse;
    bp.rgb_out = ps ? p.rgb_fine : p.rgb_coarse;
    bp.target = a->target; bp.loss_grad = loss_grad;
    bp.dsigma = pb.dsigma; bp.dprergb = pb.dprergb;
    bp.amax_bits = L[ps].amax;
    bp.status = d->status;
    TRY(launch(what, train_skip_bwd_kernel, grid_blocks(ceil_div(p.n, kSkipWarps), 1), kSkipWarps * 32, 0, s, bp));
    float* const ds_out = ps ? a->dsigma_fine : a->dsigma_coarse;
    float* const dp_out = ps ? a->dprergb_fine : a->dprergb_coarse;
    if (ds_out)
      TRY(launch(what, train_skip_copy_rows_kernel, grid_blocks(w.cap[ps], 256), 256, 0, s, pb.dsigma, ds_out, rows, 1));
    if (dp_out)
      TRY(launch(what, train_skip_copy_rows_kernel, grid_blocks(3 * w.cap[ps], 256), 256, 0, s, pb.dprergb, dp_out,
                 rows, 3));
    const float* const* const p2[2] = {params[ps], params[ps]};
    float* const* const g2[2] = {grads[ps], grads[ps]};
    const uint8_t* const net[2] = {p.net[ps], p.net[ps]};
    TRY(backward_tail(L[ps], p2, g2, net, nullptr, 0, d, s, what, w.plan[ps]));
  }
  return 0;
}

// The parameter / gradient tables of network ps (every tensor non-null).
int train_skip_tables_ok(const float* const* params, float* const* grads) {
  if (!params || !grads) return fail(NERFB200_EINVAL, "train_samples_backward: params / grads tables are NULL");
  for (int i = 0; i < kNumParams; ++i)
    if (!params[i] || !grads[i]) return fail(NERFB200_EINVAL, "train_samples_backward: NULL parameter / gradient tensor");
  return 0;
}

// ------------------------------------------------------------------ image metrics (kernels: metrics_kernels.cuh)

// The product of `k` extents, each >= 1, or -1 when one is < 1 or the product exceeds 2^48 elements.
long long image_elems(const int64_t* ext, int k) {
  long long n = 1;
  for (int a = 0; a < k; ++a) {
    if (ext[a] < 1 || ext[a] > (1LL << 48) / n) return -1;
    n *= ext[a];
  }
  return n;
}

// The SSIM workspace of n pixels: one double per tile.
size_t ssim_carve(long long n, void* base, double** partial) {
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  *partial = c.take<double>(ceil_div(n, kSsimTile));
  return c.off;
}

// The visualize_depth workspace of n pixels: the (min, max) pairs of the first pass, one per block.
int depth_minmax_blocks(long long n) { return grid_blocks(n, kDepthThreads * kDepthItemsPerThread, kDepthMinMaxCtas); }
size_t depth_viz_carve(long long n, void* base, float2** partial) {
  Carver c{static_cast<uint8_t*>(base), 0, 256};
  *partial = c.take<float2>(depth_minmax_blocks(n));
  return c.off;
}

}  // namespace

extern "C" {

int nerfb200_abi_version(void) { return NERFB200_ABI_VERSION; }
const char* nerfb200_last_error(void) { return g_err; }
size_t nerfb200_packed_bytes(void) { return kPackedBytes; }
int64_t nerfb200_launch_count(void) { return g_launches.load(); }

int nerfb200_sm_count(void) {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
  return n;
}

int nerfb200_pack_weights(const float* const params[24], void* packed, void* stream) {
  PackParams2 pp2;
  TRY(fill_pack_params(&pp2.net[0], params, packed));
  pp2.net[1] = pp2.net[0];
  return launch_pack(pp2, 1, stream);
}

int nerfb200_pack_weights_pair(const float* const params_a[24], void* packed_a, const float* const params_b[24],
                               void* packed_b, void* stream) {
  PackParams2 pp2;
  TRY(fill_pack_params(&pp2.net[0], params_a, packed_a));
  TRY(fill_pack_params(&pp2.net[1], params_b, packed_b));
  return launch_pack(pp2, 2, stream);
}

int nerfb200_render_rays(const nerfb200_render_args* a, void* stream) {
  TRY(check_render_shapes(a));
  if (a->n_rays == 0) return 0;
  if (a->n_rays > 0x7fffffff) return fail(NERFB200_EINVAL, "n_rays too large");
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  if (!a->status) TRY(check_sticky_status(d));
  RenderParams p;
  p.rays = a->rays;
  p.ray_stride = a->ray_stride;
  p.n_rays = static_cast<int>(a->n_rays);
  p.net_coarse = static_cast<const uint8_t*>(a->packed_coarse);
  p.net_fine = static_cast<const uint8_t*>(a->packed_fine);
  p.n_samples = a->n_samples;
  p.n_importance = a->n_importance;
  p.use_disp = a->use_disp;
  p.perturb = a->perturb;
  p.noise_std = a->noise_std;
  p.white_back = a->white_back;
  p.test_time = a->test_time;
  p.perturb_rand = a->perturb_rand;
  p.noise_coarse = a->noise_coarse;
  p.noise_fine = a->noise_fine;
  p.u_rand = a->u_rand;
  p.rgb_coarse = a->rgb_coarse;
  p.depth_coarse = a->depth_coarse;
  p.opacity_coarse = a->opacity_coarse;
  p.rgb_fine = a->rgb_fine;
  p.depth_fine = a->depth_fine;
  p.opacity_fine = a->opacity_fine;
  p.z_fine = a->z_fine;
  p.weights_coarse = a->weights_coarse;
  p.weights_fine = a->weights_fine;
  p.status = a->status ? a->status : d->status;
  p.z_coarse = a->z_coarse;
  p.rng_seed = a->rng_seed;               // with rng_in_kernel == 2 the bits of rng_seed_dev (the union)
  p.rng_in_kernel = a->rng_in_kernel;
  p.train = 0;
  p.target = nullptr; p.loss_part = nullptr; p.loss_out = nullptr; p.loss_counter = nullptr;
  std::memset(p.tr, 0, sizeof(p.tr));
  const bool save = a->train_workspace != nullptr;
  if (save && a->test_time) return fail(NERFB200_EINVAL, "train_workspace needs test_time = 0");
  if ((a->target != nullptr) != (a->loss_out != nullptr)) return fail(NERFB200_EINVAL, "target and loss_out go together");
  if (a->target && !save) return fail(NERFB200_EINVAL, "the fused loss epilogue needs train_workspace");
  if (save) {
    TrainLayout L;
    make_train_layout(&L, static_cast<uint8_t*>(a->train_workspace), false, a->n_rays, a->n_samples, a->n_importance,
                      d->sm_count);
    p.train = 1;
    p.tr[0] = L.pass[0];
    p.tr[1] = L.pass[1];
    if (!p.z_coarse) p.z_coarse = L.pass[0].z;
    else return fail(NERFB200_EINVAL, "z_coarse is owned by the workspace in training mode");
    if (a->n_importance > 0) {
      if (p.z_fine) return fail(NERFB200_EINVAL, "z_fine is owned by the workspace in training mode");
      p.z_fine = L.pass[1].z;
    }
    if (a->target) {
      p.target = a->target;
      p.loss_out = a->loss_out;
      p.loss_part = L.loss_part;
      p.loss_counter = L.loss_counter;
    }
  }
  const int n_groups = (p.n_rays + 1) / 2;     // two rays share the coarse tile
  int ctas = d->sm_count;
  if (a->max_ctas > 0 && a->max_ctas < ctas) ctas = a->max_ctas;
  if (env_switches().max_ctas > 0 && env_switches().max_ctas < ctas) ctas = env_switches().max_ctas;
  if (n_groups < ctas) ctas = n_groups;
  return launch("render_rays launch", save ? render_rays_kernel<true> : render_rays_kernel<false>, ctas, kRenderThreads,
                kSmemTotal, stream, p);
}

int nerfb200_render_rays_host(const nerfb200_render_args* h, void* stream_v) {
  TRY(check_render_shapes(h));
  if (h->n_rays == 0) return 0;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (h->train_workspace || h->target || h->z_coarse)
    return fail(NERFB200_EINVAL, "render_rays_host: train_workspace / target / z_coarse are device-only");
  {
    // Fast path: every host buffer is page-locked and mapped into the device's address space (cudaHostAlloc /
    // cudaHostRegister; torch's pin_memory()).  The kernel then reads the rays and writes the <= 40 B of results
    // per ray straight over PCIe - no staging copies, no copy-engine round trips (each small cudaMemcpyAsync
    // costs ~8 us of latency on the stream; the bytes that cross the bus are the same) - and the call is
    // "launch + synchronise".  Random inputs may be device tensors (drawn there by the caller) or mapped too.
    bool all_mapped = true;
    auto mapped = [&](const void* p, const void** dp) -> bool {
      *dp = nullptr;
      if (!p) return true;
      cudaPointerAttributes attr;
      if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) { (void)cudaGetLastError(); return false; }
      if ((attr.type == cudaMemoryTypeHost || attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged) &&
          attr.devicePointer != nullptr) {
        *dp = attr.devicePointer;
        return true;
      }
      return false;
    };
    nerfb200_render_args a = *h;
    const void* dp = nullptr;
#define NERFB200_MAP(field, type)                                          \
    all_mapped = all_mapped && mapped(h->field, &dp);                      \
    a.field = static_cast<type>(const_cast<void*>(dp));
    NERFB200_MAP(rays, const float*)
    NERFB200_MAP(perturb_rand, const float*)
    NERFB200_MAP(noise_coarse, const float*)
    NERFB200_MAP(u_rand, const float*)
    NERFB200_MAP(noise_fine, const float*)
    NERFB200_MAP(rgb_coarse, float*)
    NERFB200_MAP(depth_coarse, float*)
    NERFB200_MAP(opacity_coarse, float*)
    NERFB200_MAP(rgb_fine, float*)
    NERFB200_MAP(depth_fine, float*)
    NERFB200_MAP(opacity_fine, float*)
    NERFB200_MAP(z_fine, float*)
    NERFB200_MAP(weights_coarse, float*)
    NERFB200_MAP(weights_fine, float*)
#undef NERFB200_MAP
    if (all_mapped) {
      int dev0 = 0;
      CUDA_TRY(cudaGetDevice(&dev0), "cudaGetDevice");
      static int* host_status[64] = {nullptr};
      {
        std::lock_guard<std::mutex> lk(g_arena_mu);
        if (!host_status[dev0])
          CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&host_status[dev0]), 256, cudaHostAllocMapped | cudaHostAllocPortable),
                   "status cudaHostAlloc");
      }
      // one in-flight host call per device at a time shares the status word: serialise
      std::lock_guard<std::mutex> lk(g_host_call_mu);
      volatile int* hs = host_status[dev0];
      *hs = 0;
      int* dstatus = nullptr;
      CUDA_TRY(cudaHostGetDevicePointer(reinterpret_cast<void**>(&dstatus), host_status[dev0], 0), "status device pointer");
      a.status = dstatus;
      TRY(nerfb200_render_rays(&a, stream));
      CUDA_TRY(cudaStreamSynchronize(stream), "render_rays_host sync");
      const int hstatus = *hs;
      if (hstatus != 0) return fail(NERFB200_EDEVICE, "render kernel reported device status %d", hstatus);
      if (h->status) *h->status = 0;
      return 0;
    }
  }
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev), "cudaGetDevice");
  const size_t n = static_cast<size_t>(h->n_rays);
  const size_t Sc = h->n_samples, K = h->n_importance, Sf = Sc + K;
  const size_t fl = sizeof(float);
  // rays + 4 random inputs + 8 float outputs (+3 optional) + status, each rounded to 256 B
  size_t need = 16 * 256 + n * fl * (8 + Sc + Sc + K + Sf + 3 + 1 + 1 + 3 + 1 + 1 + Sf + Sc + Sf) + 256;
  Arena& ar = g_arena[dev];
  std::lock_guard<std::mutex> lk(g_arena_mu);
  TRY(ar.reserve(need));
  Carver arena{ar.base, 0, 256};
  nerfb200_render_args a = *h;
  a.ray_stride = 8;
  auto up = [&](const float* src, size_t count, size_t src_stride, size_t width) -> const float* {
    if (!src) return nullptr;
    if (src_stride == width) {
      // random inputs may already live on the device (drawn there by the caller): use them in place
      cudaPointerAttributes attr;
      if (cudaPointerGetAttributes(&attr, src) == cudaSuccess && attr.type == cudaMemoryTypeDevice) return src;
      (void)cudaGetLastError();
    }
    float* dst = arena.take<float>(count);
    if (src_stride == width) {
      cudaMemcpyAsync(dst, src, count * fl, cudaMemcpyHostToDevice, stream);
    } else {
      cudaMemcpy2DAsync(dst, width * fl, src, src_stride * fl, width * fl, count / width,
                        cudaMemcpyHostToDevice, stream);
    }
    return dst;
  };
  a.rays = up(h->rays, n * 8, static_cast<size_t>(h->ray_stride), 8);
  a.perturb_rand = up(h->perturb_rand, n * Sc, Sc, Sc);
  a.noise_coarse = up(h->noise_coarse, n * Sc, Sc, Sc);
  a.u_rand = up(h->u_rand, n * K, K, K);
  a.noise_fine = up(h->noise_fine, n * Sf, Sf, Sf);
  auto dn = [&](float* hostp, size_t count) -> float* {
    return hostp ? arena.take<float>(count) : nullptr;
  };
  a.rgb_coarse = dn(h->rgb_coarse, n * 3);
  a.depth_coarse = dn(h->depth_coarse, n);
  a.opacity_coarse = dn(h->opacity_coarse, n);
  a.rgb_fine = dn(h->rgb_fine, n * 3);
  a.depth_fine = dn(h->depth_fine, n);
  a.opacity_fine = dn(h->opacity_fine, n);
  a.z_fine = dn(h->z_fine, n * Sf);
  a.weights_coarse = dn(h->weights_coarse, n * Sc);
  a.weights_fine = dn(h->weights_fine, n * Sf);
  int* dstatus = arena.take<int>(1);
  CUDA_TRY(cudaMemsetAsync(dstatus, 0, sizeof(int), stream), "status memset");
  a.status = dstatus;
  TRY(nerfb200_render_rays(&a, stream));
  auto back = [&](float* hostp, const float* devp, size_t count) {
    if (hostp) cudaMemcpyAsync(hostp, devp, count * fl, cudaMemcpyDeviceToHost, stream);
  };
  back(h->rgb_coarse, a.rgb_coarse, n * 3);
  back(h->depth_coarse, a.depth_coarse, n);
  back(h->opacity_coarse, a.opacity_coarse, n);
  back(h->rgb_fine, a.rgb_fine, n * 3);
  back(h->depth_fine, a.depth_fine, n);
  back(h->opacity_fine, a.opacity_fine, n);
  back(h->z_fine, a.z_fine, n * Sf);
  back(h->weights_coarse, a.weights_coarse, n * Sc);
  back(h->weights_fine, a.weights_fine, n * Sf);
  int hstatus = 0;
  CUDA_TRY(cudaMemcpyAsync(&hstatus, dstatus, sizeof(int), cudaMemcpyDeviceToHost, stream), "status copy");
  CUDA_TRY(cudaStreamSynchronize(stream), "render_rays_host sync");
  if (hstatus != 0) return fail(NERFB200_EDEVICE, "render kernel reported device status %d", hstatus);
  if (h->status) *h->status = hstatus;
  return 0;
}

int nerfb200_nerf_forward(const float* x, int64_t n, int64_t x_stride, const void* packed,
                          int32_t sigma_only, float* out, void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "nerf_forward: n < 0");
  if (n == 0) return 0;
  if (!x || !packed || !out) return fail(NERFB200_EINVAL, "nerf_forward: NULL argument");
  if (x_stride < (sigma_only ? kEncXyz : kEncXyz + kEncDir))
    return fail(NERFB200_EINVAL, "nerf_forward: x_stride too small for the input width");
  if (!sigma_only && (reinterpret_cast<uintptr_t>(out) & 15))
    return fail(NERFB200_EINVAL, "nerf_forward: out must be 16-byte aligned");
  MlpParams p{};
  p.x = x; p.x_stride = x_stride; p.n = n;
  p.net = static_cast<const uint8_t*>(packed);
  p.sigma_only = sigma_only;
  p.out = out;
  return launch_mlp(p, nullptr, stream, "nerf_forward launch");
}

int nerfb200_query_sigma(const float* xyz, int64_t n, int64_t xyz_stride, const void* packed, float* sigma,
                         void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "query_sigma: n < 0");
  if (n == 0) return 0;
  if (!xyz || !packed || !sigma) return fail(NERFB200_EINVAL, "query_sigma: NULL argument");
  if (xyz_stride < 3) return fail(NERFB200_EINVAL, "query_sigma: xyz_stride < 3");
  MlpParams p{};
  p.raw_xyz = 1;
  p.x = xyz; p.x_stride = xyz_stride; p.n = n;
  p.net = static_cast<const uint8_t*>(packed);
  p.sigma_only = 1;
  p.out = sigma;
  return launch_mlp(p, nullptr, stream, "query_sigma launch");
}

int nerfb200_query_rgb_sigma(const float* xyz, int64_t n, int64_t xyz_stride, const void* packed, float* rgbsigma,
                             void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "query_rgb_sigma: n < 0");
  if (n == 0) return 0;
  if (!xyz || !packed || !rgbsigma) return fail(NERFB200_EINVAL, "query_rgb_sigma: NULL argument");
  if (xyz_stride < 3) return fail(NERFB200_EINVAL, "query_rgb_sigma: xyz_stride < 3");
  if (reinterpret_cast<uintptr_t>(rgbsigma) & 15) return fail(NERFB200_EINVAL, "query_rgb_sigma: out must be 16-byte aligned");
  MlpParams p{};
  p.raw_xyz = 1;
  p.x = xyz; p.x_stride = xyz_stride; p.n = n;
  p.net = static_cast<const uint8_t*>(packed);
  p.out = rgbsigma;
  return launch_mlp(p, nullptr, stream, "query_rgb_sigma launch");
}

// ---- training a direct NeRF.forward call (models/nerf.py:83-124)
size_t nerfb200_nerf_train_workspace_bytes(int64_t n) {
  if (n <= 0 || n > 0x7fffffffLL) return 0;
  TrainLayout L;
  make_train_layout(&L, nullptr, true, n, 1, 0, nerfb200_sm_count());
  return L.bytes;
}

int nerfb200_nerf_train_workspace_init(void* ws, size_t bytes, int64_t n, void* stream_v) {
  if (n < 0 || n > 0x7fffffffLL) return fail(NERFB200_EINVAL, "nerf_train_workspace_init: n out of range");
  if (n == 0) return 0;
  if (!ws) return fail(NERFB200_EINVAL, "nerf_train_workspace_init: workspace is NULL");
  if (reinterpret_cast<uintptr_t>(ws) & 1023) return fail(NERFB200_EINVAL, "nerf train workspace must be 1024-byte aligned");
  if (bytes < nerfb200_nerf_train_workspace_bytes(n)) return fail(NERFB200_EINVAL, "nerf train workspace too small for n");
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  TrainLayout L;
  make_train_layout(&L, static_cast<uint8_t*>(ws), true, n, 1, 0, d->sm_count);
  if (bytes < L.bytes) return fail(NERFB200_EINVAL, "nerf train workspace too small for n");
  return init_train_workspace(L, ws, d->sm_count, static_cast<cudaStream_t>(stream_v));
}

int nerfb200_nerf_forward_train(const float* x, int64_t n, int64_t x_stride, const void* packed, void* ws, float* out,
                                void* stream) {
  if (n < 0 || n > 0x7fffffffLL) return fail(NERFB200_EINVAL, "nerf_forward_train: n out of range");
  if (n == 0) return 0;
  if (!x || !packed || !ws || !out) return fail(NERFB200_EINVAL, "nerf_forward_train: NULL argument");
  if (x_stride < kEncXyz + kEncDir) return fail(NERFB200_EINVAL, "nerf_forward_train: x_stride < 90");
  if ((reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(packed) & 15))
    return fail(NERFB200_EINVAL, "nerf_forward_train: out / packed must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(ws) & 1023) return fail(NERFB200_EINVAL, "nerf train workspace must be 1024-byte aligned");
  MlpParams p{};
  p.x = x; p.x_stride = x_stride; p.n = n;
  p.net = static_cast<const uint8_t*>(packed);
  p.out = out;
  return launch_mlp(p, ws, stream, "nerf_forward_train launch");
}

int nerfb200_nerf_backward(const float* g_out, int64_t n, const void* packed, const float* const params[24], void* ws,
                           float* const grads[24], void* stream_v) {
  if (n < 0 || n > 0x7fffffffLL) return fail(NERFB200_EINVAL, "nerf_backward: n out of range");
  if (n == 0) return 0;
  if (!g_out || !packed || !params || !ws || !grads) return fail(NERFB200_EINVAL, "nerf_backward: NULL argument");
  for (int i = 0; i < kNumParams; ++i)
    if (!params[i] || !grads[i]) return fail(NERFB200_EINVAL, "nerf_backward: NULL parameter / gradient tensor");
  if (reinterpret_cast<uintptr_t>(g_out) & 15) return fail(NERFB200_EINVAL, "nerf_backward: g_out must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(ws) & 1023) return fail(NERFB200_EINVAL, "nerf train workspace must be 1024-byte aligned");
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  TrainLayout L;
  make_train_layout(&L, static_cast<uint8_t*>(ws), true, n, 1, 0, d->sm_count);
  const PassBufs& pb = L.pass[0];
  // 1. seed: upstream gradient -> per-sample d sigma / d rgb_pre (replaces the compositing backward)
  MlpSeedParams sd;
  sd.n = n; sd.n_pad = pb.n_pad;
  sd.g = g_out; sd.rgb = pb.rgb; sd.dsigma = pb.dsigma; sd.dprergb = pb.dprergb;
  sd.amax_bits = L.amax;
  sd.status = d->status;
  const char* what = "nerf_backward launches";
  TRY(launch(what, mlp_seed_kernel, static_cast<int>(ceil_div(pb.n_pad, 256)), 256, 0, stream, sd));
  const float* const* const p2[2] = {params, params};
  float* const* const g2[2] = {grads, grads};
  const uint8_t* const net[2] = {static_cast<const uint8_t*>(packed), static_cast<const uint8_t*>(packed)};
  return backward_tail(L, p2, g2, net, nullptr, 0, d, stream, what);
}

int nerfb200_mse_psnr(const float* rgb_coarse, const float* rgb_fine, const float* target, int64_t n_rays,
                      float* out4, void* stream) {
  if (n_rays <= 0) return fail(NERFB200_EINVAL, "mse_psnr: n_rays <= 0");
  if ((!rgb_coarse && !rgb_fine) || !target || !out4) return fail(NERFB200_EINVAL, "mse_psnr: NULL argument");
  return launch("mse_psnr launch", mse_psnr_kernel, 1, 1024, 0, stream, rgb_coarse, rgb_fine, target, n_rays * 3, out4);
}

int nerfb200_embed(const float* x, int64_t n, int32_t n_freqs, float* out, void* stream) {
  if (n < 0 || n_freqs < 0 || n_freqs > 16) return fail(NERFB200_EINVAL, "embed: bad n / n_freqs");
  if (n == 0) return 0;
  if (!x || !out) return fail(NERFB200_EINVAL, "embed: NULL argument");
  const long long total = n * (3 + 6 * n_freqs);
  return launch("embed launch", embed_kernel, grid_blocks(total, 256, 2 * kGridStrideCtas), 256, 0, stream, x, n,
                n_freqs, out);
}

int nerfb200_searchsorted(const float* a, const float* v, int64_t* out, int64_t nrow_a,
                          int64_t nrow_v, int32_t ncol_a, int32_t ncol_v, int32_t side_right,
                          void* stream) {
  if (nrow_a < 0 || nrow_v < 0 || ncol_a < 0 || ncol_v < 0)
    return fail(NERFB200_EINVAL, "searchsorted: negative size");
  // searchsorted.py:26-29: same number of rows, or one of them has a single row
  if (nrow_a != nrow_v && nrow_a != 1 && nrow_v != 1)
    return fail(NERFB200_EINVAL, "searchsorted: a and v need the same number of rows, or 1 row");
  const long long nrow = nrow_a > nrow_v ? nrow_a : nrow_v;
  const long long total = nrow * ncol_v;
  if (total == 0) return 0;
  if (!a && ncol_a > 0) return fail(NERFB200_EINVAL, "searchsorted: a is NULL");
  if (!v || !out) return fail(NERFB200_EINVAL, "searchsorted: NULL argument");
  return launch("searchsorted launch", searchsorted_kernel, grid_blocks(total, 256, 2 * kGridStrideCtas), 256, 0, stream,
                a, v, reinterpret_cast<long long*>(out), nrow_a, nrow_v, ncol_a, ncol_v, side_right);
}

int nerfb200_sample_pdf(const float* bins, const float* weights, const float* u, int64_t n_rays,
                        int32_t n_weights, int32_t n_u, float* out, void* stream) {
  if (n_rays < 0 || n_weights < 1 || n_u < 0 || n_weights > kPdfMaxWeights)
    return fail(NERFB200_EINVAL, "sample_pdf: bad sizes");
  if (n_rays == 0 || n_u == 0) return 0;
  if (!bins || !weights || !u || !out) return fail(NERFB200_EINVAL, "sample_pdf: NULL argument");
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));           // opts sample_pdf_kernel in to its shared memory
  const int wpb = kPdfWarps;
  const size_t sh = wpb * (n_weights + 1) * sizeof(float);
  return launch("sample_pdf launch", sample_pdf_kernel, grid_blocks(n_rays, wpb), wpb * 32, sh, stream, bins, weights,
                u, n_rays, n_weights, n_u, out);
}

int nerfb200_composite(const float* sigmas, const float* rgbs, const float* z_vals,
                       const float* dirs, const float* noise, float noise_std, int32_t white_back,
                       int64_t n_rays, int32_t S, float* weights, float* rgb, float* depth,
                       float* opacity, void* stream) {
  if (n_rays < 0) return fail(NERFB200_EINVAL, "composite: n_rays < 0");
  if (S <= 0 || (S % 32) != 0 || S > kMaxSf) return fail(NERFB200_EUNSUPPORTED, "composite: S must be a multiple of 32, <= 192");
  if (n_rays == 0) return 0;
  if (!sigmas || !z_vals || !dirs || !opacity) return fail(NERFB200_EINVAL, "composite: NULL argument");
  if (rgbs && (!rgb || !depth)) return fail(NERFB200_EINVAL, "composite: rgb/depth outputs NULL");
  const int wpb = 4;
  const size_t sh = wpb * 6 * S * sizeof(float);
  return launch("composite launch", composite_kernel, grid_blocks(n_rays, wpb), wpb * 32, sh, stream, sigmas, rgbs,
                z_vals, dirs, noise, noise_std, white_back, n_rays, S, weights, rgb, depth, opacity);
}

int nerfb200_generate_rays(int32_t H, int32_t W, float focal, const float c2w_host[12], float near, float far,
                           int32_t ndc, float* rays, void* stream) {
  if (H <= 0 || W <= 0 || !(focal > 0.f)) return fail(NERFB200_EINVAL, "generate_rays: bad H / W / focal");
  if (!c2w_host || !rays) return fail(NERFB200_EINVAL, "generate_rays: NULL argument");
  if (reinterpret_cast<uintptr_t>(rays) & 15) return fail(NERFB200_EINVAL, "generate_rays: rays must be 16-byte aligned");
  RayGenParams p;
  p.H = H; p.W = W; p.focal = focal; p.near = near; p.far = far; p.ndc = ndc; p.rays = rays;
  for (int i = 0; i < 12; ++i) p.c2w[i] = c2w_host[i];
  return launch("generate_rays launch", generate_rays_kernel, grid_blocks(static_cast<long long>(H) * W, 256), 256, 0,
                stream, p);
}

int nerfb200_view_batch(const uint8_t* images, int64_t V, int32_t H, int32_t W, int32_t C, const float* c2w,
                        float focal, float near, float far, int32_t ndc, const int64_t* ids, int64_t n, float* rays,
                        float* rgbs, void* stream) {
  if (V < 1 || H < 1 || W < 1 || n < 0) return fail(NERFB200_EINVAL, "view_batch: bad V / H / W / n");
  if (C != 3 && C != 4) return fail(NERFB200_EINVAL, "view_batch: C must be 3 (RGB) or 4 (RGBA)");
  if (!(focal > 0.f)) return fail(NERFB200_EINVAL, "view_batch: focal must be > 0");
  // V * H * W * C bytes must be addressable with 64-bit ids
  if (V > INT64_MAX / (static_cast<int64_t>(H) * W * C)) return fail(NERFB200_EINVAL, "view_batch: V * H * W * C overflows");
  if (n == 0) return 0;
  if (!images || !c2w || !ids || !rays || !rgbs) return fail(NERFB200_EINVAL, "view_batch: NULL argument");
  if ((reinterpret_cast<uintptr_t>(rays) | reinterpret_cast<uintptr_t>(c2w)) & 15)
    return fail(NERFB200_EINVAL, "view_batch: rays and c2w must be 16-byte aligned");
  ViewBatchParams p;
  p.images = images; p.V = V; p.H = H; p.W = W; p.C = C;
  p.c2w = c2w; p.focal = focal; p.near = near; p.far = far; p.ndc = ndc;
  p.ids = reinterpret_cast<const long long*>(ids); p.n = n; p.rays = rays; p.rgbs = rgbs;
  return launch("view_batch launch", view_batch_kernel, grid_blocks(n, 256), 256, 0, stream, p);
}

int nerfb200_to_uint8(const float* src, int64_t n, uint8_t* dst, void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "to_uint8: n < 0");
  if (n == 0) return 0;
  if (!src || !dst) return fail(NERFB200_EINVAL, "to_uint8: NULL argument");
  return launch("to_uint8 launch", to_uint8_kernel, grid_blocks(n, 256), 256, 0, stream, src, n, dst);
}

size_t nerfb200_train_workspace_bytes(int64_t n_rays, int32_t n_samples, int32_t n_importance) {
  if (n_rays <= 0 || n_samples <= 0 || n_importance < 0) return 0;
  TrainLayout L;
  make_train_layout(&L, nullptr, false, n_rays, n_samples, n_importance, nerfb200_sm_count());
  return L.bytes;
}

int nerfb200_train_workspace_init(void* workspace, size_t bytes, int64_t n_rays, int32_t n_samples,
                                  int32_t n_importance, void* stream_v) {
  if (!workspace || n_rays <= 0) return fail(NERFB200_EINVAL, "train_workspace_init: bad argument");
  if (reinterpret_cast<uintptr_t>(workspace) & 1023) return fail(NERFB200_EINVAL, "train workspace must be 1024-byte aligned");
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  TrainLayout L;
  make_train_layout(&L, static_cast<uint8_t*>(workspace), false, n_rays, n_samples, n_importance, d->sm_count);
  if (bytes < L.bytes) return fail(NERFB200_EINVAL, "train workspace too small");
  return init_train_workspace(L, workspace, d->sm_count, static_cast<cudaStream_t>(stream_v));
}

int nerfb200_render_backward(const nerfb200_backward_args* b, void* stream_v) {
  if (!b || !b->render) return fail(NERFB200_EINVAL, "render_backward: NULL argument");
  const nerfb200_render_args* a = b->render;
  TRY(check_render_shapes(a));
  if (a->n_rays == 0) return 0;
  if (!a->train_workspace || a->test_time) return fail(NERFB200_EINVAL, "render_backward needs the forward's train_workspace, test_time = 0");
  const bool fine = a->n_importance > 0;
  if (!b->params_coarse || !b->grads_coarse || (fine && (!b->params_fine || !b->grads_fine)))
    return fail(NERFB200_EINVAL, "render_backward: params / grads tables are NULL");
  for (int i = 0; i < kNumParams; ++i)
    if (!b->params_coarse[i] || !b->grads_coarse[i] || (fine && (!b->params_fine[i] || !b->grads_fine[i])))
      return fail(NERFB200_EINVAL, "render_backward: NULL parameter / gradient tensor");
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  TrainLayout L;
  make_train_layout(&L, static_cast<uint8_t*>(a->train_workspace), false, a->n_rays, a->n_samples, a->n_importance,
                    d->sm_count);
  const float* const* const params[2] = {b->params_coarse, b->params_fine};
  float* const* const grads[2] = {b->grads_coarse, b->grads_fine};
  const uint8_t* const net[2] = {static_cast<const uint8_t*>(a->packed_coarse), static_cast<const uint8_t*>(a->packed_fine)};
  const float* g_rgb[2] = {b->g_rgb_coarse, b->g_rgb_fine};
  const float* g_depth[2] = {b->g_depth_coarse, b->g_depth_fine};
  const float* g_opac[2] = {b->g_opacity_coarse, b->g_opacity_fine};
  const float* rgb_out[2] = {a->rgb_coarse, a->rgb_fine};
  const float* noise[2] = {a->noise_coarse, a->noise_fine};
  const char* what = "render_backward launches";

  // 1. compositing backward -> per-sample d sigma / d rgb_pre
  for (int ps = 0; ps < L.n_pass; ++ps) {
    CompBwdParams cp;
    cp.n_rays = L.n_rays; cp.S = L.pass[ps].S; cp.n_pad = L.pass[ps].n_pad;
    cp.z = L.pass[ps].z; cp.sigma = L.pass[ps].sigma; cp.rgb = L.pass[ps].rgb;
    cp.rays = a->rays; cp.ray_stride = a->ray_stride;
    cp.noise = a->noise_std > 0.f ? noise[ps] : nullptr;
    cp.noise_std = a->noise_std; cp.white_back = a->white_back;
    cp.g_rgb = g_rgb[ps]; cp.g_depth = g_depth[ps]; cp.g_opac = g_opac[ps];
    cp.rgb_out = rgb_out[ps]; cp.target = b->target; cp.loss_grad = b->loss_grad;
    cp.dsigma = L.pass[ps].dsigma; cp.dprergb = L.pass[ps].dprergb;
    cp.amax_bits = L.amax + 2 * ps;
    cp.status = d->status;
    TRY(launch(what, composite_bwd_kernel, (L.n_rays + 3) / 4, 128, 0, stream, cp));
  }
  return backward_tail(L, params, grads, net, a->rays, a->ray_stride, d, stream, what);
}

int nerfb200_adam_step(int32_t n_tensors, float* const* params, const float* const* grads, float* const* exp_avg,
                       float* const* exp_avg_sq, const int64_t* numel, float lr, float beta1, float beta2, float eps,
                       float weight_decay, int64_t step, void* stream) {
  if (n_tensors < 0 || n_tensors > kAdamMaxTensors) return fail(NERFB200_EINVAL, "adam_step: at most 64 tensors per call");
  if (n_tensors == 0) return 0;
  if (!params || !grads || !exp_avg || !exp_avg_sq || !numel || step < 1)
    return fail(NERFB200_EINVAL, "adam_step: NULL argument / step < 1");
  AdamParams a;
  int blocks = 0;
  TRY(fill_adam_table(a, n_tensors, params, grads, exp_avg, exp_avg_sq, numel, nullptr, beta1, beta2, eps, weight_decay,
                      "adam_step", &blocks));
  // in double, rounded once: 1 - b2^t in fp32 cancels at small t (~50 ulps of the update at t = 2..3)
  a.step_size = static_cast<float>(static_cast<double>(lr) / (1.0 - std::pow(static_cast<double>(beta1), static_cast<double>(step))));
  a.bias2_sqrt = static_cast<float>(std::sqrt(1.0 - std::pow(static_cast<double>(beta2), static_cast<double>(step))));
  if (blocks == 0) return 0;
  return launch("adam_step launch", adam_kernel, blocks, 256, 0, stream, a);
}

int nerfb200_adam_step_dev(int32_t n_tensors, float* const* params, const float* const* grads, float* const* exp_avg,
                           float* const* exp_avg_sq, const int64_t* numel, const float* lr_dev,
                           const float* const* steps, float beta1, float beta2, float eps, float weight_decay,
                           void* stream) {
  if (n_tensors < 0 || n_tensors > kAdamMaxTensors) return fail(NERFB200_EINVAL, "adam_step_dev: at most 64 tensors per call");
  if (n_tensors == 0) return 0;
  if (!params || !grads || !exp_avg || !exp_avg_sq || !numel || !lr_dev || !steps)
    return fail(NERFB200_EINVAL, "adam_step_dev: NULL argument");
  AdamDevParams d;
  AdamParams& a = d.a;
  int blocks = 0;
  TRY(fill_adam_table(a, n_tensors, params, grads, exp_avg, exp_avg_sq, numel, steps, beta1, beta2, eps, weight_decay,
                      "adam_step_dev", &blocks));
  for (int i = 0; i < n_tensors; ++i) d.step[i] = steps[i];
  a.step_size = a.bias2_sqrt = 0.f;
  d.lr = lr_dev;
  if (blocks == 0) return 0;
  return launch("adam_step_dev launch", adam_dev_kernel, blocks, 256, 0, stream, d);
}

int nerfb200_check_status(void) {
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  return check_sticky_status(d);
}

// ---- coloured mesh extraction (extract_color_mesh.py; kernels: mesh_kernels.cuh)
size_t nerfb200_sigma_grid_workspace_bytes(int64_t chunk) {
  if (chunk <= 0) return 0;
  Carver c{nullptr, 0, 256};
  c.take<float>(static_cast<size_t>(chunk) * 3);     // the positions of one chunk
  return c.off;
}

int nerfb200_grid_positions(int64_t N, const double ranges_host[6], int64_t start, int64_t count, float* xyz,
                            void* stream) {
  if (N < 2 || start < 0 || count < 0 || start + count > N * N * N)
    return fail(NERFB200_EINVAL, "grid_positions: bad N / start / count");
  if (count == 0) return 0;
  if (!ranges_host || !xyz) return fail(NERFB200_EINVAL, "grid_positions: NULL argument");
  GridParams p;
  for (int a = 0; a < 3; ++a) { p.lo[a] = ranges_host[2 * a]; p.hi[a] = ranges_host[2 * a + 1]; }
  p.N = N; p.start = start; p.count = count; p.xyz = xyz;
  return launch("grid_positions launch", mesh_grid_positions_kernel, grid_blocks(count, 256), 256, 0, stream, p);
}

int nerfb200_sigma_grid(const void* packed, int64_t N, const double ranges_host[6], int64_t chunk, void* ws,
                        size_t bytes, float* sigma, void* stream) {
  if (N < 2 || chunk <= 0) return fail(NERFB200_EINVAL, "sigma_grid: N < 2 or chunk <= 0");
  if (!packed || !ranges_host || !ws || !sigma) return fail(NERFB200_EINVAL, "sigma_grid: NULL argument");
  if (bytes < nerfb200_sigma_grid_workspace_bytes(chunk))
    return fail(NERFB200_EINVAL, "sigma_grid: workspace smaller than nerfb200_sigma_grid_workspace_bytes(chunk)");
  return grid_chunks(N, ranges_host, chunk, ws, stream, [&](float* xyz, long long s, long long n) {
    TRY(nerfb200_query_sigma(xyz, n, 3, packed, sigma + s, stream));
    return launch("sigma_grid relu launch", mesh_relu_kernel, grid_blocks(n, 256), 256, 0, stream, sigma + s, n);
  });
}

int nerfb200_rgb_sigma_grid(const void* packed, int64_t N, const double ranges_host[6], int64_t chunk, void* ws,
                            size_t bytes, float* rgbsigma, void* stream) {
  if (N < 2 || N > kVolMaxN || chunk <= 0) return fail(NERFB200_EINVAL, "rgb_sigma_grid: N not in [2, 1625] or chunk <= 0");
  if (!packed || !ranges_host || !ws || !rgbsigma) return fail(NERFB200_EINVAL, "rgb_sigma_grid: NULL argument");
  if (reinterpret_cast<uintptr_t>(rgbsigma) & 15) return fail(NERFB200_EINVAL, "rgb_sigma_grid: out must be 16-byte aligned");
  if (bytes < nerfb200_sigma_grid_workspace_bytes(chunk))
    return fail(NERFB200_EINVAL, "rgb_sigma_grid: workspace smaller than nerfb200_sigma_grid_workspace_bytes(chunk)");
  return grid_chunks(N, ranges_host, chunk, ws, stream, [&](float* xyz, long long s, long long n) {
    return nerfb200_query_rgb_sigma(xyz, n, 3, packed, rgbsigma + s * 4, stream);
  });
}

size_t nerfb200_volume_workspace_bytes(int64_t N) {
  if (N < 2 || N > kVolMaxN) return 0;
  VolumeParams p;
  CubScratch sc;
  return volume_carve(N, nullptr, &p, &sc);
}

int nerfb200_volume_count(const float* rgbsigma, int64_t N, double xmin, double xmax, void* ws, size_t bytes,
                          int64_t* count_host, void* stream) {
  VolumeParams p;
  CubScratch sc;
  TRY(volume_prepare(rgbsigma, N, xmin, xmax, ws, bytes, &p, &sc, "volume_count"));
  if (!count_host) return fail(NERFB200_EINVAL, "volume_count: count_host is NULL");
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long tiles = ceil_div(p.P, kVolTile);
  CUDA_TRY(cudaMemsetAsync(p.tcnt + tiles, 0, sizeof(unsigned long long), s), "volume_count memset");
  TRY(launch("volume_count launch", volume_count_kernel, grid_blocks(tiles * kVolThreads, 256), kVolThreads, 0, s, p));
  size_t tb = sc.temp_bytes;
  TRY(cub_launch(cub::DeviceScan::ExclusiveSum(sc.temp, tb, p.tcnt, p.tofs, static_cast<int>(tiles + 1), s),
                 "volume scan"));
  unsigned long long h = 0;
  CUDA_TRY(cudaMemcpyAsync(&h, p.tofs + tiles, sizeof(h), cudaMemcpyDeviceToHost, s), "volume_count readback");
  CUDA_TRY(cudaStreamSynchronize(s), "volume_count readback");
  *count_host = static_cast<int64_t>(h);
  return 0;
}

int nerfb200_volume_emit(const float* rgbsigma, int64_t N, double xmin, double xmax, void* ws, size_t bytes,
                         uint32_t* packed_out, void* stream) {
  VolumeParams p;
  CubScratch sc;
  TRY(volume_prepare(rgbsigma, N, xmin, xmax, ws, bytes, &p, &sc, "volume_emit"));
  if (!packed_out) return fail(NERFB200_EINVAL, "volume_emit: out is NULL");
  if (reinterpret_cast<uintptr_t>(packed_out) & 7) return fail(NERFB200_EINVAL, "volume_emit: out must be 8-byte aligned");
  p.out = reinterpret_cast<uint2*>(packed_out);
  const long long tiles = ceil_div(p.P, kVolTile);
  return launch("volume_emit launch", volume_emit_kernel, grid_blocks(tiles * kVolThreads, 256), kVolThreads, 0, stream,
                p);
}

size_t nerfb200_mc_workspace_bytes(int64_t n0, int64_t n1, int64_t n2) {
  if (n0 < 2 || n1 < 2 || n2 < 2 || n0 * n1 * n2 > kMcMaxPoints) return 0;
  McParams p;
  CubScratch sc;
  return mc_carve(n0 * n1 * n2, (n0 - 1) * (n1 - 1) * (n2 - 1), nullptr, &p, &sc);
}

int nerfb200_mc_count(const float* sigma, int64_t n0, int64_t n1, int64_t n2, double threshold, void* ws, size_t bytes,
                      int64_t counts_host[2], void* stream) {
  McParams p;
  CubScratch sc;
  TRY(mc_prepare(sigma, n0, n1, n2, threshold, ws, bytes, &p, &sc, "mc_count"));
  if (!counts_host) return fail(NERFB200_EINVAL, "mc_count: counts_host is NULL");
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long P = n0 * n1 * n2, C = (n0 - 1) * (n1 - 1) * (n2 - 1);
  CUDA_TRY(cudaMemsetAsync(p.vcnt + P, 0, 1, s), "mc_count memset");
  CUDA_TRY(cudaMemsetAsync(p.ccnt + C, 0, 1, s), "mc_count memset");
  TRY(launch("mc_classify launch", mc_classify_kernel, grid_blocks(P, 256), 256, 0, s, p));
  size_t tb = sc.temp_bytes;
  TRY(cub_launch(cub::DeviceScan::ExclusiveSum(sc.temp, tb, U8It(p.vcnt, U8ToInt()), p.vofs, static_cast<int>(P + 1), s),
                 "mc vertex scan"));
  tb = sc.temp_bytes;
  TRY(cub_launch(cub::DeviceScan::ExclusiveSum(sc.temp, tb, U8It(p.ccnt, U8ToInt()), p.cofs, static_cast<int>(C + 1), s),
                 "mc triangle scan"));
  return read_two_counts(p.vofs + P, p.cofs + C, counts_host, s, "mc_count readback");
}

int nerfb200_mc_emit(const float* sigma, int64_t n0, int64_t n1, int64_t n2, double threshold, void* ws, size_t bytes,
                     double* vertices, int32_t* triangles, void* stream) {
  McParams p;
  CubScratch sc;
  TRY(mc_prepare(sigma, n0, n1, n2, threshold, ws, bytes, &p, &sc, "mc_emit"));
  p.vertices = vertices;
  p.triangles = triangles;
  const long long P = n0 * n1 * n2, C = (n0 - 1) * (n1 - 1) * (n2 - 1);
  if (vertices) TRY(launch("mc_emit_vertices launch", mc_emit_vertices_kernel, grid_blocks(P, 256), 256, 0, stream, p));
  if (triangles)
    TRY(launch("mc_emit_triangles launch", mc_emit_triangles_kernel, grid_blocks(C, 256), 256, 0, stream, p));
  return 0;
}

int nerfb200_mesh_to_world(const double* vertices, int64_t n, int64_t N, const double ranges_host[6], float* out,
                           void* stream) {
  if (n < 0 || N < 1) return fail(NERFB200_EINVAL, "mesh_to_world: bad n / N");
  if (n == 0) return 0;
  if (!vertices || !ranges_host || !out) return fail(NERFB200_EINVAL, "mesh_to_world: NULL argument");
  ToWorldParams p;
  p.v = vertices; p.n = n; p.N = static_cast<double>(N); p.out = out;
  // column 0 takes y_range, column 1 x_range (extract_color_mesh.py:150-151)
  const int src[3] = {1, 0, 2};
  for (int c = 0; c < 3; ++c) {
    const double lo = ranges_host[2 * src[c]], hi = ranges_host[2 * src[c] + 1];
    p.scale[c] = static_cast<float>(hi - lo);
    p.offset[c] = static_cast<float>(lo);
  }
  return launch("mesh_to_world launch", mesh_to_world_kernel, grid_blocks(n, 256), 256, 0, stream, p);
}

size_t nerfb200_mesh_cluster_workspace_bytes(int64_t n_vertices, int64_t n_triangles) {
  if (n_vertices < 0 || n_triangles <= 0 || n_triangles > 0x7fffffffLL / 3 || n_vertices > 0x7fffffffLL) return 0;
  ClusterParams p;
  CubScratch sc;
  return cluster_carve(n_vertices, n_triangles, nullptr, &p, &sc);
}

int nerfb200_mesh_cluster_count(const int32_t* triangles, int64_t n_tris, int64_t n_verts, void* ws, size_t bytes,
                                int64_t counts_host[2], void* stream) {
  ClusterParams p;
  CubScratch sc;
  TRY(cluster_prepare(triangles, n_tris, n_verts, ws, bytes, &p, &sc, "mesh_cluster_count"));
  if (!counts_host) return fail(NERFB200_EINVAL, "mesh_cluster_count: counts_host is NULL");
  if (n_tris == 0) { counts_host[0] = counts_host[1] = 0; return 0; }
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long E = 3 * n_tris;
  const int bits = bits_for(n_verts);
  TRY(launch("cluster edges launch", cluster_edges_kernel, grid_blocks(n_tris, 256), 256, 0, s, p));
  TRY(launch("cluster edges launch", cluster_pack_keys_kernel, grid_blocks(E, 256), 256, 0, s, p.keys, E, bits));
  cub::DoubleBuffer<unsigned long long> kb(p.keys, static_cast<unsigned long long*>(sc.keys_alt));
  cub::DoubleBuffer<int> vb(p.vals, static_cast<int*>(sc.vals_alt));
  size_t tb = sc.temp_bytes;
  TRY(cub_launch(cub::DeviceRadixSort::SortPairs(sc.temp, tb, kb, vb, static_cast<int>(E), 0, 2 * bits, s),
                 "cluster edge sort"));
  p.keys = kb.Current();
  p.vals = vb.Current();
  CUDA_TRY(cudaMemsetAsync(p.best, 0, sizeof(unsigned long long), s), "cluster memset");
  CUDA_TRY(cudaMemsetAsync(p.vflag, 0, n_verts + 1, s), "cluster memset");
  CUDA_TRY(cudaMemsetAsync(p.tflag + n_tris, 0, 1, s), "cluster memset");
  const char* uf = "cluster union-find launch";
  TRY(launch(uf, cluster_union_kernel, grid_blocks(E, 256), 256, 0, s, p));
  TRY(launch(uf, cluster_label_kernel, grid_blocks(n_tris, 256), 256, 0, s, p));
  TRY(launch(uf, cluster_best_kernel, grid_blocks(n_tris, 256), 256, 0, s, p));
  TRY(launch(uf, cluster_flag_kernel, grid_blocks(n_tris, 256), 256, 0, s, p));
  tb = sc.temp_bytes;
  TRY(cub_launch(cub::DeviceScan::ExclusiveSum(sc.temp, tb, U8It(p.tflag, U8ToInt()), p.tofs, static_cast<int>(n_tris + 1),
                                               s), "cluster triangle scan"));
  tb = sc.temp_bytes;
  TRY(cub_launch(cub::DeviceScan::ExclusiveSum(sc.temp, tb, U8It(p.vflag, U8ToInt()), p.vofs,
                                               static_cast<int>(n_verts + 1), s), "cluster vertex scan"));
  return read_two_counts(p.vofs + n_verts, p.tofs + n_tris, counts_host, s, "mesh_cluster_count readback");
}

int nerfb200_mesh_cluster_emit(const float* vertices, const int32_t* triangles, int64_t n_tris, int64_t n_verts, void* ws,
                               size_t bytes, float* vertices_out, int32_t* triangles_out, void* stream) {
  ClusterParams p;
  CubScratch sc;
  TRY(cluster_prepare(triangles, n_tris, n_verts, ws, bytes, &p, &sc, "mesh_cluster_emit"));
  if (n_tris == 0) return 0;
  if (!vertices || !vertices_out || !triangles_out) return fail(NERFB200_EINVAL, "mesh_cluster_emit: NULL argument");
  p.vin = vertices; p.vout = vertices_out; p.tout = triangles_out;
  const long long n = n_tris > n_verts ? n_tris : n_verts;
  return launch("mesh_cluster_emit launch", cluster_emit_kernel, grid_blocks(n, 256), 256, 0, stream, p);
}

int nerfb200_remap_bilinear(const uint8_t* image, int32_t H, int32_t W, const float* xy, int64_t n, uint8_t* out,
                            void* stream) {
  if (H <= 0 || W <= 0 || n < 0) return fail(NERFB200_EINVAL, "remap_bilinear: bad H / W / n");
  if (n == 0) return 0;
  if (!image || !xy || !out) return fail(NERFB200_EINVAL, "remap_bilinear: NULL argument");
  return launch("remap_bilinear launch", remap_bilinear_kernel, grid_blocks(n, 256), 256, 0, stream, image, H, W, xy, n,
                out);
}

int nerfb200_color_project(const float* vertices, int64_t n, const double w2c_host[12], const float origin_host[3],
                           float focal, int32_t W, int32_t H, const uint8_t* image, float near, uint8_t* colors,
                           double* depth, float* rays, void* stream) {
  if (n < 0 || H <= 0 || W <= 0) return fail(NERFB200_EINVAL, "color_project: bad n / H / W");
  if (n == 0) return 0;
  if (!vertices || !w2c_host || !origin_host || !image || !colors || !depth || !rays)
    return fail(NERFB200_EINVAL, "color_project: NULL argument");
  ColorProjectParams p;
  p.vertices = vertices; p.n = n;
  for (int i = 0; i < 12; ++i) p.w2c[i] = w2c_host[i];
  for (int i = 0; i < 3; ++i) p.origin[i] = origin_host[i];
  p.focal = focal; p.W = W; p.H = H; p.image = image; p.near = near;
  p.colors = colors; p.depth = depth; p.rays = rays;
  return launch("color_project launch", color_project_kernel, grid_blocks(n, 256), 256, 0, stream, p);
}

int nerfb200_color_accumulate(const uint8_t* colors, const double* depth, const float* opacity, int64_t n,
                              float occ_threshold, double* sum4, void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "color_accumulate: n < 0");
  if (n == 0) return 0;
  if (!colors || !depth || !opacity || !sum4) return fail(NERFB200_EINVAL, "color_accumulate: NULL argument");
  return launch("color_accumulate launch", color_accumulate_kernel, grid_blocks(n, 256), 256, 0, stream, colors, depth,
                opacity, n, occ_threshold, sum4);
}

int nerfb200_color_finalize(const double* sum4, int64_t n, uint8_t* colors, void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "color_finalize: n < 0");
  if (n == 0) return 0;
  if (!sum4 || !colors) return fail(NERFB200_EINVAL, "color_finalize: NULL argument");
  return launch("color_finalize launch", color_finalize_kernel, grid_blocks(n, 256), 256, 0, stream, sum4, n, colors);
}

size_t nerfb200_vertex_normals_workspace_bytes(int64_t n_verts, int64_t n_tris) {
  if (!normals_size_ok(n_verts, n_tris)) return 0;
  NormalsParams p;
  CubScratch sc;
  return normals_carve(n_verts, n_tris, nullptr, &p, &sc);
}

int nerfb200_vertex_normals(const float* vertices, int64_t n_verts, const int32_t* triangles, int64_t n_tris, void* ws,
                            size_t bytes, double* normals, void* stream) {
  if (!normals_size_ok(n_verts, n_tris)) return fail(NERFB200_EINVAL, "vertex_normals: bad mesh size");
  if (n_verts == 0) {
    if (n_tris == 0) return 0;
    return fail(NERFB200_EINVAL, "vertex_normals: a triangle index is outside [0, n_verts) (n_verts = 0)");
  }
  if ((n_verts > 0 && (!vertices || !normals)) || (n_tris > 0 && !triangles) || !ws)
    return fail(NERFB200_EINVAL, "vertex_normals: NULL argument");
  NormalsParams p;
  CubScratch sc;
  if (bytes < normals_carve(n_verts, n_tris, ws, &p, &sc))
    return fail(NERFB200_EINVAL, "vertex_normals: workspace smaller than nerfb200_vertex_normals_workspace_bytes");
  p.vertices = vertices; p.tris = triangles; p.n_verts = n_verts; p.n_tris = n_tris;
  p.normals = normals;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemsetAsync(p.bad, 0, sizeof(int), s), "vertex_normals memset");
  if (n_tris > 0) {
    TRY(launch("vertex_normals triangle launch", normals_triangle_kernel, grid_blocks(n_tris, 256), 256, 0, s, p));
    cub::DoubleBuffer<int> kb(p.keys, static_cast<int*>(sc.keys_alt));
    cub::DoubleBuffer<int> vb(p.vals, static_cast<int*>(sc.vals_alt));
    size_t tb = sc.temp_bytes;
    TRY(cub_launch(cub::DeviceRadixSort::SortPairs(sc.temp, tb, kb, vb, static_cast<int>(3 * n_tris), 0,
                                                   bits_for(n_verts + 1), s), "vertex_normals corner sort"));
    p.keys = kb.Current();
    p.vals = vb.Current();
  }
  if (n_verts > 0)
    TRY(launch("vertex_normals vertex launch", normals_vertex_kernel, grid_blocks(n_verts, 256), 256, 0, s, p));
  int bad = 0;
  CUDA_TRY(cudaMemcpyAsync(&bad, p.bad, sizeof(int), cudaMemcpyDeviceToHost, s), "vertex_normals readback");
  CUDA_TRY(cudaStreamSynchronize(s), "vertex_normals readback");
  if (bad) return fail(NERFB200_EINVAL, "vertex_normals: a triangle index is outside [0, n_verts)");
  return 0;
}

int nerfb200_normal_rays(const float* vertices, const double* normals, int64_t n, float near, float far, float near_t,
                         float* rays, void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "normal_rays: n < 0");
  if (n == 0) return 0;
  if (!vertices || !normals || !rays) return fail(NERFB200_EINVAL, "normal_rays: NULL argument");
  return launch("normal_rays launch", normal_rays_kernel, grid_blocks(n, 256), 256, 0, stream, vertices, normals, n, near,
                far, near_t, rays);
}

// ---- empty-space skipping (kernels: occupancy_kernels.cuh)
size_t nerfb200_occupancy_workspace_bytes(int64_t grid_N) {
  int64_t N;
  int32_t levels;
  grid_n(grid_N, &N, &levels);
  if (N < 2 || N > kVolMaxN || levels > kMaxLevels) return 0;
  uint8_t* buf[2];
  return occupancy_carve((N - 1) * (N - 1) * (N - 1), nullptr, buf);
}

int nerfb200_occupancy_pack(const float* sigma, int64_t grid_N, double sigma_threshold, int32_t dilate, void* ws,
                            size_t bytes, uint32_t* bits, void* stream) {
  int64_t N;
  int32_t levels;
  grid_n(grid_N, &N, &levels);
  if (N < 2 || N > kVolMaxN) return fail(NERFB200_EINVAL, "occupancy_pack: N must be in [2, 1625]");
  if (levels < 1 || levels > kMaxLevels) return fail(NERFB200_EINVAL, "occupancy_pack: levels must be in [1, 8]");
  if (dilate < 0) return fail(NERFB200_EINVAL, "occupancy_pack: dilate < 0");
  if (sigma_threshold != sigma_threshold) return fail(NERFB200_EINVAL, "occupancy_pack: sigma_threshold is NaN");
  if (!sigma || !ws || !bits) return fail(NERFB200_EINVAL, "occupancy_pack: NULL argument");
  if (bytes < nerfb200_occupancy_workspace_bytes(N))
    return fail(NERFB200_EINVAL, "occupancy_pack: workspace smaller than nerfb200_occupancy_workspace_bytes");
  const long long M = N - 1, C = M * M * M, words = ceil_div(C, 32);
  uint8_t* buf[2];
  occupancy_carve(C, ws, buf);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  for (int k = 0; k < levels; ++k) {
    const long long ia = k ? inner_lo(M) : 0, ib = k ? std::max(inner_hi(M), ia) : 0;
    TRY(launch("occupancy cells launch", occ_cells_kernel, grid_blocks(C, 256), 256, 0, s, sigma + k * N * N * N, N,
               sigma_threshold, ia, ib, buf[0]));
    TRY(occupancy_finish(buf[0], buf[1], M, ia, ib, dilate, bits + k * words, s, "occupancy dilate launch",
                         "occupancy pack launch"));
  }
  return 0;
}

int nerfb200_occupancy_popcount(const uint32_t* bits, int64_t grid_N, int64_t* count, void* stream) {
  int64_t N;
  int32_t levels;
  grid_n(grid_N, &N, &levels);
  if (N < 2 || N > kVolMaxN) return fail(NERFB200_EINVAL, "occupancy_popcount: N must be in [2, 1625]");
  if (levels < 1 || levels > kMaxLevels) return fail(NERFB200_EINVAL, "occupancy_popcount: levels must be in [1, 8]");
  if (!bits || !count) return fail(NERFB200_EINVAL, "occupancy_popcount: NULL argument");
  const long long C = (N - 1) * (N - 1) * (N - 1), words = (C + 31) / 32 * levels;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemsetAsync(count, 0, sizeof(*count), s), "occupancy_popcount memset");
  return launch("occupancy_popcount launch", occ_popcount_kernel, grid_blocks(words, 256), 256, 0, s, bits, words,
                reinterpret_cast<unsigned long long*>(count));
}

size_t nerfb200_cull_workspace_bytes(int64_t n_rays) {
  CullParams p;
  return n_rays < 0 ? 0 : cull_carve(n_rays, nullptr, &p);
}

int nerfb200_cull_count(const float* rays, int64_t n_rays, const uint32_t* bits, int64_t grid_N,
                        const double ranges_host[6], void* ws, size_t bytes, uint8_t* flag, int64_t* n_live_host,
                        void* stream) {
  int64_t N;
  int32_t levels;
  grid_n(grid_N, &N, &levels);
  CullParams p;
  TRY(cull_prepare(rays, n_rays, ws, bytes, &p, "cull_count"));
  if (N < 2 || N > kVolMaxN) return fail(NERFB200_EINVAL, "cull_count: N must be in [2, 1625]");
  if (!n_live_host || !ranges_host) return fail(NERFB200_EINVAL, "cull_count: NULL argument");
  TRY(skip_grid(bits, N, levels, ranges_host, &p.grid, "cull_count"));
  *n_live_host = 0;
  if (n_rays == 0) return 0;
  if (!bits || !flag) return fail(NERFB200_EINVAL, "cull_count: NULL argument");
  p.flag = flag;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long tiles = ceil_div(n_rays, kCullTile);
  TRY(launch("cull classify launch", cull_classify_kernel, grid_blocks(tiles, 1), kCullTile, 0, s, p));
  TRY(launch("cull scan launch", cull_scan_kernel, 1, 1024, 0, s, p.tcnt, p.tofs, tiles));
  long long h = 0;
  CUDA_TRY(cudaMemcpyAsync(&h, p.tofs + tiles, sizeof(h), cudaMemcpyDeviceToHost, s), "cull_count readback");
  CUDA_TRY(cudaStreamSynchronize(s), "cull_count readback");
  *n_live_host = h;
  return 0;
}

int nerfb200_cull_emit(const float* rays, int64_t n_rays, const uint8_t* flag, void* ws, size_t bytes,
                       int64_t* live_idx, float* live_rays, void* stream) {
  CullParams p;
  TRY(cull_prepare(rays, n_rays, ws, bytes, &p, "cull_emit"));
  if (n_rays == 0) return 0;
  if (!flag || !live_idx || !live_rays) return fail(NERFB200_EINVAL, "cull_emit: NULL argument");
  if (reinterpret_cast<uintptr_t>(live_rays) & 15) return fail(NERFB200_EINVAL, "cull_emit: live_rays must be 16-byte aligned");
  p.flag = const_cast<uint8_t*>(flag);
  p.live_idx = reinterpret_cast<long long*>(live_idx);
  p.live_rays = live_rays;
  return launch("cull emit launch", cull_emit_kernel, grid_blocks(ceil_div(n_rays, kCullTile), 1), kCullTile, 0, stream,
                p);
}

int nerfb200_scatter_results(const float* const src_host[6], float* const dst_host[6], const int64_t* live_idx,
                             int64_t n_live, int64_t n_rays, int32_t white_back, void* stream) {
  if (n_rays < 0 || n_live < 0 || n_live > n_rays) return fail(NERFB200_EINVAL, "scatter_results: bad n_live / n_rays");
  if (!src_host || !dst_host) return fail(NERFB200_EINVAL, "scatter_results: NULL argument");
  if (n_rays == 0) return 0;
  if (n_live > 0 && !live_idx) return fail(NERFB200_EINVAL, "scatter_results: live_idx is NULL");
  ScatterParams p;
  bool any = false;
  for (int k = 0; k < 6; ++k) {
    if (n_live > 0 && (src_host[k] == nullptr) != (dst_host[k] == nullptr))
      return fail(NERFB200_EINVAL, "scatter_results: a result is NULL on one side only");
    p.src[k] = src_host[k]; p.dst[k] = dst_host[k];
    any |= dst_host[k] != nullptr;
  }
  if (!any) return fail(NERFB200_EINVAL, "scatter_results: no result to write");
  p.live_idx = reinterpret_cast<const long long*>(live_idx);
  p.n_live = n_live; p.n = n_rays; p.bg = white_back ? 1.f : 0.f;
  return launch("scatter_results launch", scatter_results_kernel, grid_blocks(n_rays, 256), 256, 0, stream, p);
}

// ---- per-sample skipping (kernels: sample_skip_kernels.cuh)
size_t nerfb200_samples_workspace_bytes(int64_t n_rays, int32_t n_samples, int32_t n_importance) {
  SkipParams p;
  return samples_shape_ok(n_rays, n_samples, n_importance) ? samples_carve(n_rays, n_samples, n_importance, nullptr, &p)
                                                           : 0;
}

int nerfb200_render_samples(const nerfb200_samples_args* a, void* ws, size_t bytes, int64_t* live_samples_host,
                            void* stream) {
  if (!a || !live_samples_host) return fail(NERFB200_EINVAL, "render_samples: NULL argument");
  if (!samples_shape_ok(a->n_rays, a->n_samples, a->n_importance))
    return fail(NERFB200_EUNSUPPORTED, "render_samples: needs N_samples in {32, 64, 128}, N_importance a multiple of "
                "32, N_samples + N_importance <= 192 and 0 <= n_rays <= 2^22");
  if (!(a->early_stop >= 0.f && a->early_stop <= 1.f))
    return fail(NERFB200_EINVAL, "render_samples: early_stop must be in [0, 1]");
  const bool early_stop = a->early_stop > 0.f;
  if (early_stop && a->n_importance > 0)
    return fail(NERFB200_EUNSUPPORTED, "render_samples: early_stop needs N_importance = 0: with importance samples "
                "at most about 5 %% of the evaluated fine samples lie behind the cut (DESIGN.md §10f), and cutting the "
                "coarse pass would change z_vals_fine");
  if (early_stop && (a->perturb > 0.f || a->noise_std > 0.f))
    return fail(NERFB200_EINVAL, "render_samples: early_stop needs perturb = 0 and noise_std = 0");
  SkipParams p{};
  TRY(skip_grid(a->bits, a->N, a->levels ? a->levels : 1, a->ranges, &p.grid, "render_samples"));
  live_samples_host[0] = live_samples_host[1] = 0;
  if (a->n_rays == 0) return 0;
  const bool fine = a->n_importance > 0, coarse_rgb = a->test_time == 0;
  if (!a->rays || !a->packed_coarse || !a->bits || !a->opacity_coarse || !ws)
    return fail(NERFB200_EINVAL, "render_samples: NULL argument");
  if (coarse_rgb && (!a->rgb_coarse || !a->depth_coarse))
    return fail(NERFB200_EINVAL, "render_samples: rgb_coarse / depth_coarse is NULL with test_time=0");
  if (fine && (!a->packed_fine || !a->rgb_fine || !a->depth_fine || !a->opacity_fine))
    return fail(NERFB200_EINVAL, "render_samples: packed_fine / fine outputs are NULL with N_importance>0");
  TRY(skip_randoms(a, "render_samples", &p));
  if (a->rng_ray_offset < 0 || a->rng_ray_offset > (1LL << 32) - a->n_rays)
    return fail(NERFB200_EINVAL, "render_samples: rng_ray_offset must be >= 0 with rng_ray_offset + n_rays <= 2^32");
  if ((reinterpret_cast<uintptr_t>(a->rays) | reinterpret_cast<uintptr_t>(a->packed_coarse) |
       reinterpret_cast<uintptr_t>(a->packed_fine) | reinterpret_cast<uintptr_t>(a->samples_coarse) |
       reinterpret_cast<uintptr_t>(a->samples_fine)) & 15)
    return fail(NERFB200_EINVAL, "render_samples: rays, packed images and samples must be 16-byte aligned");
  if (bytes < samples_carve(a->n_rays, a->n_samples, a->n_importance, ws, &p))
    return fail(NERFB200_EINVAL, "render_samples: workspace smaller than nerfb200_samples_workspace_bytes");
  if (!(a->perturb > 0.f)) p.zc = nullptr;     // unperturbed: every kernel takes z_base's depths
  p.ray0 = static_cast<uint32_t>(a->rng_ray_offset);
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  p.rays = a->rays; p.n = static_cast<int>(a->n_rays); p.live_flag = a->live_flag;
  p.Sc = a->n_samples; p.K = a->n_importance; p.use_disp = a->use_disp; p.white_back = a->white_back;
  p.test_time = a->test_time;
  p.net[0] = static_cast<const uint8_t*>(a->packed_coarse);
  p.net[1] = static_cast<const uint8_t*>(a->packed_fine);
  if (a->mask_coarse) p.mask[0] = a->mask_coarse;
  if (a->mask_fine) p.mask[1] = a->mask_fine;
  p.rgb_coarse = a->rgb_coarse; p.depth_coarse = a->depth_coarse; p.opacity_coarse = a->opacity_coarse;
  p.rgb_fine = a->rgb_fine; p.depth_fine = a->depth_fine; p.opacity_fine = a->opacity_fine;
  p.z_fine = a->z_fine; p.weights_coarse = a->weights_coarse; p.weights_fine = a->weights_fine;
  p.samples[0] = a->samples_coarse; p.samples[1] = a->samples_fine;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int ray_blocks = grid_blocks(ceil_div(p.n, kSkipWarps), 1);
  // coarse pass
  TRY(launch("render_samples classify launch", skip_classify_kernel, ray_blocks, kSkipWarps * 32, 0, s, p));
  long long n_c = 0, n_f = 0;
  if (early_stop && p.Sc > 32) {
    TRY(samples_early_stop(p, a->early_stop, a->cut_coarse, ray_blocks, s, &n_c));
    live_samples_host[0] = n_c;
    return 0;
  }
  if (early_stop && a->cut_coarse)     // one word: nothing can be dropped, no ray is cut
    CUDA_TRY(cudaMemsetAsync(a->cut_coarse, 0xff, sizeof(int32_t) * p.n, s), "render_samples cut_coarse");
  TRY(samples_scan(p, s, &n_c));
  bool have_bias = false;
  if (n_c > 0) {
    TRY(launch("render_samples emit launch", skip_emit_kernel, ray_blocks, kSkipWarps * 32, 0, s, p, 0));
    if (coarse_rgb) {
      TRY(launch("render_samples dir_bias launch", skip_dir_bias_kernel, grid_blocks(p.n, 1), kDirW, 0, s, p, 0,
                 fine ? 2 : 1));
      have_bias = true;
    }
    TRY(samples_mlp(p, 0, n_c, !coarse_rgb, s));
  }
  TRY(launch("render_samples coarse stage launch", skip_coarse_stage_kernel, ray_blocks, kSkipWarps * 32, 0, s, p));
  live_samples_host[0] = n_c;
  if (!fine) return 0;
  // fine pass
  TRY(samples_scan(p, s, &n_f));
  if (n_f > 0) {
    TRY(launch("render_samples emit launch", skip_emit_kernel, ray_blocks, kSkipWarps * 32, 0, s, p, 1));
    if (!have_bias)
      TRY(launch("render_samples dir_bias launch", skip_dir_bias_kernel, grid_blocks(p.n, 1), kDirW, 0, s, p, 1, 2));
    TRY(samples_mlp(p, 1, n_f, false, s));
  }
  TRY(launch("render_samples fine stage launch", skip_fine_stage_kernel, ray_blocks, kSkipWarps * 32, 0, s, p));
  live_samples_host[1] = n_f;
  return 0;
}

// ---- training with empty samples skipped (kernels: sample_skip_kernels.cuh, train_skip_kernels.cuh)
size_t nerfb200_train_samples_workspace_bytes(int64_t n_rays, int32_t n_samples, int32_t n_importance) {
  if (!samples_shape_ok(n_rays, n_samples, n_importance) || n_rays < 1) return 0;
  TrainSkipWs w;
  return train_skip_carve(n_rays, n_samples, n_importance, nullptr, nerfb200_sm_count(), &w);
}

int nerfb200_train_samples_forward(const nerfb200_train_samples_args* a, void* ws, size_t bytes,
                                   int64_t* live_samples_host, void* stream) {
  if (!live_samples_host) return fail(NERFB200_EINVAL, "train_samples_forward: NULL argument");
  TrainSkipWs w;
  TRY(train_skip_setup(a, ws, bytes, nerfb200_sm_count(), &w, "train_samples_forward"));
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  TRY(check_sticky_status(d));
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  live_samples_host[0] = live_samples_host[1] = 0;
  return train_skip_forward(a, w, w.live, live_samples_host, d, s);
}

int nerfb200_train_samples_forward_dev(const nerfb200_train_samples_args* a, void* ws, size_t bytes,
                                       int64_t* live_samples_dev, void* stream) {
  if (!live_samples_dev) return fail(NERFB200_EINVAL, "train_samples_forward_dev: NULL argument");
  TrainSkipWs w;
  TRY(train_skip_setup(a, ws, bytes, nerfb200_sm_count(), &w, "train_samples_forward_dev"));
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  TRY(check_sticky_status(d));
  return train_skip_forward(a, w, reinterpret_cast<long long*>(live_samples_dev), nullptr, d,
                            static_cast<cudaStream_t>(stream));
}

int nerfb200_train_samples_backward(const nerfb200_train_samples_args* a, void* ws, size_t bytes,
                                    const int64_t* live_samples_host, const float* loss_grad,
                                    const float* const params_coarse[24], const float* const params_fine[24],
                                    float* const grads_coarse[24], float* const grads_fine[24], void* stream) {
  if (!live_samples_host) return fail(NERFB200_EINVAL, "train_samples_backward: NULL argument");
  TrainSkipWs w;
  TRY(train_skip_setup(a, ws, bytes, nerfb200_sm_count(), &w, "train_samples_backward"));
  const int n_net = w.p.K > 0 ? 2 : 1;
  const float* const* const params[2] = {params_coarse, params_fine};
  float* const* const grads[2] = {grads_coarse, grads_fine};
  for (int ps = 0; ps < n_net; ++ps) {
    if (live_samples_host[ps] < 0 || live_samples_host[ps] > w.cap[ps])
      return fail(NERFB200_EINVAL, "train_samples_backward: live sample count out of range");
    if (live_samples_host[ps] > 0) TRY(train_skip_tables_ok(params[ps], grads[ps]));
  }
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  const bool run[2] = {live_samples_host[0] > 0, n_net > 1 && live_samples_host[1] > 0};
  if (!run[0] && !run[1]) return 0;
  return train_skip_backward(a, w, run, loss_grad, params, grads, d, static_cast<cudaStream_t>(stream));
}

int nerfb200_train_samples_backward_dev(const nerfb200_train_samples_args* a, void* ws, size_t bytes,
                                        const float* loss_grad, const float* const params_coarse[24],
                                        const float* const params_fine[24], float* const grads_coarse[24],
                                        float* const grads_fine[24], void* stream) {
  TrainSkipWs w;
  TRY(train_skip_setup(a, ws, bytes, nerfb200_sm_count(), &w, "train_samples_backward_dev"));
  const int n_net = w.p.K > 0 ? 2 : 1;
  const float* const* const params[2] = {params_coarse, params_fine};
  float* const* const grads[2] = {grads_coarse, grads_fine};
  for (int ps = 0; ps < n_net; ++ps) TRY(train_skip_tables_ok(params[ps], grads[ps]));
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  const bool run[2] = {true, n_net > 1};
  return train_skip_backward(a, w, run, loss_grad, params, grads, d, static_cast<cudaStream_t>(stream));
}

// ---- image metrics (kernels: metrics_kernels.cuh)
size_t nerfb200_ssim_workspace_bytes(int64_t b, int64_t c, int64_t h, int64_t w) {
  const int64_t ext[4] = {b, c, h, w};
  const long long n = image_elems(ext, 4);
  double* partial;
  return n < 0 ? 0 : ssim_carve(n, nullptr, &partial);
}

int nerfb200_ssim(const float* pred, const int64_t pred_strides_host[4], const float* gt,
                  const int64_t gt_strides_host[4], int64_t b, int64_t c, int64_t h, int64_t w, int32_t reduction,
                  void* ws, size_t bytes, float* out, void* stream) {
  const int64_t ext[4] = {b, c, h, w};
  const long long n = image_elems(ext, 4);
  if (n < 0) return fail(NERFB200_EINVAL, "ssim: b, c, h and w must be >= 1 (and at most 2^48 pixels)");
  if (reduction != NERFB200_SSIM_MEAN && reduction != NERFB200_SSIM_SUM && reduction != NERFB200_SSIM_NONE)
    return fail(NERFB200_EINVAL, "ssim: reduction must be NERFB200_SSIM_MEAN, _SUM or _NONE");
  if (!pred || !gt || !pred_strides_host || !gt_strides_host || !out) return fail(NERFB200_EINVAL, "ssim: NULL argument");
  SsimParams p;
  for (int a = 0; a < 4; ++a) {
    if (pred_strides_host[a] < 0 || gt_strides_host[a] < 0) return fail(NERFB200_EINVAL, "ssim: negative stride");
    p.xs[a] = pred_strides_host[a];
    p.ys[a] = gt_strides_host[a];
  }
  p.x = pred; p.y = gt; p.C = c; p.H = h; p.W = w; p.n = n;
  // kornia's window: exp(-x^2 / (2 sigma^2)) at x = -1, 0, 1 with sigma = 1.5, normalised to sum 1
  const double e = std::exp(-1.0 / (2.0 * 1.5 * 1.5));
  p.g[0] = e / (1.0 + 2.0 * e);
  p.g[1] = 1.0 / (1.0 + 2.0 * e);
  p.map = nullptr; p.partial = nullptr;
  const long long tiles = ceil_div(n, kSsimTile);
  if (reduction == NERFB200_SSIM_NONE) {
    p.map = out;
    return launch("ssim launch", ssim_kernel, grid_blocks(tiles, 1), kSsimTile, 0, stream, p);
  }
  if (!ws) return fail(NERFB200_EINVAL, "ssim: NULL workspace");
  if (bytes < ssim_carve(n, ws, &p.partial))
    return fail(NERFB200_EINVAL, "ssim: workspace smaller than nerfb200_ssim_workspace_bytes");
  TRY(launch("ssim launch", ssim_kernel, grid_blocks(tiles, 1), kSsimTile, 0, stream, p));
  const double denom = reduction == NERFB200_SSIM_MEAN ? static_cast<double>(n) : 1.0;
  return launch("ssim finish launch", ssim_finish_kernel, 1, kSsimFinishThreads, 0, stream, p.partial, tiles, denom,
                out);
}

size_t nerfb200_visualize_depth_workspace_bytes(int64_t h, int64_t w) {
  const int64_t ext[2] = {h, w};
  const long long n = image_elems(ext, 2);
  float2* partial;
  return n < 0 ? 0 : depth_viz_carve(n, nullptr, &partial);
}

int nerfb200_visualize_depth(const float* depth, int64_t h, int64_t w, int64_t stride_h, int64_t stride_w, void* ws,
                             size_t bytes, float* out, void* stream) {
  const int64_t ext[2] = {h, w};
  const long long n = image_elems(ext, 2);
  if (n < 0) return fail(NERFB200_EINVAL, "visualize_depth: h and w must be >= 1 (and at most 2^48 pixels)");
  if (stride_h < 0 || stride_w < 0) return fail(NERFB200_EINVAL, "visualize_depth: negative stride");
  if (!depth || !ws || !out) return fail(NERFB200_EINVAL, "visualize_depth: NULL argument");
  DepthVizParams p;
  if (bytes < depth_viz_carve(n, ws, &p.partial))
    return fail(NERFB200_EINVAL, "visualize_depth: workspace smaller than nerfb200_visualize_depth_workspace_bytes");
  p.depth = depth; p.H = h; p.W = w; p.sh = stride_h; p.sw = stride_w; p.out = out;
  p.n_partial = depth_minmax_blocks(n);
  TRY(launch("visualize_depth min/max launch", depth_minmax_kernel, p.n_partial, kDepthThreads, 0, stream, p));
  return launch("visualize_depth colour launch", depth_color_kernel, grid_blocks(n, kDepthThreads), kDepthThreads, 0,
                stream, p);
}

// ---- the density grid (kernels: density_kernels.cuh)
size_t nerfb200_density_workspace_bytes(int64_t grid_N, int64_t chunk) {
  int64_t N;
  int32_t levels;
  grid_n(grid_N, &N, &levels);
  if (N < 2 || N > kVolMaxN || levels > kMaxLevels || chunk < 1) return 0;
  const long long C = (N - 1) * (N - 1) * (N - 1);
  float *xyz, *sigma;
  uint8_t* buf[2];
  return density_carve(C, chunk < C ? chunk : C, nullptr, &xyz, &sigma, buf);
}

int nerfb200_density_points(int64_t grid_N, const double ranges_host[6], const int64_t* key_dev, int64_t start,
                            int64_t count, float* xyz, void* stream) {
  int64_t N;
  int32_t levels;
  grid_n(grid_N, &N, &levels);
  TRY(levels_ok(N, levels, ranges_host, "density_points"));
  long long total = 0;
  for (int k = 0; k < levels; ++k) {
    DensityBox b;
    TRY(density_box(N, levels, ranges_host, k, &b, "density_points"));
    total += level_cells(b);
  }
  if (start < 0 || count < 0 || start > total || count > total - start)
    return fail(NERFB200_EINVAL, "density_points: cells [start, start + count) outside the grid");
  if (count == 0) return 0;
  if (!key_dev || !xyz) return fail(NERFB200_EINVAL, "density_points: NULL argument");
  // the points of each level the range meets, level 0's cells first, then each further level's non-inner cells
  long long base = 0;
  for (int k = 0; k < levels; ++k) {
    DensityBox b;
    TRY(density_box(N, levels, ranges_host, k, &b, "density_points"));
    const long long Ck = level_cells(b), lo = std::max<long long>(start, base),
                    hi = std::min<long long>(start + count, base + Ck);
    if (lo < hi)
      TRY(launch("density_points launch", density_points_kernel, grid_blocks(hi - lo, 256), 256, 0, stream, b,
                 reinterpret_cast<const long long*>(key_dev), lo - base, hi - lo, xyz + (lo - start) * 3));
    base += Ck;
  }
  return 0;
}

int nerfb200_density_update(const void* packed, int64_t grid_N, const double ranges_host[6], double sigma_threshold,
                            float decay, int32_t dilate, int64_t chunk, int64_t* key_dev, float* density,
                            uint32_t* bits, void* ws, size_t bytes, void* stream) {
  int64_t N;
  int32_t levels;
  grid_n(grid_N, &N, &levels);
  TRY(levels_ok(N, levels, ranges_host, "density_update"));
  if (sigma_threshold != sigma_threshold) return fail(NERFB200_EINVAL, "density_update: sigma_threshold is NaN");
  if (!(decay >= 0.f && decay <= 1.f)) return fail(NERFB200_EINVAL, "density_update: decay must be in [0, 1]");
  if (dilate < 0) return fail(NERFB200_EINVAL, "density_update: dilate < 0");
  if (chunk < 1) return fail(NERFB200_EINVAL, "density_update: chunk < 1");
  if (!packed || !key_dev || !density || !bits || !ws) return fail(NERFB200_EINVAL, "density_update: NULL argument");
  if (bytes < nerfb200_density_workspace_bytes(N, chunk))
    return fail(NERFB200_EINVAL, "density_update: workspace smaller than nerfb200_density_workspace_bytes");
  const long long M = N - 1, C = M * M * M, ch = chunk < C ? chunk : C, words = ceil_div(C, 32);
  float *xyz, *sigma;
  uint8_t* buf[2];
  density_carve(C, ch, ws, &xyz, &sigma, buf);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  long long* key = reinterpret_cast<long long*>(key_dev);
  for (int k = 0; k < levels; ++k) {
    DensityBox b;
    TRY(density_box(N, levels, ranges_host, k, &b, "density_update"));
    const long long Ck = level_cells(b);
    // no launch below writes the inner cells' bytes: 0 for the dilation
    if (b.ib > b.ia) CUDA_TRY(cudaMemsetAsync(buf[0], 0, C, s), "density_update memset");
    for (long long c0 = 0; c0 < Ck; c0 += ch) {
      const long long n = Ck - c0 < ch ? Ck - c0 : ch;
      TRY(launch("density_points launch", density_points_kernel, grid_blocks(n, 256), 256, 0, s, b,
                 reinterpret_cast<const long long*>(key_dev), c0, n, xyz));
      TRY(nerfb200_query_sigma(xyz, n, 3, packed, sigma, stream));
      TRY(launch("density decay launch", density_decay_kernel, grid_blocks(n, 256), 256, 0, s, sigma, b, c0, n, decay,
                 sigma_threshold, density + k * C, buf[0], k + 1 == levels && c0 + n == Ck ? key : nullptr));
    }
    // the dilation and packing of nerfb200_occupancy_pack
    TRY(occupancy_finish(buf[0], buf[1], M, b.ia, b.ib, dilate, bits + k * words, s, "density dilate launch",
                         "density pack launch"));
  }
  return 0;
}

// ---- grids through an occupancy grid (kernels: masked_grid_kernels.cuh)
size_t nerfb200_masked_grid_workspace_bytes(int64_t chunk) {
  if (chunk < 1) return 0;
  MaskedGridParams p;
  CubScratch sc;
  return masked_grid_carve(chunk, nullptr, &p, &sc);
}

int nerfb200_sigma_grid_masked(const void* packed, int64_t N, const double ranges_host[6], const uint32_t* bits,
                               int64_t occ_N, const double occ_ranges_host[6], int64_t chunk, void* ws, size_t bytes,
                               float* sigma_out, int64_t* evaluated_host, void* stream) {
  if (N < 2) return fail(NERFB200_EINVAL, "sigma_grid_masked: N < 2");
  return masked_grid(packed, N, ranges_host, bits, occ_N, occ_ranges_host, chunk, ws, bytes, sigma_out,
                     evaluated_host, 1, stream, "sigma_grid_masked");
}

int nerfb200_rgb_sigma_grid_masked(const void* packed, int64_t N, const double ranges_host[6], const uint32_t* bits,
                                   int64_t occ_N, const double occ_ranges_host[6], int64_t chunk, void* ws,
                                   size_t bytes, float* rgbsigma_out, int64_t* evaluated_host, void* stream) {
  if (N < 2 || N > kVolMaxN) return fail(NERFB200_EINVAL, "rgb_sigma_grid_masked: N not in [2, 1625]");
  if (reinterpret_cast<uintptr_t>(rgbsigma_out) & 15)
    return fail(NERFB200_EINVAL, "rgb_sigma_grid_masked: out must be 16-byte aligned");
  return masked_grid(packed, N, ranges_host, bits, occ_N, occ_ranges_host, chunk, ws, bytes, rgbsigma_out,
                     evaluated_host, 4, stream, "rgb_sigma_grid_masked");
}

// ---- sparse marching cubes (include/nerf_pl_b200_sparse_mc.h, kernels: sparse_mc_kernels.cuh)
size_t nerfb200_sparse_mc_plan_workspace_bytes(int64_t N) {
  if (N < 2 || N > kSmcMaxN) return 0;
  SparseMcParams p{};
  CubScratch sc;
  return smc_plan_carve(N, nullptr, &p, &sc);
}

int nerfb200_sparse_mc_plan(int64_t N, const double ranges_host[6], const uint32_t* bits, int64_t occ_N,
                            const double occ_ranges_host[6], void* plan_ws, size_t plan_bytes, int64_t bricks_host[2],
                            void* stream) {
  const char* who = "sparse_mc_plan";
  SparseMcParams p{};
  TRY(smc_grids(N, ranges_host, bits, occ_N, occ_ranges_host, &p, who));
  if (!plan_ws || !bricks_host) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  CubScratch sc;
  if (plan_bytes < smc_plan_carve(N, plan_ws, &p, &sc))
    return fail(NERFB200_EINVAL, "%s: plan workspace smaller than nerfb200_sparse_mc_plan_workspace_bytes(N)", who);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long B = p.nb * p.nb * p.nb;
  TRY(launch("sparse_mc candidate launch", smc_candidate_kernel, grid_blocks(B, 256), 256, 0, s, p));
  TRY(smc_select(p, sc, p.cand, p.nsel + 0, s, "sparse_mc candidate select"));
  TRY(launch("sparse_mc classify launch", smc_classify_kernel, grid_blocks(B, 1), kBrickPoints, 0, s, p));
  TRY(smc_select(p, sc, p.active, p.nsel + 1, s, "sparse_mc active select"));
  TRY(launch("sparse_mc map launch", smc_map_kernel, grid_blocks(B, 256), 256, 0, s, p));
  TRY(launch("sparse_mc march flag launch", smc_march_flag_kernel, grid_blocks(B, 256), 256, 0, s, p));
  TRY(smc_select(p, sc, p.march, p.nsel + 2, s, "sparse_mc march select"));
  int h[2] = {0, 0};
  CUDA_TRY(cudaMemcpyAsync(h, p.nsel + 1, sizeof(h), cudaMemcpyDeviceToHost, s), "sparse_mc plan readback");
  CUDA_TRY(cudaStreamSynchronize(s), "sparse_mc plan readback");
  bricks_host[0] = h[0];
  bricks_host[1] = h[1];
  return 0;
}

size_t nerfb200_sparse_mc_workspace_bytes(int64_t N, int64_t active, int64_t march) {
  if (!smc_counts_ok(N, active, march)) return 0;
  SparseMcParams p{};
  unsigned long long *rcnt, *vt;
  CubScratch sc;
  return smc_carve(active, march, nullptr, &p, &rcnt, &vt, &sc);
}

int nerfb200_sparse_mc_count(const void* packed, int64_t N, const double ranges_host[6], const uint32_t* bits,
                             int64_t occ_N, const double occ_ranges_host[6], double threshold, void* plan_ws,
                             size_t plan_bytes, const int64_t bricks_host[2], void* ws, size_t bytes,
                             int64_t counts_host[2], void* stream) {
  const char* who = "sparse_mc_count";
  SparseMcParams p{};
  TRY(smc_grids(N, ranges_host, bits, occ_N, occ_ranges_host, &p, who));
  if (!packed || !plan_ws || !bricks_host || !ws || !counts_host) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  const long long A = bricks_host[0], Mb = bricks_host[1];
  if (!smc_counts_ok(N, A, Mb)) return fail(NERFB200_EINVAL, "%s: bricks_host is not a plan's {active, march}", who);
  CubScratch sc;
  if (plan_bytes < smc_plan_carve(N, plan_ws, &p, &sc))
    return fail(NERFB200_EINVAL, "%s: plan workspace smaller than nerfb200_sparse_mc_plan_workspace_bytes(N)", who);
  unsigned long long *rcnt, *vt;
  if (bytes < smc_carve(A, Mb, ws, &p, &rcnt, &vt, &sc))
    return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_sparse_mc_workspace_bytes(N, active, march)", who);
  p.thr = threshold;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int h[2] = {0, 0};
  CUDA_TRY(cudaMemcpyAsync(h, p.nsel + 1, sizeof(h), cudaMemcpyDeviceToHost, s), "sparse_mc count readback");
  CUDA_TRY(cudaStreamSynchronize(s), "sparse_mc count readback");
  if (h[0] != A || h[1] != Mb) return fail(NERFB200_EINVAL, "%s: bricks_host differs from the plan's", who);
  if (A == 0) {
    CUDA_TRY(cudaMemsetAsync(vt, 0, 2 * sizeof(unsigned long long), s), "sparse_mc count memset");
    counts_host[0] = counts_host[1] = 0;
    return 0;
  }
  // sigma: rows of the active bricks in order, one point query per kSmcChunkBricks bricks
  CUDA_TRY(cudaMemsetAsync(p.vals, 0, static_cast<size_t>(A) * kBrickPoints * sizeof(float), s), "sparse_mc memset");
  TRY(smc_query(p, sc, rcnt, A, packed, 1, nullptr, s, [&](long long rows) {
    return launch("sparse_mc sigma scatter launch", smc_sigma_scatter_kernel, grid_blocks(rows, 256), 256, 0, s, p, rows);
  }));
  // march: vertices and triangles per march brick
  CUDA_TRY(cudaMemsetAsync(p.bcnt + Mb, 0, sizeof(unsigned), s), "sparse_mc count memset");
  TRY(launch("sparse_mc march count launch", smc_march_count_kernel, grid_blocks(Mb, 1), kBrickPoints, 0, s, p));
  size_t tb = sc.temp_bytes;
  TRY(cub_launch(cub::DeviceScan::ExclusiveSum(sc.temp, tb, SmcVertIt(p.bcnt, SmcVerts()), p.vofs,
                                               static_cast<int>(Mb + 1), s), "sparse_mc vertex scan"));
  tb = sc.temp_bytes;
  TRY(cub_launch(cub::DeviceScan::ExclusiveSum(sc.temp, tb, SmcTriIt(p.bcnt, SmcTris()), p.tofs,
                                               static_cast<int>(Mb + 1), s), "sparse_mc triangle scan"));
  CUDA_TRY(cudaMemcpyAsync(vt, p.vofs + Mb, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s), "sparse_mc count copy");
  CUDA_TRY(cudaMemcpyAsync(vt + 1, p.tofs + Mb, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s), "sparse_mc count copy");
  unsigned long long c2[2] = {0, 0};
  CUDA_TRY(cudaMemcpyAsync(c2, vt, sizeof(c2), cudaMemcpyDeviceToHost, s), "sparse_mc count readback");
  CUDA_TRY(cudaStreamSynchronize(s), "sparse_mc count readback");
  if (c2[0] > static_cast<unsigned long long>(kSmcMaxCount) || c2[1] > static_cast<unsigned long long>(kSmcMaxCount))
    return fail(NERFB200_EUNSUPPORTED, "%s: %llu vertices and %llu triangles: both must stay below 2^31", who, c2[0], c2[1]);
  counts_host[0] = static_cast<int64_t>(c2[0]);
  counts_host[1] = static_cast<int64_t>(c2[1]);
  return 0;
}

size_t nerfb200_sparse_mc_emit_workspace_bytes(int64_t n_vertices, int64_t n_triangles) {
  if (n_vertices < 0 || n_triangles < 0 || n_vertices > kSmcMaxCount || n_triangles > kSmcMaxCount) return 0;
  unsigned long long *vk[2], *tk[2];
  CubScratch sc;
  return smc_emit_carve(n_vertices, n_triangles, nullptr, vk, tk, &sc);
}

int nerfb200_sparse_mc_emit(int64_t N, double threshold, void* plan_ws, size_t plan_bytes,
                            const int64_t bricks_host[2], void* ws, size_t bytes, const int64_t counts_host[2],
                            void* emit_ws, size_t emit_bytes, double* vertices, int32_t* triangles, void* stream) {
  const char* who = "sparse_mc_emit";
  if (N < 2 || N > kSmcMaxN) return fail(NERFB200_EINVAL, "%s: N must be in [2, 2048]", who);
  if (!plan_ws || !bricks_host || !ws || !counts_host || !emit_ws) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  const long long A = bricks_host[0], Mb = bricks_host[1], V = counts_host[0], T = counts_host[1];
  if (!smc_counts_ok(N, A, Mb)) return fail(NERFB200_EINVAL, "%s: bricks_host is not a plan's {active, march}", who);
  if (V < 0 || T < 0 || V > kSmcMaxCount || T > kSmcMaxCount || (V == 0 && T > 0))
    return fail(NERFB200_EINVAL, "%s: counts_host is not count's {V, T}", who);
  if ((V > 0 && !vertices) || (T > 0 && !triangles)) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  SparseMcParams p{};
  p.m.N = N;
  p.nb = smc_bricks(N);
  p.thr = threshold;
  CubScratch sc, se;
  if (plan_bytes < smc_plan_carve(N, plan_ws, &p, &sc))
    return fail(NERFB200_EINVAL, "%s: plan workspace smaller than nerfb200_sparse_mc_plan_workspace_bytes(N)", who);
  unsigned long long *rcnt, *vt;
  if (bytes < smc_carve(A, Mb, ws, &p, &rcnt, &vt, &sc))
    return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_sparse_mc_workspace_bytes(N, active, march)", who);
  unsigned long long *vk[2], *tk[2];
  if (emit_bytes < smc_emit_carve(V, T, emit_ws, vk, tk, &se))
    return fail(NERFB200_EINVAL, "%s: emit workspace smaller than nerfb200_sparse_mc_emit_workspace_bytes(V, T)", who);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  unsigned long long c2[2] = {0, 0};
  CUDA_TRY(cudaMemcpyAsync(c2, vt, sizeof(c2), cudaMemcpyDeviceToHost, s), "sparse_mc emit readback");
  CUDA_TRY(cudaStreamSynchronize(s), "sparse_mc emit readback");
  if (c2[0] != static_cast<unsigned long long>(V) || c2[1] != static_cast<unsigned long long>(T))
    return fail(NERFB200_EINVAL, "%s: counts_host differs from count's", who);
  if (V == 0) return 0;
  p.vkeys = vk[0];
  p.tkeys = tk[0];
  TRY(launch("sparse_mc march emit launch", smc_march_emit_kernel, grid_blocks(Mb, 1), kBrickPoints, 0, s, p));
  cub::DoubleBuffer<unsigned long long> vb(vk[0], vk[1]), tbuf(tk[0], tk[1]);
  size_t tb = se.temp_bytes;
  TRY(cub_launch(cub::DeviceRadixSort::SortKeys(se.temp, tb, vb, static_cast<int>(V), 0, bits_for(3 * N * N * N), s),
                 "sparse_mc vertex sort"));
  tb = se.temp_bytes;
  TRY(cub_launch(cub::DeviceRadixSort::SortKeys(se.temp, tb, tbuf, static_cast<int>(T), 0,
                                                bits_for(5 * (N - 1) * (N - 1) * (N - 1)), s), "sparse_mc triangle sort"));
  p.vkeys = vb.Current();
  p.tkeys = tbuf.Current();
  p.n_verts = V;
  p.n_tris = T;
  p.vertices = vertices;
  p.triangles = triangles;
  TRY(launch("sparse_mc vertices launch", smc_vertices_kernel, grid_blocks(V, 256), 256, 0, s, p));
  TRY(launch("sparse_mc triangles launch", smc_triangles_kernel, grid_blocks(T, 256), 256, 0, s, p));
  return 0;
}

// ---- baked volumes (include/nerf_pl_b200_baked.h, kernels: baked_kernels.cuh)
size_t nerfb200_baked_bytes(int64_t N, int64_t bricks) {
  return baked_bricks_ok(N, bricks) ? baked_bytes(N, bricks) : 0;
}

size_t nerfb200_baked_workspace_bytes(int64_t N, int64_t active, int64_t march) {
  if (!smc_counts_ok(N, active, march)) return 0;
  SparseMcParams p{};
  unsigned long long* rcnt;
  CubScratch sc;
  return baked_carve(active, nullptr, &p, &rcnt, &sc);
}

int nerfb200_baked_bake(const void* packed, int64_t N, const double ranges_host[6], const uint32_t* bits, int64_t occ_N,
                        const double occ_ranges_host[6], void* plan_ws, size_t plan_bytes, const int64_t bricks_host[2],
                        void* ws, size_t bytes, void* volume, size_t volume_bytes, void* stream) {
  return baked_bake<1>("baked_bake", packed, N, ranges_host, bits, occ_N, occ_ranges_host, plan_ws, plan_bytes,
                       bricks_host, ws, bytes, volume, volume_bytes, stream);
}

int nerfb200_baked_from_grid_count(const float* rgbsigma, int64_t N, void* plan_ws, size_t plan_bytes,
                                   int64_t bricks_host[1], void* stream) {
  return baked_from_grid_count<1>("baked_from_grid_count", rgbsigma, N, plan_ws, plan_bytes, bricks_host, stream);
}

int nerfb200_baked_from_grid(const float* rgbsigma, int64_t N, void* plan_ws, size_t plan_bytes, int64_t bricks,
                             void* volume, size_t volume_bytes, void* stream) {
  return baked_from_grid<1>("baked_from_grid", rgbsigma, N, plan_ws, plan_bytes, bricks, volume, volume_bytes, stream);
}

int nerfb200_baked_to_dense(const void* volume, size_t volume_bytes, int64_t N, int64_t bricks, float* rgbsigma,
                            void* stream) {
  return baked_to_dense<1>("baked_to_dense", volume, volume_bytes, N, bricks, rgbsigma, stream);
}

int nerfb200_baked_render(const void* volume, size_t volume_bytes, int64_t N, const double ranges_host[6], int64_t bricks,
                          const float* rays, int64_t n_rays, double step, int32_t white_back, double early_stop,
                          float* rgb, float* depth, float* opacity, void* stream) {
  return baked_render<1>("baked_render", volume, volume_bytes, N, ranges_host, bricks, rays, n_rays, step, white_back,
                         early_stop, rgb, depth, opacity, stream);
}

// ---- view-dependent baked volumes (include/nerf_pl_b200_baked_sh.h)
size_t nerfb200_baked_sh_bytes(int64_t N, int64_t bricks) {
  return baked_bricks_ok(N, bricks, 7) ? baked_bytes(N, bricks, 7) : 0;
}

size_t nerfb200_baked_sh_workspace_bytes(int64_t N, int64_t active, int64_t march) {
  if (N > kBakedShMaxN || !smc_counts_ok(N, active, march)) return 0;
  SparseMcParams p{};
  unsigned long long* rcnt;
  CubScratch sc;
  void* sh_ws;
  return baked_carve(active, nullptr, &p, &rcnt, &sc, 7, &sh_ws);
}

int nerfb200_baked_sh_bake(const void* packed, int64_t N, const double ranges_host[6], const uint32_t* bits,
                           int64_t occ_N, const double occ_ranges_host[6], void* plan_ws, size_t plan_bytes,
                           const int64_t bricks_host[2], void* ws, size_t bytes, void* volume, size_t volume_bytes,
                           void* stream) {
  return baked_bake<7>("baked_sh_bake", packed, N, ranges_host, bits, occ_N, occ_ranges_host, plan_ws, plan_bytes,
                       bricks_host, ws, bytes, volume, volume_bytes, stream);
}

int nerfb200_baked_sh_from_grid_count(const float* grid, int64_t N, void* plan_ws, size_t plan_bytes,
                                      int64_t bricks_host[1], void* stream) {
  return baked_from_grid_count<7>("baked_sh_from_grid_count", grid, N, plan_ws, plan_bytes, bricks_host, stream);
}

int nerfb200_baked_sh_from_grid(const float* grid, int64_t N, void* plan_ws, size_t plan_bytes, int64_t bricks,
                                void* volume, size_t volume_bytes, void* stream) {
  return baked_from_grid<7>("baked_sh_from_grid", grid, N, plan_ws, plan_bytes, bricks, volume, volume_bytes, stream);
}

int nerfb200_baked_sh_to_dense(const void* volume, size_t volume_bytes, int64_t N, int64_t bricks, float* grid,
                               void* stream) {
  return baked_to_dense<7>("baked_sh_to_dense", volume, volume_bytes, N, bricks, grid, stream);
}

int nerfb200_baked_sh_render(const void* volume, size_t volume_bytes, int64_t N, const double ranges_host[6],
                             int64_t bricks, const float* rays, int64_t n_rays, double step, int32_t white_back,
                             double early_stop, float* rgb, float* depth, float* opacity, void* stream) {
  return baked_render<7>("baked_sh_render", volume, volume_bytes, N, ranges_host, bricks, rays, n_rays, step,
                         white_back, early_stop, rgb, depth, opacity, stream);
}

size_t nerfb200_query_rgb_sh_workspace_bytes(void) { return static_cast<size_t>(kShTableFloats) * sizeof(float); }

int nerfb200_query_rgb_sh(const float* xyz, int64_t n, int64_t xyz_stride, const void* packed, void* ws, size_t bytes,
                          float* out, void* stream) {
  const char* who = "query_rgb_sh";
  if (n < 0) return fail(NERFB200_EINVAL, "%s: n < 0", who);
  if (n == 0) return 0;
  if (!xyz || !packed || !ws || !out) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  if (xyz_stride < 3) return fail(NERFB200_EINVAL, "%s: xyz_stride < 3", who);
  if (reinterpret_cast<uintptr_t>(out) & 15) return fail(NERFB200_EINVAL, "%s: out must be 16-byte aligned", who);
  if (reinterpret_cast<uintptr_t>(ws) & 15) return fail(NERFB200_EINVAL, "%s: ws must be 16-byte aligned", who);
  if (bytes < nerfb200_query_rgb_sh_workspace_bytes())
    return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_query_rgb_sh_workspace_bytes()", who);
  DeviceInfo* d = nullptr;
  TRY(device_info(&d));
  float* table = static_cast<float*>(ws);
  TRY(launch("query_rgb_sh table launch", sh_table_kernel, kShDirs, kDirW, 0, stream, sh_fit(),
             static_cast<const uint8_t*>(packed), table));
  MlpParams p{};
  p.raw_xyz = 1;
  p.x = xyz; p.x_stride = xyz_stride; p.n = n;
  p.net = static_cast<const uint8_t*>(packed);
  p.out = out;
  p.sh = table;
  return launch_mlp(p, nullptr, stream, "query_rgb_sh launch");
}

int nerfb200_sh_fit_host(float dirs[192], float proj[576]) {
  if (!dirs || !proj) return fail(NERFB200_EINVAL, "sh_fit_host: NULL argument");
  std::memcpy(dirs, sh_fit().dirs, sizeof(sh_fit().dirs));
  std::memcpy(proj, sh_fit().proj, sizeof(sh_fit().proj));
  return 0;
}

}  // extern "C"
