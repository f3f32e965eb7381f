// C ABI of libnerf_pl_b200.so (declarations + reference citations: include/nerf_pl_b200.h).
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/nerf_pl_b200.h"
#include "aux_kernels.cuh"
#include "bwd_kernels.cuh"
#include "mesh_kernels.cuh"
#include "occupancy_kernels.cuh"

#include <thrust/iterator/transform_iterator.h>

using namespace nerfb200;

namespace {

thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

int fail(int code, const char* fmt, const char* detail = "") {
  std::snprintf(g_err, sizeof(g_err), fmt, detail);
  return code;
}
int cuda_fail(cudaError_t e, const char* where) {
  std::snprintf(g_err, sizeof(g_err), "%s: %s (%s)", where, cudaGetErrorString(e), cudaGetErrorName(e));
  return static_cast<int>(e);
}
#define CUDA_TRY(expr, where)                          \
  do {                                                 \
    cudaError_t e_ = (expr);                           \
    if (e_ != cudaSuccess) return cuda_fail(e_, where); \
  } while (0)

struct DeviceInfo {
  int sm_count = 0;
  int cc_major = 0, cc_minor = 0;
  bool attrs_set = false;
  int* status = nullptr;        // device view of the mapped status word below
  volatile int* status_host = nullptr;   // pinned, mapped: the kernels write it, the host polls it without a sync
};

// Read ONCE per process.  NERFB200_MAX_CTAS caps the persistent grids (render and mesh kernels), so tests can
// show that results do not depend on the grid; unset in production.
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
std::mutex g_mu;
DeviceInfo g_dev[64];

int device_info(DeviceInfo** out) {
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev), "cudaGetDevice");
  if (dev < 0 || dev >= 64) return fail(NERFB200_EDEVICE, "device ordinal out of range%s");
  std::lock_guard<std::mutex> lk(g_mu);
  DeviceInfo& d = g_dev[dev];
  if (d.sm_count == 0) {
    CUDA_TRY(cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev), "attr sm");
    CUDA_TRY(cudaDeviceGetAttribute(&d.cc_major, cudaDevAttrComputeCapabilityMajor, dev), "attr cc");
    CUDA_TRY(cudaDeviceGetAttribute(&d.cc_minor, cudaDevAttrComputeCapabilityMinor, dev), "attr cc minor");
  }
  // the kernels are built for sm_90a (wgmma, setmaxnreg), which only compute capability 9.0 executes
  if (d.cc_major != 9 || d.cc_minor != 0) return fail(NERFB200_EDEVICE, "nerf_pl_b200 needs an sm_90 (H100) device%s");
  if (!d.attrs_set) {
    CUDA_TRY(cudaFuncSetAttribute(render_rays_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kSmemTotal)), "smem attr render");
    CUDA_TRY(cudaFuncSetAttribute(render_rays_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kSmemTotal)), "smem attr render(save)");
    CUDA_TRY(cudaFuncSetAttribute(mlp_forward_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kSmemTotal)), "smem attr mlp");
    CUDA_TRY(cudaFuncSetAttribute(mlp_forward_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kSmemTotal)), "smem attr mlp(save)");
    CUDA_TRY(cudaFuncSetAttribute(chain_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kChSmemTotal)), "smem attr chain");
    CUDA_TRY(cudaFuncSetAttribute(chain_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kChSmemTotal)), "smem attr chain (probe)");
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
// memory, code 101; a training backward whose per-sample gradients overflowed fp16, code 102)
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
    std::snprintf(g_err, sizeof(g_err), "an earlier training backward reported device status 102: a per-sample "
                  "gradient exceeded the fp16 range of its layer's scale, its weight gradients are wrong");
  else
    std::snprintf(g_err, sizeof(g_err), "an earlier nerf_pl_b200 kernel reported device status %d", st);
  return NERFB200_EDEVICE;
}

int check_render_shapes(const nerfb200_render_args* a) {
  if (a == nullptr) return fail(NERFB200_EINVAL, "args is NULL%s");
  if (a->n_rays < 0) return fail(NERFB200_EINVAL, "n_rays < 0%s");
  if (a->n_samples != 32 && a->n_samples != 64 && a->n_samples != 128)
    return fail(NERFB200_EUNSUPPORTED, "N_samples must be 32, 64 or 128%s");
  if (a->n_importance < 0 || (a->n_importance % 32) != 0)
    return fail(NERFB200_EUNSUPPORTED, "N_importance must be a multiple of 32%s");
  if (a->n_samples + a->n_importance > kMaxSf)
    return fail(NERFB200_EUNSUPPORTED, "N_samples + N_importance must be <= 192%s");
  if (a->n_rays == 0) return 0;
  if (!a->rays || !a->packed_coarse) return fail(NERFB200_EINVAL, "rays / packed_coarse is NULL%s");
  if (a->ray_stride < 8) return fail(NERFB200_EINVAL, "ray_stride < 8%s");
  if (!a->opacity_coarse) return fail(NERFB200_EINVAL, "opacity_coarse is NULL%s");
  if (!a->test_time && (!a->rgb_coarse || !a->depth_coarse))
    return fail(NERFB200_EINVAL, "rgb_coarse / depth_coarse is NULL with test_time=0%s");
  if (a->n_importance > 0) {
    if (!a->packed_fine) return fail(NERFB200_EINVAL, "packed_fine is NULL with N_importance>0%s");
    if (!a->rgb_fine || !a->depth_fine || !a->opacity_fine)
      return fail(NERFB200_EINVAL, "fine outputs are NULL with N_importance>0%s");
  }
  if (a->rng_in_kernel == 2 && !a->rng_seed_dev) return fail(NERFB200_EINVAL, "rng_in_kernel = 2 needs rng_seed_dev%s");
  if (a->perturb > 0.f && !a->rng_in_kernel) {
    if (!a->perturb_rand) return fail(NERFB200_EINVAL, "perturb>0 needs perturb_rand%s");
    if (a->n_importance > 0 && !a->u_rand) return fail(NERFB200_EINVAL, "perturb>0 needs u_rand%s");
  }
  if (a->noise_std > 0.f) {
    if (!a->noise_coarse) return fail(NERFB200_EINVAL, "noise_std>0 needs noise_coarse%s");
    if (a->n_importance > 0 && !a->noise_fine) return fail(NERFB200_EINVAL, "noise_std>0 needs noise_fine%s");
  }
  if ((reinterpret_cast<uintptr_t>(a->packed_coarse) & 15) ||
      (reinterpret_cast<uintptr_t>(a->packed_fine) & 15))
    return fail(NERFB200_EINVAL, "packed images must be 16-byte aligned%s");
  return 0;
}


// ------------------------------------------------------------------ training workspace layout
// One device buffer per (n_rays, N_samples, N_importance); the layout is a pure function of those
// numbers and the SM count, recomputed on every call (no state kept in the library).
struct WgJobPlan { int ps, kind, split, n_split; };
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

void plan_wgrad(TrainLayout* L, int n_cta, WgradJob* jobs, int* cta_first);

void job_shape(int kind, int* a_fb, int* b_fb) {
  *a_fb = (kind == kJ9 || kind == kJDir) ? 2 : 4;
  *b_fb = (kind == kJ1 || kind == kJ5a || kind == kJDir) ? 1 : 4;
}

// The per-pass buffers of a training workspace, in PassBufs order, each from one call of `take`.
template <class Take>
void take_pass_bufs(PassBufs& b, Take&& take) {
  const size_t np = static_cast<size_t>(b.n_pad);
  b.enc = take(np * 128);
  b.act = take(np * 512 * 8);
  b.mask = reinterpret_cast<uint2*>(take(np * 32 * 8));
  b.d = take(np * 256);
  b.sigma = reinterpret_cast<float*>(take(np * 4));
  b.rgb = reinterpret_cast<float*>(take(np * 12));
  b.z = reinterpret_cast<float*>(take(static_cast<size_t>(b.n) * 4));
  b.dsigma = reinterpret_cast<float*>(take(np * 4));
  b.dprergb = reinterpret_cast<float*>(take(np * 12));
  b.dd = take(np * 256);
  b.dpre = take(np * 512 * 8);
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
  size_t off = 0;
  auto take = [&](size_t bytes) -> uint8_t* {
    uint8_t* ptr = base ? base + off : nullptr;
    off += (bytes + 1023) & ~static_cast<size_t>(1023);
    return ptr;
  };
  std::memset(L, 0, sizeof(*L));
  L->n_pass = n_importance > 0 ? 2 : 1;
  L->n_kinds = mlp ? kNumJobKindsMlp : kNumJobKinds;
  for (int ps = 0; ps < L->n_pass; ++ps) {
    PassBufs& b = L->pass[ps];
    b.S = ps ? n_samples + n_importance : n_samples;
    b.n = n * b.S;
    b.n_pad = (b.n + 127) / 128 * 128;
    take_pass_bufs(b, take);
  }
  if (mlp) L->xdir = take(static_cast<size_t>(L->pass[0].n_pad) * 128);
  const int64_t head_rays = mlp ? L->pass[0].n_pad / kMlpPseudoRay : n;
  L->n_rays = static_cast<int>(head_rays);
  plan_wgrad(L, sm_count > 0 ? sm_count : 148, nullptr, nullptr);
  L->jobs_dev = reinterpret_cast<WgradJob*>(take(sizeof(WgradJob) * kMaxWgJobs));
  L->cta_first_dev = reinterpret_cast<int*>(take(sizeof(int) * (kMaxWgCtas + 1)));
  L->wg_part = reinterpret_cast<float*>(take(static_cast<size_t>(L->n_cta) * kWgSlotFloats * 4));
  L->head_grid = static_cast<int>((L->n_pass * head_rays + kHeadWarps - 1) / kHeadWarps);
  if (!mlp) L->direnc = reinterpret_cast<float*>(take(static_cast<size_t>(n) * 28 * 4));
  for (int ps = 0; ps < (mlp ? 1 : 2); ++ps) {
    L->head_part[ps] = reinterpret_cast<float*>(take(static_cast<size_t>(L->head_grid) * kHeadPartFloats * 4));
    if (!mlp) {
      L->raysum[ps] = reinterpret_cast<float*>(take(static_cast<size_t>(n) * 128 * 4));
      L->dir_part[ps] = reinterpret_cast<float*>(take(static_cast<size_t>(kDirSlices) * 128 * 27 * 4));
    }
    L->gWp[ps] = reinterpret_cast<float*>(take(128 * 256 * 4));
    L->gbp[ps] = reinterpret_cast<float*>(take(128 * 4));
  }
  L->lscale = reinterpret_cast<float*>(take(2 * kLevels * 4));
  L->linv = reinterpret_cast<float*>(take(2 * kLevels * 4));
  L->lamax = reinterpret_cast<unsigned*>(take(2 * kLevels * 4));
  L->amax = reinterpret_cast<unsigned*>(take(16));
  if (!mlp) {
    L->loss_part = reinterpret_cast<float*>(take(1024 * 2 * 4));
    L->loss_counter = reinterpret_cast<unsigned*>(take(16));
  }
  L->bytes = off;
}

// The wgrad plan of a layout: CTA counts per (pass, layer) (always), and when `jobs` / `cta_first` are
// given the host image of the piece table and of the per-CTA piece ranges.
void job_operands(const TrainLayout& L, int ps, int k, const uint8_t** A, const uint8_t** B) {
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

void fill_piece(TrainLayout* L, WgradJob* jobs, int piece, int cta, int ps, int k, long long c0, long long c1,
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

void plan_wgrad(TrainLayout* L, int n_cta, WgradJob* jobs, int* cta_first) {
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
      const double share = static_cast<double>(work[ps][k]) * n_cta / static_cast<double>(total);
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
      n_cta_used += static_cast<int>(std::min<long long>(n_of[ps][k], L->pass[ps].n_pad / 64));
  const int max_pieces = kMaxWgJobs / n_cta_used;        // per CTA
  int piece = 0, cta = 0;
  for (int ps = 0; ps < L->n_pass; ++ps)
    for (int k = 0; k < kinds; ++k) {
      const long long chunks = L->pass[ps].n_pad / 64;
      int g = n_of[ps][k];
      if (g > chunks) g = static_cast<int>(chunks);
      L->first_cta[ps][k] = cta;
      for (int j = 0; j < g; ++j, ++cta) {
        const long long mine = (chunks - j + g - 1) / g;
        const long long len = std::max<long long>(kWgPieceChunks, (mine + max_pieces - 1) / max_pieces);
        if (cta_first) cta_first[cta] = piece;
        for (long long s = 0; s < mine; s += len, ++piece)
          fill_piece(L, jobs, piece, cta, ps, k, j + s * g, std::min(chunks, j + (s + len) * g), g, s > 0);
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
  size_t off = 0;
  int reserve(size_t bytes) {
    if (bytes <= cap) return 0;
    if (base) cudaFree(base);
    base = nullptr; cap = 0;
    cudaError_t e = cudaMalloc(&base, bytes);
    if (e != cudaSuccess) return cuda_fail(e, "arena cudaMalloc");
    cap = bytes;
    return 0;
  }
  void* take(size_t bytes) {
    void* p = base + off;
    off += (bytes + 255) & ~static_cast<size_t>(255);
    return p;
  }
};
Arena g_arena[64];
std::mutex g_host_call_mu;
std::mutex g_arena_mu;   // separate from g_mu: the host entry calls nerfb200_render_rays (device_info locks g_mu)

// Step 3 of a training backward: the chain kernel's probe pass over pt0 + pt1 tiles spread evenly over each pass, the
// phase-1 scales, then the real pass over all t0 + t1 tiles (the probe's first).  cp: everything but the visit order.
void launch_chain(ChainParams& cp, long long t0, long long t1, long long pt0, long long pt1, ScaleParams& sp, int sm_count,
                  cudaStream_t stream) {
  const long long span[2] = {t0, t1}, pt[2] = {pt0, pt1};
  auto gcd = [](long long x, long long y) {
    while (y != 0) { const long long r = x % y; x = y; y = r; }
    return x;
  };
  for (int ps = 0; ps < 2; ++ps) {
    long long s = (pt[ps] > 0 && span[ps] > pt[ps]) ? span[ps] / pt[ps] : 1;
    while (span[ps] > 1 && gcd(s, span[ps]) != 1) ++s;
    cp.span[ps] = span[ps] > 0 ? span[ps] : 1;
    cp.stride[ps] = s;
  }
  cp.tiles[0] = cp.head[0] = pt0;
  cp.tiles[1] = cp.head[1] = pt1;
  const int pc = static_cast<int>(pt0 + pt1);
  chain_bwd_kernel<true><<<pc, kThreads, kChSmemTotal, stream>>>(cp);
  g_launches++;
  sp.phase = 1;
  bwd_scale_kernel<<<1, 128, 0, stream>>>(sp);
  g_launches++;
  cp.head[0] = pt0;
  cp.head[1] = pt1;
  cp.tiles[0] = t0;
  cp.tiles[1] = t1;
  const long long total = t0 + t1;
  const int ctas = static_cast<int>(total < sm_count ? total : sm_count);
  chain_bwd_kernel<false><<<ctas, kThreads, kChSmemTotal, stream>>>(cp);
  g_launches++;
}

// Step 5: the reduction items of pass ps that both training backwards share (wgrad GEMMs of layers 1..8 and of the
// folded W', the head partials), appended to `tab`.  g: the pass's 24 gradient tensors.
void add_reduce_items(ReduceTable& tab, const TrainLayout& L, int ps, float* const* g) {
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

// Steps 2-6 of both training backwards, once step 1 has left each pass's per-sample d sigma / d rgb_pre and their
// maxima in the workspace.  params / grads / net: per pass.  rays: the render path's rays, whose directions the head
// kernel embeds for the per-ray direction part of gW_dir; null for a direct NeRF.forward call, whose head kernel walks
// pseudo-rays of 64 samples and whose direction part is the wgrad GEMM kJDir.
int backward_tail(const TrainLayout& L, const float* const* const params[2], float* const* const grads[2],
                  const uint8_t* const net[2], const float* rays, long long ray_stride, const DeviceInfo* d,
                  cudaStream_t stream, const char* what) {
  const int q1 = L.n_pass > 1 ? 1 : 0;        // table entry of the second pass: a single pass fills both slots
  ScaleParams sp;
  sp.n_pass = L.n_pass; sp.phase = 0;
  sp.amax = L.amax; sp.lamax = L.lamax; sp.lscale = L.lscale; sp.linv = L.linv;
  sp.w_rgb[0] = params[0][22]; sp.w_rgb[1] = params[q1][22];
  sp.w_sigma[0] = params[0][20]; sp.w_sigma[1] = params[q1][20];
  bwd_scale_kernel<<<1, 128, 0, stream>>>(sp);
  g_launches++;
  // 2. rgb head, ReLU of the direction layer (both passes in one launch), direction part of gW_dir
  HeadBwdParams hp;
  hp.n_rays = L.n_rays; hp.n_pass = L.n_pass;
  hp.pass[0] = L.pass[0]; hp.pass[1] = L.pass[1];
  if (!rays) {
    hp.pass[0].S = kMlpPseudoRay;
    hp.pass[1] = hp.pass[0];
  }
  hp.w_rgb[0] = params[0][22]; hp.w_rgb[1] = params[q1][22];
  hp.lscale = L.lscale;
  hp.rays = rays; hp.ray_stride = ray_stride;
  hp.raysum[0] = L.raysum[0]; hp.raysum[1] = L.raysum[1];
  hp.direnc = L.direnc;
  hp.part[0] = L.head_part[0]; hp.part[1] = L.head_part[1];
  head_bwd_kernel<<<L.head_grid, kHeadWarps * 32, 0, stream>>>(hp);
  g_launches++;
  if (rays) {
    DirGradParams dp;
    dp.n_rays = L.n_rays;
    dp.raysum[0] = L.raysum[0]; dp.raysum[1] = L.raysum[1];
    dp.direnc = L.direnc;
    dp.part[0] = L.dir_part[0]; dp.part[1] = L.dir_part[1];
    dir_grad_kernel<<<dim3(kDirSlices, L.n_pass), 128, 0, stream>>>(dp);
    g_launches++;
  }
  // 3. dgrad chain (wgmma): a probe pass over one tile per SM picks the per-layer scales, then the real pass.
  // The probe's tiles are spread evenly over each pass: gradients are not uniform over a batch (rays whose
  // colour is already right carry almost none), and scales taken from the first tiles alone saturate the rest.
  // Both launches visit the tiles of a pass in the order j -> j * stride mod span (stride coprime to span, about
  // span / probe tiles), the real pass the probe's tiles first, so its first wave finds them in L2.  A tile the
  // probe did not see can still exceed its level's range: the wgrad kernel reports that (status 102).
  ChainParams cp;
  cp.n_pass = L.n_pass;
  cp.pass[0] = L.pass[0]; cp.pass[1] = L.pass[1];
  cp.net[0] = net[0]; cp.net[1] = net[1];
  cp.lscale = L.lscale;
  cp.lamax = L.lamax;
  cp.status = d->status;
  const long long t0 = L.pass[0].n_pad / 128, t1 = q1 ? L.pass[1].n_pad / 128 : 0;
  const long long probe = q1 ? (d->sm_count + 1) / 2 : d->sm_count;      // probe tiles per pass, at most
  launch_chain(cp, t0, t1, t0 < probe ? t0 : probe, t1 < probe ? t1 : probe, sp, d->sm_count, stream);
  // 4. split-K wgrad (wgmma)
  wgrad_kernel<<<L.n_cta, kWgThreads, kWgSmemTotal, stream>>>(L.jobs_dev, L.cta_first_dev, d->status);
  g_launches++;
  // 5. partial sums -> gradient tensors (fixed order), 6. unfold W'
  ReduceTable tab;
  tab.n = 0;
  for (int ps = 0; ps < L.n_pass; ++ps) add_reduce_items(tab, L, ps, grads[ps]);
  wgrad_reduce_kernel<<<dim3(64, tab.n), 256, 0, stream>>>(tab);   // latency-bound: 64 blocks per item (16 measured 40 us)
  g_launches++;
  UnfoldParams up;
  for (int ps = 0; ps < 2; ++ps) {
    const int q = ps ? q1 : 0;
    up.gWp[ps] = L.gWp[q]; up.gbp[ps] = L.gbp[q];
    up.Wf[ps] = params[q][16]; up.bf[ps] = params[q][17]; up.Wd[ps] = params[q][18];
    up.gWd[ps] = grads[q][18]; up.gbd[ps] = grads[q][19]; up.gWf[ps] = grads[q][16]; up.gbf[ps] = grads[q][17];
  }
  // warps: one per gWd output (128 x 256), then one thread per gWf / gbf output
  unfold_kernel<<<dim3((128 * 256 + (256 * 256 + 256 + 31) / 32 + 7) / 8, L.n_pass), 256, 0, stream>>>(up);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), what);
  return 0;
}

// The four entries of mlp_forward_kernel, after their own checks: one CTA per 128-row tile, at most one per SM.  With
// a NeRF.forward training workspace `ws` the save-mode instantiation also stores what nerfb200_nerf_backward reads.
int launch_mlp(MlpParams p, void* ws, void* stream, const char* what) {
  DeviceInfo* d = nullptr;
  int rc = device_info(&d);
  if (rc) return rc;
  if ((rc = check_sticky_status(d)) != 0) return rc;
  p.status = d->status;
  const long long tiles = (p.n + 127) / 128;
  const int ctas = static_cast<int>(tiles < d->sm_count ? tiles : d->sm_count);
  if (ws) {
    TrainLayout L;
    make_train_layout(&L, static_cast<uint8_t*>(ws), true, p.n, 1, 0, d->sm_count);
    p.tr = L.pass[0];
    p.xdir = L.xdir;
    mlp_forward_kernel<true><<<ctas, kThreads, kSmemTotal, static_cast<cudaStream_t>(stream)>>>(p);
  } else {
    mlp_forward_kernel<false><<<ctas, kThreads, kSmemTotal, static_cast<cudaStream_t>(stream)>>>(p);
  }
  g_launches++;
  CUDA_TRY(cudaGetLastError(), what);
  return 0;
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

static int fill_pack_params(PackParams* pp, const float* const params[24], void* packed) {
  if (!params || !packed) return fail(NERFB200_EINVAL, "pack_weights: NULL argument%s");
  if (reinterpret_cast<uintptr_t>(packed) & 15) return fail(NERFB200_EINVAL, "packed must be 16-byte aligned%s");
  for (int i = 0; i < kNumParams; ++i) {
    if (!params[i]) return fail(NERFB200_EINVAL, "pack_weights: NULL parameter tensor%s");
    pp->p[i] = params[i];
  }
  pp->out = static_cast<uint8_t*>(packed);
  return 0;
}

static int launch_pack(const PackParams2& pp2, int n_nets, void* stream) {
  const long long total = kHalfRegionBytes / 2 + kF32Count + static_cast<long long>(kNumSlicesBwd) * 256 * 64;
  const int threads = 256;
  const int blocks = static_cast<int>((total + threads - 1) / threads);
  pack_weights_kernel<<<dim3(blocks, n_nets), threads, 0, static_cast<cudaStream_t>(stream)>>>(pp2);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "pack_weights launch");
  return 0;
}

int nerfb200_pack_weights(const float* const params[24], void* packed, void* stream) {
  PackParams2 pp2;
  int rc = fill_pack_params(&pp2.net[0], params, packed);
  if (rc) return rc;
  pp2.net[1] = pp2.net[0];
  return launch_pack(pp2, 1, stream);
}

int nerfb200_pack_weights_pair(const float* const params_a[24], void* packed_a, const float* const params_b[24],
                               void* packed_b, void* stream) {
  PackParams2 pp2;
  int rc = fill_pack_params(&pp2.net[0], params_a, packed_a);
  if (rc) return rc;
  rc = fill_pack_params(&pp2.net[1], params_b, packed_b);
  if (rc) return rc;
  return launch_pack(pp2, 2, stream);
}

int nerfb200_render_rays(const nerfb200_render_args* a, void* stream) {
  int rc = check_render_shapes(a);
  if (rc) return rc;
  if (a->n_rays == 0) return 0;
  if (a->n_rays > 0x7fffffff) return fail(NERFB200_EINVAL, "n_rays too large%s");
  DeviceInfo* d = nullptr;
  rc = device_info(&d);
  if (rc) return rc;
  if (!a->status && (rc = check_sticky_status(d)) != 0) return rc;
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
  if (save && a->test_time) return fail(NERFB200_EINVAL, "train_workspace needs test_time = 0%s");
  if ((a->target != nullptr) != (a->loss_out != nullptr)) return fail(NERFB200_EINVAL, "target and loss_out go together%s");
  if (a->target && !save) return fail(NERFB200_EINVAL, "the fused loss epilogue needs train_workspace%s");
  if (save) {
    TrainLayout L;
    make_train_layout(&L, static_cast<uint8_t*>(a->train_workspace), false, a->n_rays, a->n_samples, a->n_importance,
                      d->sm_count);
    p.train = 1;
    p.tr[0] = L.pass[0];
    p.tr[1] = L.pass[1];
    if (!p.z_coarse) p.z_coarse = L.pass[0].z;
    else return fail(NERFB200_EINVAL, "z_coarse is owned by the workspace in training mode%s");
    if (a->n_importance > 0) {
      if (p.z_fine) return fail(NERFB200_EINVAL, "z_fine is owned by the workspace in training mode%s");
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
  if (save)
    render_rays_kernel<true><<<ctas, kRenderThreads, kSmemTotal, static_cast<cudaStream_t>(stream)>>>(p);
  else
    render_rays_kernel<false><<<ctas, kRenderThreads, kSmemTotal, static_cast<cudaStream_t>(stream)>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "render_rays launch");
  return 0;
}

int nerfb200_render_rays_host(const nerfb200_render_args* h, void* stream_v) {
  int rc = check_render_shapes(h);
  if (rc) return rc;
  if (h->n_rays == 0) return 0;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (h->train_workspace || h->target || h->z_coarse)
    return fail(NERFB200_EINVAL, "render_rays_host: train_workspace / target / z_coarse are device-only%s");
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
      rc = nerfb200_render_rays(&a, stream);
      if (rc) return rc;
      CUDA_TRY(cudaStreamSynchronize(stream), "render_rays_host sync");
      const int hstatus = *hs;
      if (hstatus != 0) {
        std::snprintf(g_err, sizeof(g_err), "render kernel reported device status %d", hstatus);
        return NERFB200_EDEVICE;
      }
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
  rc = ar.reserve(need);
  if (rc) return rc;
  ar.off = 0;
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
    float* dst = static_cast<float*>(ar.take(count * fl));
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
    return hostp ? static_cast<float*>(ar.take(count * fl)) : nullptr;
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
  int* dstatus = static_cast<int*>(ar.take(sizeof(int)));
  CUDA_TRY(cudaMemsetAsync(dstatus, 0, sizeof(int), stream), "status memset");
  a.status = dstatus;
  rc = nerfb200_render_rays(&a, stream);
  if (rc) return rc;
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
  if (hstatus != 0) {
    std::snprintf(g_err, sizeof(g_err), "render kernel reported device status %d", hstatus);
    return NERFB200_EDEVICE;
  }
  if (h->status) *h->status = hstatus;
  return 0;
}

int nerfb200_nerf_forward(const float* x, int64_t n, int64_t x_stride, const void* packed,
                          int32_t sigma_only, float* out, void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "nerf_forward: n < 0%s");
  if (n == 0) return 0;
  if (!x || !packed || !out) return fail(NERFB200_EINVAL, "nerf_forward: NULL argument%s");
  if (x_stride < (sigma_only ? kEncXyz : kEncXyz + kEncDir))
    return fail(NERFB200_EINVAL, "nerf_forward: x_stride too small for the input width%s");
  if (!sigma_only && (reinterpret_cast<uintptr_t>(out) & 15))
    return fail(NERFB200_EINVAL, "nerf_forward: out must be 16-byte aligned%s");
  MlpParams p{};
  p.x = x; p.x_stride = x_stride; p.n = n;
  p.net = static_cast<const uint8_t*>(packed);
  p.sigma_only = sigma_only;
  p.out = out;
  return launch_mlp(p, nullptr, stream, "nerf_forward launch");
}

int nerfb200_query_sigma(const float* xyz, int64_t n, int64_t xyz_stride, const void* packed, float* sigma,
                         void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "query_sigma: n < 0%s");
  if (n == 0) return 0;
  if (!xyz || !packed || !sigma) return fail(NERFB200_EINVAL, "query_sigma: NULL argument%s");
  if (xyz_stride < 3) return fail(NERFB200_EINVAL, "query_sigma: xyz_stride < 3%s");
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
  if (n < 0) return fail(NERFB200_EINVAL, "query_rgb_sigma: n < 0%s");
  if (n == 0) return 0;
  if (!xyz || !packed || !rgbsigma) return fail(NERFB200_EINVAL, "query_rgb_sigma: NULL argument%s");
  if (xyz_stride < 3) return fail(NERFB200_EINVAL, "query_rgb_sigma: xyz_stride < 3%s");
  if (reinterpret_cast<uintptr_t>(rgbsigma) & 15) return fail(NERFB200_EINVAL, "query_rgb_sigma: out must be 16-byte aligned%s");
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
  if (n < 0 || n > 0x7fffffffLL) return fail(NERFB200_EINVAL, "nerf_train_workspace_init: n out of range%s");
  if (n == 0) return 0;
  if (!ws) return fail(NERFB200_EINVAL, "nerf_train_workspace_init: workspace is NULL%s");
  if (reinterpret_cast<uintptr_t>(ws) & 1023) return fail(NERFB200_EINVAL, "nerf train workspace must be 1024-byte aligned%s");
  if (bytes < nerfb200_nerf_train_workspace_bytes(n)) return fail(NERFB200_EINVAL, "nerf train workspace too small for n%s");
  DeviceInfo* d = nullptr;
  int rc = device_info(&d);
  if (rc) return rc;
  TrainLayout L;
  make_train_layout(&L, static_cast<uint8_t*>(ws), true, n, 1, 0, d->sm_count);
  if (bytes < L.bytes) return fail(NERFB200_EINVAL, "nerf train workspace too small for n%s");
  return init_train_workspace(L, ws, d->sm_count, static_cast<cudaStream_t>(stream_v));
}

int nerfb200_nerf_forward_train(const float* x, int64_t n, int64_t x_stride, const void* packed, void* ws, float* out,
                                void* stream) {
  if (n < 0 || n > 0x7fffffffLL) return fail(NERFB200_EINVAL, "nerf_forward_train: n out of range%s");
  if (n == 0) return 0;
  if (!x || !packed || !ws || !out) return fail(NERFB200_EINVAL, "nerf_forward_train: NULL argument%s");
  if (x_stride < kEncXyz + kEncDir) return fail(NERFB200_EINVAL, "nerf_forward_train: x_stride < 90%s");
  if ((reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(packed) & 15))
    return fail(NERFB200_EINVAL, "nerf_forward_train: out / packed must be 16-byte aligned%s");
  if (reinterpret_cast<uintptr_t>(ws) & 1023) return fail(NERFB200_EINVAL, "nerf train workspace must be 1024-byte aligned%s");
  MlpParams p{};
  p.x = x; p.x_stride = x_stride; p.n = n;
  p.net = static_cast<const uint8_t*>(packed);
  p.out = out;
  return launch_mlp(p, ws, stream, "nerf_forward_train launch");
}

int nerfb200_nerf_backward(const float* g_out, int64_t n, const void* packed, const float* const params[24], void* ws,
                           float* const grads[24], void* stream_v) {
  if (n < 0 || n > 0x7fffffffLL) return fail(NERFB200_EINVAL, "nerf_backward: n out of range%s");
  if (n == 0) return 0;
  if (!g_out || !packed || !params || !ws || !grads) return fail(NERFB200_EINVAL, "nerf_backward: NULL argument%s");
  for (int i = 0; i < kNumParams; ++i)
    if (!params[i] || !grads[i]) return fail(NERFB200_EINVAL, "nerf_backward: NULL parameter / gradient tensor%s");
  if (reinterpret_cast<uintptr_t>(g_out) & 15) return fail(NERFB200_EINVAL, "nerf_backward: g_out must be 16-byte aligned%s");
  if (reinterpret_cast<uintptr_t>(ws) & 1023) return fail(NERFB200_EINVAL, "nerf train workspace must be 1024-byte aligned%s");
  DeviceInfo* d = nullptr;
  int rc = device_info(&d);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  TrainLayout L;
  make_train_layout(&L, static_cast<uint8_t*>(ws), true, n, 1, 0, d->sm_count);
  const PassBufs& pb = L.pass[0];
  // 1. seed: upstream gradient -> per-sample d sigma / d rgb_pre (replaces the compositing backward)
  MlpSeedParams sd;
  sd.n = n; sd.n_pad = pb.n_pad;
  sd.g = g_out; sd.rgb = pb.rgb; sd.dsigma = pb.dsigma; sd.dprergb = pb.dprergb;
  sd.amax_bits = L.amax;
  mlp_seed_kernel<<<static_cast<int>((pb.n_pad + 255) / 256), 256, 0, stream>>>(sd);
  g_launches++;
  const float* const* const p2[2] = {params, params};
  float* const* const g2[2] = {grads, grads};
  const uint8_t* const net[2] = {static_cast<const uint8_t*>(packed), static_cast<const uint8_t*>(packed)};
  return backward_tail(L, p2, g2, net, nullptr, 0, d, stream, "nerf_backward launches");
}

int nerfb200_mse_psnr(const float* rgb_coarse, const float* rgb_fine, const float* target, int64_t n_rays,
                      float* out4, void* stream) {
  if (n_rays <= 0) return fail(NERFB200_EINVAL, "mse_psnr: n_rays <= 0%s");
  if ((!rgb_coarse && !rgb_fine) || !target || !out4) return fail(NERFB200_EINVAL, "mse_psnr: NULL argument%s");
  mse_psnr_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(rgb_coarse, rgb_fine, target, n_rays * 3, out4);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "mse_psnr launch");
  return 0;
}

int nerfb200_embed(const float* x, int64_t n, int32_t n_freqs, float* out, void* stream) {
  if (n < 0 || n_freqs < 0 || n_freqs > 16) return fail(NERFB200_EINVAL, "embed: bad n / n_freqs%s");
  if (n == 0) return 0;
  if (!x || !out) return fail(NERFB200_EINVAL, "embed: NULL argument%s");
  const long long total = n * (3 + 6 * n_freqs);
  const int threads = 256;
  long long blocks = (total + threads - 1) / threads;
  if (blocks > 148 * 16) blocks = 148 * 16;
  embed_kernel<<<static_cast<int>(blocks), threads, 0, static_cast<cudaStream_t>(stream)>>>(x, n, n_freqs, out);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "embed launch");
  return 0;
}

int nerfb200_searchsorted(const float* a, const float* v, int64_t* out, int64_t nrow_a,
                          int64_t nrow_v, int32_t ncol_a, int32_t ncol_v, int32_t side_right,
                          void* stream) {
  if (nrow_a < 0 || nrow_v < 0 || ncol_a < 0 || ncol_v < 0)
    return fail(NERFB200_EINVAL, "searchsorted: negative size%s");
  // searchsorted.py:26-29: same number of rows, or one of them has a single row
  if (nrow_a != nrow_v && nrow_a != 1 && nrow_v != 1)
    return fail(NERFB200_EINVAL, "searchsorted: a and v need the same number of rows, or 1 row%s");
  const long long nrow = nrow_a > nrow_v ? nrow_a : nrow_v;
  const long long total = nrow * ncol_v;
  if (total == 0) return 0;
  if (!a && ncol_a > 0) return fail(NERFB200_EINVAL, "searchsorted: a is NULL%s");
  if (!v || !out) return fail(NERFB200_EINVAL, "searchsorted: NULL argument%s");
  const int threads = 256;
  long long blocks = (total + threads - 1) / threads;
  if (blocks > 148 * 16) blocks = 148 * 16;
  searchsorted_kernel<<<static_cast<int>(blocks), threads, 0, static_cast<cudaStream_t>(stream)>>>(
      a, v, reinterpret_cast<long long*>(out), nrow_a, nrow_v, ncol_a, ncol_v, side_right);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "searchsorted launch");
  return 0;
}

int nerfb200_sample_pdf(const float* bins, const float* weights, const float* u, int64_t n_rays,
                        int32_t n_weights, int32_t n_u, float* out, void* stream) {
  if (n_rays < 0 || n_weights < 1 || n_u < 0 || n_weights > kPdfMaxWeights)
    return fail(NERFB200_EINVAL, "sample_pdf: bad sizes%s");
  if (n_rays == 0 || n_u == 0) return 0;
  if (!bins || !weights || !u || !out) return fail(NERFB200_EINVAL, "sample_pdf: NULL argument%s");
  DeviceInfo* d = nullptr;
  const int rc = device_info(&d);           // opts sample_pdf_kernel in to its shared memory
  if (rc) return rc;
  const int wpb = kPdfWarps;
  const size_t sh = wpb * (n_weights + 1) * sizeof(float);
  long long blocks = (n_rays + wpb - 1) / wpb;
  if (blocks > 148 * 8) blocks = 148 * 8;
  sample_pdf_kernel<<<static_cast<int>(blocks), wpb * 32, sh, static_cast<cudaStream_t>(stream)>>>(
      bins, weights, u, n_rays, n_weights, n_u, out);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "sample_pdf launch");
  return 0;
}

int nerfb200_composite(const float* sigmas, const float* rgbs, const float* z_vals,
                       const float* dirs, const float* noise, float noise_std, int32_t white_back,
                       int64_t n_rays, int32_t S, float* weights, float* rgb, float* depth,
                       float* opacity, void* stream) {
  if (n_rays < 0) return fail(NERFB200_EINVAL, "composite: n_rays < 0%s");
  if (S <= 0 || (S % 32) != 0 || S > kMaxSf) return fail(NERFB200_EUNSUPPORTED, "composite: S must be a multiple of 32, <= 192%s");
  if (n_rays == 0) return 0;
  if (!sigmas || !z_vals || !dirs || !opacity) return fail(NERFB200_EINVAL, "composite: NULL argument%s");
  if (rgbs && (!rgb || !depth)) return fail(NERFB200_EINVAL, "composite: rgb/depth outputs NULL%s");
  const int wpb = 4;
  const size_t sh = wpb * 6 * S * sizeof(float);
  long long blocks = (n_rays + wpb - 1) / wpb;
  if (blocks > 148 * 8) blocks = 148 * 8;
  composite_kernel<<<static_cast<int>(blocks), wpb * 32, sh, static_cast<cudaStream_t>(stream)>>>(
      sigmas, rgbs, z_vals, dirs, noise, noise_std, white_back, n_rays, S, weights, rgb, depth, opacity);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "composite launch");
  return 0;
}

int nerfb200_generate_rays(int32_t H, int32_t W, float focal, const float c2w_host[12], float near, float far,
                           int32_t ndc, float* rays, void* stream) {
  if (H <= 0 || W <= 0 || !(focal > 0.f)) return fail(NERFB200_EINVAL, "generate_rays: bad H / W / focal%s");
  if (!c2w_host || !rays) return fail(NERFB200_EINVAL, "generate_rays: NULL argument%s");
  if (reinterpret_cast<uintptr_t>(rays) & 15) return fail(NERFB200_EINVAL, "generate_rays: rays must be 16-byte aligned%s");
  RayGenParams p;
  p.H = H; p.W = W; p.focal = focal; p.near = near; p.far = far; p.ndc = ndc; p.rays = rays;
  for (int i = 0; i < 12; ++i) p.c2w[i] = c2w_host[i];
  const long long total = static_cast<long long>(H) * W;
  long long blocks = (total + 255) / 256;
  if (blocks > 148 * 8) blocks = 148 * 8;
  generate_rays_kernel<<<static_cast<int>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "generate_rays launch");
  return 0;
}

int nerfb200_to_uint8(const float* src, int64_t n, uint8_t* dst, void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "to_uint8: n < 0%s");
  if (n == 0) return 0;
  if (!src || !dst) return fail(NERFB200_EINVAL, "to_uint8: NULL argument%s");
  long long blocks = (n + 255) / 256;
  if (blocks > 148 * 8) blocks = 148 * 8;
  to_uint8_kernel<<<static_cast<int>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(src, n, dst);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "to_uint8 launch");
  return 0;
}

size_t nerfb200_train_workspace_bytes(int64_t n_rays, int32_t n_samples, int32_t n_importance) {
  if (n_rays <= 0 || n_samples <= 0 || n_importance < 0) return 0;
  TrainLayout L;
  make_train_layout(&L, nullptr, false, n_rays, n_samples, n_importance, nerfb200_sm_count());
  return L.bytes;
}

int nerfb200_train_workspace_init(void* workspace, size_t bytes, int64_t n_rays, int32_t n_samples,
                                  int32_t n_importance, void* stream_v) {
  if (!workspace || n_rays <= 0) return fail(NERFB200_EINVAL, "train_workspace_init: bad argument%s");
  if (reinterpret_cast<uintptr_t>(workspace) & 1023) return fail(NERFB200_EINVAL, "train workspace must be 1024-byte aligned%s");
  DeviceInfo* d = nullptr;
  int rc = device_info(&d);
  if (rc) return rc;
  TrainLayout L;
  make_train_layout(&L, static_cast<uint8_t*>(workspace), false, n_rays, n_samples, n_importance, d->sm_count);
  if (bytes < L.bytes) return fail(NERFB200_EINVAL, "train workspace too small%s");
  return init_train_workspace(L, workspace, d->sm_count, static_cast<cudaStream_t>(stream_v));
}

int nerfb200_render_backward(const nerfb200_backward_args* b, void* stream_v) {
  if (!b || !b->render) return fail(NERFB200_EINVAL, "render_backward: NULL argument%s");
  const nerfb200_render_args* a = b->render;
  int rc = check_render_shapes(a);
  if (rc) return rc;
  if (a->n_rays == 0) return 0;
  if (!a->train_workspace || a->test_time) return fail(NERFB200_EINVAL, "render_backward needs the forward's train_workspace, test_time = 0%s");
  const bool fine = a->n_importance > 0;
  if (!b->params_coarse || !b->grads_coarse || (fine && (!b->params_fine || !b->grads_fine)))
    return fail(NERFB200_EINVAL, "render_backward: params / grads tables are NULL%s");
  for (int i = 0; i < kNumParams; ++i)
    if (!b->params_coarse[i] || !b->grads_coarse[i] || (fine && (!b->params_fine[i] || !b->grads_fine[i])))
      return fail(NERFB200_EINVAL, "render_backward: NULL parameter / gradient tensor%s");
  DeviceInfo* d = nullptr;
  rc = device_info(&d);
  if (rc) return rc;
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
    composite_bwd_kernel<<<(L.n_rays + 3) / 4, 128, 0, stream>>>(cp);
    g_launches++;
  }
  return backward_tail(L, params, grads, net, a->rays, a->ray_stride, d, stream, "render_backward launches");
}

int nerfb200_adam_step(int32_t n_tensors, float* const* params, const float* const* grads, float* const* exp_avg,
                       float* const* exp_avg_sq, const int64_t* numel, float lr, float beta1, float beta2, float eps,
                       float weight_decay, int64_t step, void* stream) {
  if (n_tensors < 0 || n_tensors > kAdamMaxTensors) return fail(NERFB200_EINVAL, "adam_step: at most 64 tensors per call%s");
  if (n_tensors == 0) return 0;
  if (!params || !grads || !exp_avg || !exp_avg_sq || !numel || step < 1)
    return fail(NERFB200_EINVAL, "adam_step: NULL argument / step < 1%s");
  AdamParams a;
  int blocks = 0;
  const int rc = fill_adam_table(a, n_tensors, params, grads, exp_avg, exp_avg_sq, numel, nullptr, beta1, beta2, eps,
                                 weight_decay, "adam_step", &blocks);
  if (rc) return rc;
  // in double, rounded once: 1 - b2^t in fp32 cancels at small t (~50 ulps of the update at t = 2..3)
  a.step_size = static_cast<float>(static_cast<double>(lr) / (1.0 - std::pow(static_cast<double>(beta1), static_cast<double>(step))));
  a.bias2_sqrt = static_cast<float>(std::sqrt(1.0 - std::pow(static_cast<double>(beta2), static_cast<double>(step))));
  if (blocks == 0) return 0;
  adam_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "adam_step launch");
  return 0;
}

int nerfb200_adam_step_dev(int32_t n_tensors, float* const* params, const float* const* grads, float* const* exp_avg,
                           float* const* exp_avg_sq, const int64_t* numel, const float* lr_dev,
                           const float* const* steps, float beta1, float beta2, float eps, float weight_decay,
                           void* stream) {
  if (n_tensors < 0 || n_tensors > kAdamMaxTensors) return fail(NERFB200_EINVAL, "adam_step_dev: at most 64 tensors per call%s");
  if (n_tensors == 0) return 0;
  if (!params || !grads || !exp_avg || !exp_avg_sq || !numel || !lr_dev || !steps)
    return fail(NERFB200_EINVAL, "adam_step_dev: NULL argument%s");
  AdamDevParams d;
  AdamParams& a = d.a;
  int blocks = 0;
  const int rc = fill_adam_table(a, n_tensors, params, grads, exp_avg, exp_avg_sq, numel, steps, beta1, beta2, eps,
                                 weight_decay, "adam_step_dev", &blocks);
  if (rc) return rc;
  for (int i = 0; i < n_tensors; ++i) d.step[i] = steps[i];
  a.step_size = a.bias2_sqrt = 0.f;
  d.lr = lr_dev;
  if (blocks == 0) return 0;
  adam_dev_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(d);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "adam_step_dev launch");
  return 0;
}

int nerfb200_check_status(void) {
  DeviceInfo* d = nullptr;
  int rc = device_info(&d);
  if (rc) return rc;
  return check_sticky_status(d);
}


}  // extern "C"

// ---- coloured mesh extraction (extract_color_mesh.py; kernels: mesh_kernels.cuh) --------------------
namespace {

size_t align256(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }

struct U8ToInt {
  __host__ __device__ __forceinline__ int operator()(uint8_t v) const { return v; }
};
using U8It = thrust::transform_iterator<U8ToInt, const uint8_t*, int>;

// grid-stride launches: one wave of 8 CTAs per SM, capped by NERFB200_MAX_CTAS (the results do not depend on it)
int mesh_blocks(long long n) {
  long long b = (n + 255) / 256;
  if (b > 148 * 8) b = 148 * 8;
  const int cap = env_switches().max_ctas;
  if (cap > 0 && b > cap) b = cap;
  return static_cast<int>(b < 1 ? 1 : b);
}

constexpr long long kMcMaxPoints = 400LL * 1000 * 1000;   // keeps 3 P vertices and 5 C triangles in int32

struct McLayout {
  size_t vcnt, vofs, ccnt, cofs, temp, temp_bytes, bytes;
};
McLayout mc_layout(long long P, long long C) {
  size_t t1 = 0, t2 = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, t1, U8It(nullptr, U8ToInt()), static_cast<int*>(nullptr), static_cast<int>(P + 1));
  cub::DeviceScan::ExclusiveSum(nullptr, t2, U8It(nullptr, U8ToInt()), static_cast<int*>(nullptr), static_cast<int>(C + 1));
  McLayout L;
  size_t o = 0;
  L.vcnt = o; o += align256(P + 1);
  L.vofs = o; o += align256((P + 1) * sizeof(int));
  L.ccnt = o; o += align256(C + 1);
  L.cofs = o; o += align256((C + 1) * sizeof(int));
  L.temp = o; L.temp_bytes = t1 > t2 ? t1 : t2; o += align256(L.temp_bytes);
  L.bytes = o;
  return L;
}

int mc_prepare(const float* sigma, int64_t n0, int64_t n1, int64_t n2, double thr, void* ws, size_t bytes, McParams* p,
               McLayout* L, const char* who) {
  if (n0 < 2 || n1 < 2 || n2 < 2) return fail(NERFB200_EINVAL, "%s: every grid dimension must be >= 2", who);
  if (n0 * n1 * n2 > kMcMaxPoints) return fail(NERFB200_EUNSUPPORTED, "%s: grid larger than 4e8 points", who);
  if (!sigma || !ws) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  const long long P = n0 * n1 * n2, C = (n0 - 1) * (n1 - 1) * (n2 - 1);
  *L = mc_layout(P, C);
  if (bytes < L->bytes) return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_mc_workspace_bytes", who);
  char* w = static_cast<char*>(ws);
  p->sigma = sigma; p->n0 = n0; p->n1 = n1; p->n2 = n2; p->thr = thr;
  p->vcnt = reinterpret_cast<uint8_t*>(w + L->vcnt);
  p->vofs = reinterpret_cast<int*>(w + L->vofs);
  p->ccnt = reinterpret_cast<uint8_t*>(w + L->ccnt);
  p->cofs = reinterpret_cast<int*>(w + L->cofs);
  p->vertices = nullptr; p->triangles = nullptr;
  return 0;
}

struct ClusterLayout {
  size_t keys, keys_alt, vals, vals_alt, parent, count, best, tflag, tofs, vflag, vofs, temp, temp_bytes, bytes;
};
int bits_for(long long v) {
  int b = 1;
  while ((1LL << b) < v) ++b;
  return b;
}
ClusterLayout cluster_layout(long long V, long long T) {
  const long long E = 3 * T;
  size_t t1 = 0, t2 = 0, t3 = 0;
  cub::DoubleBuffer<unsigned long long> kb(nullptr, nullptr);
  cub::DoubleBuffer<int> vb(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, t1, kb, vb, static_cast<int>(E), 0, 2 * bits_for(V));
  cub::DeviceScan::ExclusiveSum(nullptr, t2, U8It(nullptr, U8ToInt()), static_cast<int*>(nullptr), static_cast<int>(T + 1));
  cub::DeviceScan::ExclusiveSum(nullptr, t3, U8It(nullptr, U8ToInt()), static_cast<int*>(nullptr), static_cast<int>(V + 1));
  ClusterLayout L;
  size_t o = 0;
  L.keys = o; o += align256(E * 8);
  L.keys_alt = o; o += align256(E * 8);
  L.vals = o; o += align256(E * 4);
  L.vals_alt = o; o += align256(E * 4);
  L.parent = o; o += align256(T * 4);
  L.count = o; o += align256(T * 4);
  L.best = o; o += 256;
  L.tflag = o; o += align256(T + 1);
  L.tofs = o; o += align256((T + 1) * 4);
  L.vflag = o; o += align256(V + 1);
  L.vofs = o; o += align256((V + 1) * 4);
  size_t tb = t1 > t2 ? t1 : t2;
  tb = tb > t3 ? tb : t3;
  L.temp = o; L.temp_bytes = tb; o += align256(tb);
  L.bytes = o;
  return L;
}

int cluster_prepare(const int32_t* tris, int64_t n_tris, int64_t n_verts, void* ws, size_t bytes, ClusterParams* p,
                    ClusterLayout* L, const char* who) {
  if (n_tris < 0 || n_verts < 0 || n_tris > 0x7fffffffLL / 3 || n_verts > 0x7fffffffLL)
    return fail(NERFB200_EINVAL, "%s: bad mesh size", who);
  if (n_tris > 0 && (!tris || !ws)) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  *L = cluster_layout(n_verts, n_tris);
  if (n_tris > 0 && bytes < L->bytes) return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_mesh_cluster_workspace_bytes", who);
  char* w = static_cast<char*>(ws);
  p->tris = tris; p->n_tris = n_tris; p->n_verts = n_verts;
  p->keys = reinterpret_cast<unsigned long long*>(w + L->keys);
  p->vals = reinterpret_cast<int*>(w + L->vals);
  p->parent = reinterpret_cast<int*>(w + L->parent);
  p->count = reinterpret_cast<int*>(w + L->count);
  p->best = reinterpret_cast<unsigned long long*>(w + L->best);
  p->tflag = reinterpret_cast<uint8_t*>(w + L->tflag);
  p->tofs = reinterpret_cast<int*>(w + L->tofs);
  p->vflag = reinterpret_cast<uint8_t*>(w + L->vflag);
  p->vofs = reinterpret_cast<int*>(w + L->vofs);
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

struct VolumeLayout {
  long long tiles;
  size_t tcnt, tofs, temp, temp_bytes, bytes;
};
VolumeLayout volume_layout(long long N) {
  VolumeLayout L;
  L.tiles = (N * N * N + kVolTile - 1) / kVolTile;
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, static_cast<const unsigned long long*>(nullptr),
                                static_cast<unsigned long long*>(nullptr), static_cast<int>(L.tiles + 1));
  size_t o = 0;
  L.tcnt = o; o += align256((L.tiles + 1) * sizeof(unsigned long long));
  L.tofs = o; o += align256((L.tiles + 1) * sizeof(unsigned long long));
  L.temp = o; L.temp_bytes = tb; o += align256(tb);
  L.bytes = o;
  return L;
}

int volume_prepare(const float* rgbsigma, int64_t N, double xmin, double xmax, void* ws, size_t bytes, VolumeParams* p,
                   VolumeLayout* L, const char* who) {
  if (N < 2 || N > kVolMaxN) return fail(NERFB200_EINVAL, "%s: N must be in [2, 1625] (uint32 indices)", who);
  if (!rgbsigma || !ws) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  if (reinterpret_cast<uintptr_t>(rgbsigma) & 15) return fail(NERFB200_EINVAL, "%s: rgbsigma must be 16-byte aligned", who);
  *L = volume_layout(N);
  if (bytes < L->bytes) return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_volume_workspace_bytes", who);
  char* w = static_cast<char*>(ws);
  p->rgbsigma = reinterpret_cast<const float4*>(rgbsigma);
  p->P = N * N * N;
  // -(xmax - xmin) / N is a Python float; numpy rounds it to float32 before the multiply
  p->c = static_cast<float>(-(xmax - xmin) / static_cast<double>(N));
  p->tcnt = reinterpret_cast<unsigned long long*>(w + L->tcnt);
  p->tofs = reinterpret_cast<unsigned long long*>(w + L->tofs);
  p->out = nullptr;
  return 0;
}

// Vertex normals: corner keys / triangle ids (and their sort buffers), triangle normals, the index flag.
struct NormalsLayout {
  size_t keys, keys_alt, vals, vals_alt, tri_n, bad, temp, temp_bytes, bytes;
};
NormalsLayout normals_layout(long long V, long long T) {
  const long long E = 3 * T;
  size_t tb = 0;
  cub::DoubleBuffer<int> kb(nullptr, nullptr), vb(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, tb, kb, vb, static_cast<int>(E), 0, bits_for(V + 1));
  NormalsLayout L;
  size_t o = 0;
  L.keys = o; o += align256(E * 4);
  L.keys_alt = o; o += align256(E * 4);
  L.vals = o; o += align256(E * 4);
  L.vals_alt = o; o += align256(E * 4);
  L.tri_n = o; o += align256(T * 3 * sizeof(double));
  L.bad = o; o += 256;
  L.temp = o; L.temp_bytes = tb; o += align256(tb);
  L.bytes = o;
  return L;
}

// V + 1 (the key of an out-of-range corner) and 3T stay in int32
bool normals_size_ok(long long V, long long T) {
  return V >= 0 && T >= 0 && V < 0x7fffffffLL && T <= 0x7fffffffLL / 3;
}

}  // namespace

extern "C" {

size_t nerfb200_sigma_grid_workspace_bytes(int64_t chunk) {
  return chunk > 0 ? align256(static_cast<size_t>(chunk) * 3 * sizeof(float)) : 0;
}

int nerfb200_grid_positions(int64_t N, const double ranges_host[6], int64_t start, int64_t count, float* xyz,
                            void* stream) {
  if (N < 2 || start < 0 || count < 0 || start + count > N * N * N)
    return fail(NERFB200_EINVAL, "grid_positions: bad N / start / count%s");
  if (count == 0) return 0;
  if (!ranges_host || !xyz) return fail(NERFB200_EINVAL, "grid_positions: NULL argument%s");
  GridParams p;
  for (int a = 0; a < 3; ++a) { p.lo[a] = ranges_host[2 * a]; p.hi[a] = ranges_host[2 * a + 1]; }
  p.N = N; p.start = start; p.count = count; p.xyz = xyz;
  mesh_grid_positions_kernel<<<mesh_blocks(count), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "grid_positions launch");
  return 0;
}

int nerfb200_sigma_grid(const void* packed, int64_t N, const double ranges_host[6], int64_t chunk, void* ws,
                        size_t bytes, float* sigma, void* stream) {
  if (N < 2 || chunk <= 0) return fail(NERFB200_EINVAL, "sigma_grid: N < 2 or chunk <= 0%s");
  if (!packed || !ranges_host || !ws || !sigma) return fail(NERFB200_EINVAL, "sigma_grid: NULL argument%s");
  if (bytes < nerfb200_sigma_grid_workspace_bytes(chunk))
    return fail(NERFB200_EINVAL, "sigma_grid: workspace smaller than nerfb200_sigma_grid_workspace_bytes(chunk)%s");
  float* xyz = static_cast<float*>(ws);
  const long long total = N * N * N;
  for (long long s = 0; s < total; s += chunk) {
    const long long n = total - s < chunk ? total - s : chunk;
    int rc = nerfb200_grid_positions(N, ranges_host, s, n, xyz, stream);
    if (rc) return rc;
    if ((rc = nerfb200_query_sigma(xyz, n, 3, packed, sigma + s, stream)) != 0) return rc;
    mesh_relu_kernel<<<mesh_blocks(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(sigma + s, n);
    g_launches++;
    CUDA_TRY(cudaGetLastError(), "sigma_grid relu launch");
  }
  return 0;
}

int nerfb200_rgb_sigma_grid(const void* packed, int64_t N, const double ranges_host[6], int64_t chunk, void* ws,
                            size_t bytes, float* rgbsigma, void* stream) {
  if (N < 2 || N > kVolMaxN || chunk <= 0) return fail(NERFB200_EINVAL, "rgb_sigma_grid: N not in [2, 1625] or chunk <= 0%s");
  if (!packed || !ranges_host || !ws || !rgbsigma) return fail(NERFB200_EINVAL, "rgb_sigma_grid: NULL argument%s");
  if (reinterpret_cast<uintptr_t>(rgbsigma) & 15) return fail(NERFB200_EINVAL, "rgb_sigma_grid: out must be 16-byte aligned%s");
  if (bytes < nerfb200_sigma_grid_workspace_bytes(chunk))
    return fail(NERFB200_EINVAL, "rgb_sigma_grid: workspace smaller than nerfb200_sigma_grid_workspace_bytes(chunk)%s");
  float* xyz = static_cast<float*>(ws);
  const long long total = N * N * N;
  for (long long s = 0; s < total; s += chunk) {
    const long long n = total - s < chunk ? total - s : chunk;
    int rc = nerfb200_grid_positions(N, ranges_host, s, n, xyz, stream);
    if (rc) return rc;
    if ((rc = nerfb200_query_rgb_sigma(xyz, n, 3, packed, rgbsigma + s * 4, stream)) != 0) return rc;
  }
  return 0;
}

size_t nerfb200_volume_workspace_bytes(int64_t N) {
  if (N < 2 || N > kVolMaxN) return 0;
  return volume_layout(N).bytes;
}

int nerfb200_volume_count(const float* rgbsigma, int64_t N, double xmin, double xmax, void* ws, size_t bytes,
                          int64_t* count_host, void* stream) {
  VolumeParams p;
  VolumeLayout L;
  int rc = volume_prepare(rgbsigma, N, xmin, xmax, ws, bytes, &p, &L, "volume_count");
  if (rc) return rc;
  if (!count_host) return fail(NERFB200_EINVAL, "volume_count: count_host is NULL%s");
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemsetAsync(p.tcnt + L.tiles, 0, sizeof(unsigned long long), s), "volume_count memset");
  volume_count_kernel<<<mesh_blocks(L.tiles * kVolThreads), kVolThreads, 0, s>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "volume_count launch");
  size_t tb = L.temp_bytes;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(static_cast<char*>(ws) + L.temp, tb, p.tcnt, p.tofs,
                                         static_cast<int>(L.tiles + 1), s), "volume scan");
  g_launches++;
  unsigned long long h = 0;
  CUDA_TRY(cudaMemcpyAsync(&h, p.tofs + L.tiles, sizeof(h), cudaMemcpyDeviceToHost, s), "volume_count readback");
  CUDA_TRY(cudaStreamSynchronize(s), "volume_count readback");
  *count_host = static_cast<int64_t>(h);
  return 0;
}

int nerfb200_volume_emit(const float* rgbsigma, int64_t N, double xmin, double xmax, void* ws, size_t bytes,
                         uint32_t* packed_out, void* stream) {
  VolumeParams p;
  VolumeLayout L;
  int rc = volume_prepare(rgbsigma, N, xmin, xmax, ws, bytes, &p, &L, "volume_emit");
  if (rc) return rc;
  if (!packed_out) return fail(NERFB200_EINVAL, "volume_emit: out is NULL%s");
  if (reinterpret_cast<uintptr_t>(packed_out) & 7) return fail(NERFB200_EINVAL, "volume_emit: out must be 8-byte aligned%s");
  p.out = reinterpret_cast<uint2*>(packed_out);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  volume_emit_kernel<<<mesh_blocks(L.tiles * kVolThreads), kVolThreads, 0, s>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "volume_emit launch");
  return 0;
}

size_t nerfb200_mc_workspace_bytes(int64_t n0, int64_t n1, int64_t n2) {
  if (n0 < 2 || n1 < 2 || n2 < 2 || n0 * n1 * n2 > kMcMaxPoints) return 0;
  return mc_layout(n0 * n1 * n2, (n0 - 1) * (n1 - 1) * (n2 - 1)).bytes;
}

int nerfb200_mc_count(const float* sigma, int64_t n0, int64_t n1, int64_t n2, double threshold, void* ws, size_t bytes,
                      int64_t counts_host[2], void* stream) {
  McParams p;
  McLayout L;
  int rc = mc_prepare(sigma, n0, n1, n2, threshold, ws, bytes, &p, &L, "mc_count");
  if (rc) return rc;
  if (!counts_host) return fail(NERFB200_EINVAL, "mc_count: counts_host is NULL%s");
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long P = n0 * n1 * n2, C = (n0 - 1) * (n1 - 1) * (n2 - 1);
  CUDA_TRY(cudaMemsetAsync(p.vcnt + P, 0, 1, s), "mc_count memset");
  CUDA_TRY(cudaMemsetAsync(p.ccnt + C, 0, 1, s), "mc_count memset");
  mc_classify_kernel<<<mesh_blocks(P), 256, 0, s>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "mc_classify launch");
  void* temp = static_cast<char*>(ws) + L.temp;
  size_t tb = L.temp_bytes;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(temp, tb, U8It(p.vcnt, U8ToInt()), p.vofs, static_cast<int>(P + 1), s), "mc vertex scan");
  tb = L.temp_bytes;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(temp, tb, U8It(p.ccnt, U8ToInt()), p.cofs, static_cast<int>(C + 1), s), "mc triangle scan");
  g_launches += 2;
  return read_two_counts(p.vofs + P, p.cofs + C, counts_host, s, "mc_count readback");
}

int nerfb200_mc_emit(const float* sigma, int64_t n0, int64_t n1, int64_t n2, double threshold, void* ws, size_t bytes,
                     double* vertices, int32_t* triangles, void* stream) {
  McParams p;
  McLayout L;
  int rc = mc_prepare(sigma, n0, n1, n2, threshold, ws, bytes, &p, &L, "mc_emit");
  if (rc) return rc;
  p.vertices = vertices;
  p.triangles = triangles;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long P = n0 * n1 * n2, C = (n0 - 1) * (n1 - 1) * (n2 - 1);
  if (vertices) {
    mc_emit_vertices_kernel<<<mesh_blocks(P), 256, 0, s>>>(p);
    g_launches++;
    CUDA_TRY(cudaGetLastError(), "mc_emit_vertices launch");
  }
  if (triangles) {
    mc_emit_triangles_kernel<<<mesh_blocks(C), 256, 0, s>>>(p);
    g_launches++;
    CUDA_TRY(cudaGetLastError(), "mc_emit_triangles launch");
  }
  return 0;
}

int nerfb200_mesh_to_world(const double* vertices, int64_t n, int64_t N, const double ranges_host[6], float* out,
                           void* stream) {
  if (n < 0 || N < 1) return fail(NERFB200_EINVAL, "mesh_to_world: bad n / N%s");
  if (n == 0) return 0;
  if (!vertices || !ranges_host || !out) return fail(NERFB200_EINVAL, "mesh_to_world: NULL argument%s");
  ToWorldParams p;
  p.v = vertices; p.n = n; p.N = static_cast<double>(N); p.out = out;
  // column 0 takes y_range, column 1 x_range (extract_color_mesh.py:150-151)
  const int src[3] = {1, 0, 2};
  for (int c = 0; c < 3; ++c) {
    const double lo = ranges_host[2 * src[c]], hi = ranges_host[2 * src[c] + 1];
    p.scale[c] = static_cast<float>(hi - lo);
    p.offset[c] = static_cast<float>(lo);
  }
  mesh_to_world_kernel<<<mesh_blocks(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "mesh_to_world launch");
  return 0;
}

size_t nerfb200_mesh_cluster_workspace_bytes(int64_t n_vertices, int64_t n_triangles) {
  if (n_vertices < 0 || n_triangles <= 0 || n_triangles > 0x7fffffffLL / 3 || n_vertices > 0x7fffffffLL) return 0;
  return cluster_layout(n_vertices, n_triangles).bytes;
}

int nerfb200_mesh_cluster_count(const int32_t* triangles, int64_t n_tris, int64_t n_verts, void* ws, size_t bytes,
                                int64_t counts_host[2], void* stream) {
  ClusterParams p;
  ClusterLayout L;
  int rc = cluster_prepare(triangles, n_tris, n_verts, ws, bytes, &p, &L, "mesh_cluster_count");
  if (rc) return rc;
  if (!counts_host) return fail(NERFB200_EINVAL, "mesh_cluster_count: counts_host is NULL%s");
  if (n_tris == 0) { counts_host[0] = counts_host[1] = 0; return 0; }
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* w = static_cast<char*>(ws);
  const long long E = 3 * n_tris;
  const int bits = bits_for(n_verts);
  cluster_edges_kernel<<<mesh_blocks(n_tris), 256, 0, s>>>(p);
  cluster_pack_keys_kernel<<<mesh_blocks(E), 256, 0, s>>>(p.keys, E, bits);
  g_launches += 2;
  CUDA_TRY(cudaGetLastError(), "cluster edges launch");
  cub::DoubleBuffer<unsigned long long> kb(p.keys, reinterpret_cast<unsigned long long*>(w + L.keys_alt));
  cub::DoubleBuffer<int> vb(p.vals, reinterpret_cast<int*>(w + L.vals_alt));
  size_t tb = L.temp_bytes;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(w + L.temp, tb, kb, vb, static_cast<int>(E), 0, 2 * bits, s), "cluster edge sort");
  g_launches++;
  p.keys = kb.Current();
  p.vals = vb.Current();
  CUDA_TRY(cudaMemsetAsync(p.best, 0, sizeof(unsigned long long), s), "cluster memset");
  CUDA_TRY(cudaMemsetAsync(p.vflag, 0, n_verts + 1, s), "cluster memset");
  CUDA_TRY(cudaMemsetAsync(p.tflag + n_tris, 0, 1, s), "cluster memset");
  cluster_union_kernel<<<mesh_blocks(E), 256, 0, s>>>(p);
  cluster_label_kernel<<<mesh_blocks(n_tris), 256, 0, s>>>(p);
  cluster_best_kernel<<<mesh_blocks(n_tris), 256, 0, s>>>(p);
  cluster_flag_kernel<<<mesh_blocks(n_tris), 256, 0, s>>>(p);
  g_launches += 4;
  CUDA_TRY(cudaGetLastError(), "cluster union-find launch");
  tb = L.temp_bytes;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(w + L.temp, tb, U8It(p.tflag, U8ToInt()), p.tofs, static_cast<int>(n_tris + 1), s),
           "cluster triangle scan");
  tb = L.temp_bytes;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(w + L.temp, tb, U8It(p.vflag, U8ToInt()), p.vofs, static_cast<int>(n_verts + 1), s),
           "cluster vertex scan");
  g_launches += 2;
  return read_two_counts(p.vofs + n_verts, p.tofs + n_tris, counts_host, s, "mesh_cluster_count readback");
}

int nerfb200_mesh_cluster_emit(const float* vertices, const int32_t* triangles, int64_t n_tris, int64_t n_verts, void* ws,
                               size_t bytes, float* vertices_out, int32_t* triangles_out, void* stream) {
  ClusterParams p;
  ClusterLayout L;
  int rc = cluster_prepare(triangles, n_tris, n_verts, ws, bytes, &p, &L, "mesh_cluster_emit");
  if (rc) return rc;
  if (n_tris == 0) return 0;
  if (!vertices || !vertices_out || !triangles_out) return fail(NERFB200_EINVAL, "mesh_cluster_emit: NULL argument%s");
  p.vin = vertices; p.vout = vertices_out; p.tout = triangles_out;
  const long long n = n_tris > n_verts ? n_tris : n_verts;
  cluster_emit_kernel<<<mesh_blocks(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "mesh_cluster_emit launch");
  return 0;
}

int nerfb200_remap_bilinear(const uint8_t* image, int32_t H, int32_t W, const float* xy, int64_t n, uint8_t* out,
                            void* stream) {
  if (H <= 0 || W <= 0 || n < 0) return fail(NERFB200_EINVAL, "remap_bilinear: bad H / W / n%s");
  if (n == 0) return 0;
  if (!image || !xy || !out) return fail(NERFB200_EINVAL, "remap_bilinear: NULL argument%s");
  remap_bilinear_kernel<<<mesh_blocks(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(image, H, W, xy, n, out);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "remap_bilinear launch");
  return 0;
}

int nerfb200_color_project(const float* vertices, int64_t n, const double w2c_host[12], const float origin_host[3],
                           float focal, int32_t W, int32_t H, const uint8_t* image, float near, uint8_t* colors,
                           double* depth, float* rays, void* stream) {
  if (n < 0 || H <= 0 || W <= 0) return fail(NERFB200_EINVAL, "color_project: bad n / H / W%s");
  if (n == 0) return 0;
  if (!vertices || !w2c_host || !origin_host || !image || !colors || !depth || !rays)
    return fail(NERFB200_EINVAL, "color_project: NULL argument%s");
  ColorProjectParams p;
  p.vertices = vertices; p.n = n;
  for (int i = 0; i < 12; ++i) p.w2c[i] = w2c_host[i];
  for (int i = 0; i < 3; ++i) p.origin[i] = origin_host[i];
  p.focal = focal; p.W = W; p.H = H; p.image = image; p.near = near;
  p.colors = colors; p.depth = depth; p.rays = rays;
  color_project_kernel<<<mesh_blocks(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "color_project launch");
  return 0;
}

int nerfb200_color_accumulate(const uint8_t* colors, const double* depth, const float* opacity, int64_t n,
                              float occ_threshold, double* sum4, void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "color_accumulate: n < 0%s");
  if (n == 0) return 0;
  if (!colors || !depth || !opacity || !sum4) return fail(NERFB200_EINVAL, "color_accumulate: NULL argument%s");
  color_accumulate_kernel<<<mesh_blocks(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(colors, depth, opacity, n,
                                                                                          occ_threshold, sum4);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "color_accumulate launch");
  return 0;
}

int nerfb200_color_finalize(const double* sum4, int64_t n, uint8_t* colors, void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "color_finalize: n < 0%s");
  if (n == 0) return 0;
  if (!sum4 || !colors) return fail(NERFB200_EINVAL, "color_finalize: NULL argument%s");
  color_finalize_kernel<<<mesh_blocks(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(sum4, n, colors);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "color_finalize launch");
  return 0;
}

size_t nerfb200_vertex_normals_workspace_bytes(int64_t n_verts, int64_t n_tris) {
  if (!normals_size_ok(n_verts, n_tris)) return 0;
  return normals_layout(n_verts, n_tris).bytes;
}

int nerfb200_vertex_normals(const float* vertices, int64_t n_verts, const int32_t* triangles, int64_t n_tris, void* ws,
                            size_t bytes, double* normals, void* stream) {
  if (!normals_size_ok(n_verts, n_tris)) return fail(NERFB200_EINVAL, "vertex_normals: bad mesh size%s");
  if (n_verts == 0) {
    if (n_tris == 0) return 0;
    return fail(NERFB200_EINVAL, "vertex_normals: a triangle index is outside [0, n_verts) (n_verts = 0)%s");
  }
  if ((n_verts > 0 && (!vertices || !normals)) || (n_tris > 0 && !triangles) || !ws)
    return fail(NERFB200_EINVAL, "vertex_normals: NULL argument%s");
  const NormalsLayout L = normals_layout(n_verts, n_tris);
  if (bytes < L.bytes) return fail(NERFB200_EINVAL, "vertex_normals: workspace smaller than nerfb200_vertex_normals_workspace_bytes%s");
  char* w = static_cast<char*>(ws);
  NormalsParams p;
  p.vertices = vertices; p.tris = triangles; p.n_verts = n_verts; p.n_tris = n_tris;
  p.keys = reinterpret_cast<int*>(w + L.keys);
  p.vals = reinterpret_cast<int*>(w + L.vals);
  p.tri_n = reinterpret_cast<double*>(w + L.tri_n);
  p.bad = reinterpret_cast<int*>(w + L.bad);
  p.normals = normals;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemsetAsync(p.bad, 0, sizeof(int), s), "vertex_normals memset");
  if (n_tris > 0) {
    normals_triangle_kernel<<<mesh_blocks(n_tris), 256, 0, s>>>(p);
    g_launches++;
    CUDA_TRY(cudaGetLastError(), "vertex_normals triangle launch");
    cub::DoubleBuffer<int> kb(p.keys, reinterpret_cast<int*>(w + L.keys_alt));
    cub::DoubleBuffer<int> vb(p.vals, reinterpret_cast<int*>(w + L.vals_alt));
    size_t tb = L.temp_bytes;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(w + L.temp, tb, kb, vb, static_cast<int>(3 * n_tris), 0,
                                             bits_for(n_verts + 1), s), "vertex_normals corner sort");
    g_launches++;
    p.keys = kb.Current();
    p.vals = vb.Current();
  }
  if (n_verts > 0) {
    normals_vertex_kernel<<<mesh_blocks(n_verts), 256, 0, s>>>(p);
    g_launches++;
    CUDA_TRY(cudaGetLastError(), "vertex_normals vertex launch");
  }
  int bad = 0;
  CUDA_TRY(cudaMemcpyAsync(&bad, p.bad, sizeof(int), cudaMemcpyDeviceToHost, s), "vertex_normals readback");
  CUDA_TRY(cudaStreamSynchronize(s), "vertex_normals readback");
  if (bad) return fail(NERFB200_EINVAL, "vertex_normals: a triangle index is outside [0, n_verts)%s");
  return 0;
}

int nerfb200_normal_rays(const float* vertices, const double* normals, int64_t n, float near, float far, float near_t,
                         float* rays, void* stream) {
  if (n < 0) return fail(NERFB200_EINVAL, "normal_rays: n < 0%s");
  if (n == 0) return 0;
  if (!vertices || !normals || !rays) return fail(NERFB200_EINVAL, "normal_rays: NULL argument%s");
  normal_rays_kernel<<<mesh_blocks(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(vertices, normals, n, near, far,
                                                                                     near_t, rays);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "normal_rays launch");
  return 0;
}

}  // extern "C"

// ---- empty-space skipping (include/nerf_pl_b200_occupancy.h; kernels: occupancy_kernels.cuh) ------------------
namespace {

struct CullLayout {
  long long tiles;
  size_t tcnt, tofs, bytes;
};
CullLayout cull_layout(long long n) {
  CullLayout L;
  L.tiles = (n + kCullTile - 1) / kCullTile;
  size_t o = 0;
  L.tcnt = o; o += align256((L.tiles + 1) * sizeof(int));
  L.tofs = o; o += align256((L.tiles + 1) * sizeof(long long));
  L.bytes = o;
  return L;
}

// one CTA per tile of rays, capped like the other grid-stride launches
int cull_blocks(long long tiles) {
  long long b = tiles < 148 * 8 ? tiles : 148 * 8;
  const int cap = env_switches().max_ctas;
  if (cap > 0 && b > cap) b = cap;
  return static_cast<int>(b < 1 ? 1 : b);
}

int cull_prepare(const float* rays, int64_t n, void* ws, size_t bytes, CullParams* p, CullLayout* L, const char* who) {
  if (n < 0) return fail(NERFB200_EINVAL, "%s: n_rays < 0", who);
  *L = cull_layout(n);
  if (n == 0) return 0;
  if (!rays || !ws) return fail(NERFB200_EINVAL, "%s: NULL argument", who);
  if (reinterpret_cast<uintptr_t>(rays) & 15) return fail(NERFB200_EINVAL, "%s: rays must be 16-byte aligned", who);
  if (bytes < L->bytes) return fail(NERFB200_EINVAL, "%s: workspace smaller than nerfb200_cull_workspace_bytes", who);
  char* w = static_cast<char*>(ws);
  p->rays = rays; p->n = n;
  p->tcnt = reinterpret_cast<int*>(w + L->tcnt);
  p->tofs = reinterpret_cast<long long*>(w + L->tofs);
  p->bits = nullptr; p->flag = nullptr; p->live_idx = nullptr; p->live_rays = nullptr;
  return 0;
}

}  // namespace

extern "C" {

size_t nerfb200_occupancy_workspace_bytes(int64_t N) {
  if (N < 2 || N > kVolMaxN) return 0;
  return 2 * align256(static_cast<size_t>((N - 1) * (N - 1) * (N - 1)));
}

int nerfb200_occupancy_pack(const float* sigma, int64_t N, double sigma_threshold, int32_t dilate, void* ws,
                            size_t bytes, uint32_t* bits, void* stream) {
  if (N < 2 || N > kVolMaxN) return fail(NERFB200_EINVAL, "occupancy_pack: N must be in [2, 1625]%s");
  if (dilate < 0) return fail(NERFB200_EINVAL, "occupancy_pack: dilate < 0%s");
  if (sigma_threshold != sigma_threshold) return fail(NERFB200_EINVAL, "occupancy_pack: sigma_threshold is NaN%s");
  if (!sigma || !ws || !bits) return fail(NERFB200_EINVAL, "occupancy_pack: NULL argument%s");
  if (bytes < nerfb200_occupancy_workspace_bytes(N))
    return fail(NERFB200_EINVAL, "occupancy_pack: workspace smaller than nerfb200_occupancy_workspace_bytes%s");
  const long long M = N - 1, C = M * M * M;
  uint8_t* a = static_cast<uint8_t*>(ws);
  uint8_t* b = a + align256(static_cast<size_t>(C));
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  occ_cells_kernel<<<mesh_blocks(C), 256, 0, s>>>(sigma, N, sigma_threshold, a);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "occupancy cells launch");
  // a radius of M - 1 cells already reaches across the grid
  const int radius = static_cast<int>(dilate < M - 1 ? dilate : M - 1);
  if (radius > 0) {
    const long long stride[3] = {1, M, M * M};
    for (int ax = 0; ax < 3; ++ax) {
      occ_dilate_axis_kernel<<<mesh_blocks(C), 256, 0, s>>>(a, b, M, stride[ax], radius);
      g_launches++;
      CUDA_TRY(cudaGetLastError(), "occupancy dilate launch");
      uint8_t* t = a; a = b; b = t;
    }
  }
  occ_pack_kernel<<<mesh_blocks(C), 256, 0, s>>>(a, C, bits);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "occupancy pack launch");
  return 0;
}

int nerfb200_occupancy_popcount(const uint32_t* bits, int64_t N, int64_t* count, void* stream) {
  if (N < 2 || N > kVolMaxN) return fail(NERFB200_EINVAL, "occupancy_popcount: N must be in [2, 1625]%s");
  if (!bits || !count) return fail(NERFB200_EINVAL, "occupancy_popcount: NULL argument%s");
  const long long C = (N - 1) * (N - 1) * (N - 1), words = (C + 31) / 32;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemsetAsync(count, 0, sizeof(*count), s), "occupancy_popcount memset");
  occ_popcount_kernel<<<mesh_blocks(words), 256, 0, s>>>(bits, words, reinterpret_cast<unsigned long long*>(count));
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "occupancy_popcount launch");
  return 0;
}

size_t nerfb200_cull_workspace_bytes(int64_t n_rays) {
  return n_rays < 0 ? 0 : cull_layout(n_rays).bytes;
}

int nerfb200_cull_count(const float* rays, int64_t n_rays, const uint32_t* bits, int64_t N,
                        const double ranges_host[6], void* ws, size_t bytes, uint8_t* flag, int64_t* n_live_host,
                        void* stream) {
  CullParams p;
  CullLayout L;
  int rc = cull_prepare(rays, n_rays, ws, bytes, &p, &L, "cull_count");
  if (rc) return rc;
  if (N < 2 || N > kVolMaxN) return fail(NERFB200_EINVAL, "cull_count: N must be in [2, 1625]%s");
  if (!n_live_host || !ranges_host) return fail(NERFB200_EINVAL, "cull_count: NULL argument%s");
  for (int a = 0; a < 3; ++a) {
    const double lo = ranges_host[2 * a], hi = ranges_host[2 * a + 1];
    if (!std::isfinite(lo) || !std::isfinite(hi) || lo == hi)
      return fail(NERFB200_EINVAL, "cull_count: every range must be finite with min != max%s");
    p.lo[a] = lo;
    p.scale[a] = static_cast<double>(N - 1) / (hi - lo);
  }
  *n_live_host = 0;
  if (n_rays == 0) return 0;
  if (!bits || !flag) return fail(NERFB200_EINVAL, "cull_count: NULL argument%s");
  p.bits = bits; p.M = N - 1; p.flag = flag;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  cull_classify_kernel<<<cull_blocks(L.tiles), kCullTile, 0, s>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "cull classify launch");
  cull_scan_kernel<<<1, 1024, 0, s>>>(p.tcnt, p.tofs, L.tiles);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "cull scan launch");
  long long h = 0;
  CUDA_TRY(cudaMemcpyAsync(&h, p.tofs + L.tiles, sizeof(h), cudaMemcpyDeviceToHost, s), "cull_count readback");
  CUDA_TRY(cudaStreamSynchronize(s), "cull_count readback");
  *n_live_host = h;
  return 0;
}

int nerfb200_cull_emit(const float* rays, int64_t n_rays, const uint8_t* flag, void* ws, size_t bytes,
                       int64_t* live_idx, float* live_rays, void* stream) {
  CullParams p;
  CullLayout L;
  int rc = cull_prepare(rays, n_rays, ws, bytes, &p, &L, "cull_emit");
  if (rc) return rc;
  if (n_rays == 0) return 0;
  if (!flag || !live_idx || !live_rays) return fail(NERFB200_EINVAL, "cull_emit: NULL argument%s");
  if (reinterpret_cast<uintptr_t>(live_rays) & 15) return fail(NERFB200_EINVAL, "cull_emit: live_rays must be 16-byte aligned%s");
  p.flag = const_cast<uint8_t*>(flag);
  p.live_idx = reinterpret_cast<long long*>(live_idx);
  p.live_rays = live_rays;
  cull_emit_kernel<<<cull_blocks(L.tiles), kCullTile, 0, static_cast<cudaStream_t>(stream)>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "cull emit launch");
  return 0;
}

int nerfb200_scatter_results(const float* const src_host[6], float* const dst_host[6], const int64_t* live_idx,
                             int64_t n_live, int64_t n_rays, int32_t white_back, void* stream) {
  if (n_rays < 0 || n_live < 0 || n_live > n_rays) return fail(NERFB200_EINVAL, "scatter_results: bad n_live / n_rays%s");
  if (!src_host || !dst_host) return fail(NERFB200_EINVAL, "scatter_results: NULL argument%s");
  if (n_rays == 0) return 0;
  if (n_live > 0 && !live_idx) return fail(NERFB200_EINVAL, "scatter_results: live_idx is NULL%s");
  ScatterParams p;
  bool any = false;
  for (int k = 0; k < 6; ++k) {
    if (n_live > 0 && (src_host[k] == nullptr) != (dst_host[k] == nullptr))
      return fail(NERFB200_EINVAL, "scatter_results: a result is NULL on one side only%s");
    p.src[k] = src_host[k]; p.dst[k] = dst_host[k];
    any |= dst_host[k] != nullptr;
  }
  if (!any) return fail(NERFB200_EINVAL, "scatter_results: no result to write%s");
  p.live_idx = reinterpret_cast<const long long*>(live_idx);
  p.n_live = n_live; p.n = n_rays; p.bg = white_back ? 1.f : 0.f;
  scatter_results_kernel<<<mesh_blocks(n_rays), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  g_launches++;
  CUDA_TRY(cudaGetLastError(), "scatter_results launch");
  return 0;
}

}  // extern "C"
