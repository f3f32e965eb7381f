"""Build and load ``libnerf_pl_b200.so`` (the C-ABI library, ``include/nerf_pl_b200.h``).

The library is compiled in-tree with plain ``nvcc`` (no torch headers) so it builds in seconds,
ships to the GPU box with the repository snapshot and shows up as a loaded in-tree ``.so``.
There is no CPU fallback: if the library is missing or cannot be loaded every operator in this
package raises.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import threading
from ctypes import POINTER, c_char_p, c_double, c_float, c_int32, c_int64, c_size_t, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(_HERE, "libnerf_pl_b200.so")
if os.environ.get("NERFB200_LIB"):          # a library built elsewhere (e.g. with extra -D flags); unset in production
    LIB_PATH = os.path.abspath(os.environ["NERFB200_LIB"])
SOURCES = ["capi.cu"]
HEADERS = ["ptx.cuh", "layout.h", "mlp_engine.cuh", "render_kernel.cuh", "aux_kernels.cuh", "bwd_kernels.cuh",
           "mesh_kernels.cuh", "mc_table.h", "occupancy_kernels.cuh", "metrics_kernels.cuh", "jet_lut.h", "sample_skip_kernels.cuh",
           "train_skip_kernels.cuh", "density_kernels.cuh", "masked_grid_kernels.cuh", "early_stop_kernels.cuh",
           "sparse_mc_kernels.cuh", "baked_kernels.cuh"]
INCLUDES = ["nerf_pl_b200.h"]
# the entries of the sparse marching cubes, declared in their own header (SPARSE_MC_SIGNATURES)
SPARSE_MC_INCLUDE = "nerf_pl_b200_sparse_mc.h"
# the entries of the baked volumes, declared in their own header (BAKED_SIGNATURES)
BAKED_INCLUDE = "nerf_pl_b200_baked.h"
# the entries of the view-dependent baked volumes, declared in their own header (BAKED_SH_SIGNATURES)
BAKED_SH_INCLUDE = "nerf_pl_b200_baked_sh.h"
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--shared", "-Xcompiler", "-fPIC",
    "-diag-suppress", "550",
]

ABI_VERSION = 3


class RenderArgs(ctypes.Structure):
    """Mirror of ``nerfb200_render_args`` (include/nerf_pl_b200.h)."""

    _fields_ = [
        ("rays", c_void_p),
        ("n_rays", c_int64),
        ("ray_stride", c_int64),
        ("packed_coarse", c_void_p),
        ("packed_fine", c_void_p),
        ("n_samples", c_int32),
        ("n_importance", c_int32),
        ("use_disp", c_int32),
        ("perturb", c_float),
        ("noise_std", c_float),
        ("white_back", c_int32),
        ("test_time", c_int32),
        ("perturb_rand", c_void_p),
        ("noise_coarse", c_void_p),
        ("u_rand", c_void_p),
        ("noise_fine", c_void_p),
        ("rgb_coarse", c_void_p),
        ("depth_coarse", c_void_p),
        ("opacity_coarse", c_void_p),
        ("rgb_fine", c_void_p),
        ("depth_fine", c_void_p),
        ("opacity_fine", c_void_p),
        ("z_fine", c_void_p),
        ("weights_coarse", c_void_p),
        ("weights_fine", c_void_p),
        ("status", c_void_p),
        ("max_ctas", c_int32),
        ("z_coarse", c_void_p),
        ("train_workspace", c_void_p),
        ("target", c_void_p),
        ("loss_out", c_void_p),
        ("rng_seed", ctypes.c_uint64),          # with rng_in_kernel == 2: the device address of the seed (rng_seed_dev)
        ("rng_in_kernel", c_int32),
    ]


class BackwardArgs(ctypes.Structure):
    """Mirror of ``nerfb200_backward_args`` (include/nerf_pl_b200.h)."""

    _fields_ = [
        ("render", POINTER(RenderArgs)),
        ("params_coarse", POINTER(c_void_p)),
        ("params_fine", POINTER(c_void_p)),
        ("g_rgb_coarse", c_void_p),
        ("g_depth_coarse", c_void_p),
        ("g_opacity_coarse", c_void_p),
        ("g_rgb_fine", c_void_p),
        ("g_depth_fine", c_void_p),
        ("g_opacity_fine", c_void_p),
        ("target", c_void_p),
        ("loss_grad", c_void_p),
        ("grads_coarse", POINTER(c_void_p)),
        ("grads_fine", POINTER(c_void_p)),
    ]


class SamplesArgs(ctypes.Structure):
    """Mirror of ``nerfb200_samples_args`` (include/nerf_pl_b200.h)."""

    _fields_ = [
        ("rays", c_void_p),
        ("n_rays", c_int64),
        ("live_flag", c_void_p),
        ("packed_coarse", c_void_p),
        ("packed_fine", c_void_p),
        ("n_samples", c_int32),
        ("n_importance", c_int32),
        ("use_disp", c_int32),
        ("white_back", c_int32),
        ("test_time", c_int32),
        ("bits", c_void_p),
        ("N", c_int64),
        ("ranges", c_double * 6),
        ("rgb_coarse", c_void_p),
        ("depth_coarse", c_void_p),
        ("opacity_coarse", c_void_p),
        ("rgb_fine", c_void_p),
        ("depth_fine", c_void_p),
        ("opacity_fine", c_void_p),
        ("z_fine", c_void_p),
        ("weights_coarse", c_void_p),
        ("weights_fine", c_void_p),
        ("samples_coarse", c_void_p),
        ("samples_fine", c_void_p),
        ("mask_coarse", c_void_p),
        ("mask_fine", c_void_p),
        ("perturb", c_float),
        ("noise_std", c_float),
        ("perturb_rand", c_void_p),
        ("noise_coarse", c_void_p),
        ("u_rand", c_void_p),
        ("noise_fine", c_void_p),
        ("rng_seed", ctypes.c_uint64),
        ("rng_in_kernel", c_int32),
        ("rng_ray_offset", c_int64),
        ("early_stop", c_float),
        ("cut_coarse", c_void_p),
        ("levels", c_int32),                    # cascade levels of the occupancy grid; 0 means 1
    ]


class TrainSamplesArgs(ctypes.Structure):
    """Mirror of ``nerfb200_train_samples_args`` (include/nerf_pl_b200.h)."""

    _fields_ = [
        ("rays", c_void_p),
        ("n_rays", c_int64),
        ("packed_coarse", c_void_p),
        ("packed_fine", c_void_p),
        ("n_samples", c_int32),
        ("n_importance", c_int32),
        ("use_disp", c_int32),
        ("white_back", c_int32),
        ("perturb", c_float),
        ("noise_std", c_float),
        ("perturb_rand", c_void_p),
        ("noise_coarse", c_void_p),
        ("u_rand", c_void_p),
        ("noise_fine", c_void_p),
        ("rng_seed", ctypes.c_uint64),
        ("rng_in_kernel", c_int32),
        ("bits", c_void_p),
        ("N", c_int64),
        ("ranges", c_double * 6),
        ("target", c_void_p),
        ("rgb_coarse", c_void_p),
        ("depth_coarse", c_void_p),
        ("opacity_coarse", c_void_p),
        ("rgb_fine", c_void_p),
        ("depth_fine", c_void_p),
        ("opacity_fine", c_void_p),
        ("loss_out", c_void_p),
        ("z_coarse", c_void_p),
        ("z_fine", c_void_p),
        ("weights_coarse", c_void_p),
        ("weights_fine", c_void_p),
        ("samples_coarse", c_void_p),
        ("samples_fine", c_void_p),
        ("mask_coarse", c_void_p),
        ("mask_fine", c_void_p),
        ("dsigma_coarse", c_void_p),
        ("dsigma_fine", c_void_p),
        ("dprergb_coarse", c_void_p),
        ("dprergb_fine", c_void_p),
        ("g_rgb_coarse", c_void_p),
        ("g_depth_coarse", c_void_p),
        ("g_opacity_coarse", c_void_p),
        ("g_rgb_fine", c_void_p),
        ("g_depth_fine", c_void_p),
        ("g_opacity_fine", c_void_p),
        ("levels", c_int32),
    ]


_vp, _i32, _i64, _f32, _f64, _sz = c_void_p, c_int32, c_int64, c_float, c_double, c_size_t
_P, _RA, _BA = POINTER(c_void_p), POINTER(RenderArgs), POINTER(BackwardArgs)
_SA, _TA = POINTER(SamplesArgs), POINTER(TrainSamplesArgs)

# Every entry include/nerf_pl_b200.h declares, in header order: name -> (restype, argtypes); tests check it against
# the header's prototypes.  Pointers and arrays are c_void_p or POINTER(...).  The entries that take a stream take it
# last; ``call`` appends it.
SIGNATURES = {
    "nerfb200_abi_version": (_i32, []),
    "nerfb200_last_error": (c_char_p, []),
    "nerfb200_packed_bytes": (_sz, []),
    "nerfb200_pack_weights": (_i32, [_P, _vp, _vp]),
    "nerfb200_pack_weights_pair": (_i32, [_P, _vp, _P, _vp, _vp]),
    "nerfb200_render_rays": (_i32, [_RA, _vp]),
    "nerfb200_train_workspace_bytes": (_sz, [_i64, _i32, _i32]),
    "nerfb200_train_workspace_init": (_i32, [_vp, _sz, _i64, _i32, _i32, _vp]),
    "nerfb200_render_backward": (_i32, [_BA, _vp]),
    "nerfb200_adam_step": (_i32, [_i32, _P, _P, _P, _P, POINTER(_i64), _f32, _f32, _f32, _f32, _f32, _i64, _vp]),
    "nerfb200_adam_step_dev": (_i32, [_i32, _P, _P, _P, _P, POINTER(_i64), _vp, _P, _f32, _f32, _f32, _f32, _vp]),
    "nerfb200_render_rays_host": (_i32, [_RA, _vp]),
    "nerfb200_nerf_forward": (_i32, [_vp, _i64, _i64, _vp, _i32, _vp, _vp]),
    "nerfb200_nerf_train_workspace_bytes": (_sz, [_i64]),
    "nerfb200_nerf_train_workspace_init": (_i32, [_vp, _sz, _i64, _vp]),
    "nerfb200_nerf_forward_train": (_i32, [_vp, _i64, _i64, _vp, _vp, _vp, _vp]),
    "nerfb200_nerf_backward": (_i32, [_vp, _i64, _vp, _P, _vp, _P, _vp]),
    "nerfb200_query_sigma": (_i32, [_vp, _i64, _i64, _vp, _vp, _vp]),
    "nerfb200_mse_psnr": (_i32, [_vp, _vp, _vp, _i64, _vp, _vp]),
    "nerfb200_embed": (_i32, [_vp, _i64, _i32, _vp, _vp]),
    "nerfb200_searchsorted": (_i32, [_vp, _vp, _vp, _i64, _i64, _i32, _i32, _i32, _vp]),
    "nerfb200_sample_pdf": (_i32, [_vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp]),
    "nerfb200_composite": (_i32, [_vp, _vp, _vp, _vp, _vp, _f32, _i32, _i64, _i32, _vp, _vp, _vp, _vp, _vp]),
    "nerfb200_generate_rays": (_i32, [_i32, _i32, _f32, POINTER(_f32), _f32, _f32, _i32, _vp, _vp]),
    "nerfb200_to_uint8": (_i32, [_vp, _i64, _vp, _vp]),
    "nerfb200_grid_positions": (_i32, [_i64, POINTER(_f64), _i64, _i64, _vp, _vp]),
    "nerfb200_sigma_grid_workspace_bytes": (_sz, [_i64]),
    "nerfb200_sigma_grid": (_i32, [_vp, _i64, POINTER(_f64), _i64, _vp, _sz, _vp, _vp]),
    "nerfb200_query_rgb_sigma": (_i32, [_vp, _i64, _i64, _vp, _vp, _vp]),
    "nerfb200_rgb_sigma_grid": (_i32, [_vp, _i64, POINTER(_f64), _i64, _vp, _sz, _vp, _vp]),
    "nerfb200_volume_workspace_bytes": (_sz, [_i64]),
    "nerfb200_volume_count": (_i32, [_vp, _i64, _f64, _f64, _vp, _sz, POINTER(_i64), _vp]),
    "nerfb200_volume_emit": (_i32, [_vp, _i64, _f64, _f64, _vp, _sz, _vp, _vp]),
    "nerfb200_mc_workspace_bytes": (_sz, [_i64, _i64, _i64]),
    "nerfb200_mc_count": (_i32, [_vp, _i64, _i64, _i64, _f64, _vp, _sz, POINTER(_i64), _vp]),
    "nerfb200_mc_emit": (_i32, [_vp, _i64, _i64, _i64, _f64, _vp, _sz, _vp, _vp, _vp]),
    "nerfb200_mesh_to_world": (_i32, [_vp, _i64, _i64, POINTER(_f64), _vp, _vp]),
    "nerfb200_mesh_cluster_workspace_bytes": (_sz, [_i64, _i64]),
    "nerfb200_mesh_cluster_count": (_i32, [_vp, _i64, _i64, _vp, _sz, POINTER(_i64), _vp]),
    "nerfb200_mesh_cluster_emit": (_i32, [_vp, _vp, _i64, _i64, _vp, _sz, _vp, _vp, _vp]),
    "nerfb200_remap_bilinear": (_i32, [_vp, _i32, _i32, _vp, _i64, _vp, _vp]),
    "nerfb200_color_project": (_i32, [_vp, _i64, POINTER(_f64), POINTER(_f32), _f32, _i32, _i32, _vp, _f32, _vp, _vp,
                                      _vp, _vp]),
    "nerfb200_color_accumulate": (_i32, [_vp, _vp, _vp, _i64, _f32, _vp, _vp]),
    "nerfb200_color_finalize": (_i32, [_vp, _i64, _vp, _vp]),
    "nerfb200_vertex_normals_workspace_bytes": (_sz, [_i64, _i64]),
    "nerfb200_vertex_normals": (_i32, [_vp, _i64, _vp, _i64, _vp, _sz, _vp, _vp]),
    "nerfb200_normal_rays": (_i32, [_vp, _vp, _i64, _f32, _f32, _f32, _vp, _vp]),
    "nerfb200_occupancy_workspace_bytes": (_sz, [_i64]),
    "nerfb200_occupancy_pack": (_i32, [_vp, _i64, _f64, _i32, _vp, _sz, _vp, _vp]),
    "nerfb200_occupancy_popcount": (_i32, [_vp, _i64, _vp, _vp]),
    "nerfb200_cull_workspace_bytes": (_sz, [_i64]),
    "nerfb200_cull_count": (_i32, [_vp, _i64, _vp, _i64, POINTER(_f64), _vp, _sz, _vp, POINTER(_i64), _vp]),
    "nerfb200_cull_emit": (_i32, [_vp, _i64, _vp, _vp, _sz, _vp, _vp, _vp]),
    "nerfb200_scatter_results": (_i32, [_P, _P, _vp, _i64, _i64, _i32, _vp]),
    "nerfb200_launch_count": (_i64, []),
    "nerfb200_check_status": (_i32, []),
    "nerfb200_sm_count": (_i32, []),
    # image metrics
    "nerfb200_ssim_workspace_bytes": (_sz, [_i64, _i64, _i64, _i64]),
    "nerfb200_ssim": (_i32, [_vp, POINTER(_i64), _vp, POINTER(_i64), _i64, _i64, _i64, _i64, _i32, _vp, _sz, _vp, _vp]),
    "nerfb200_visualize_depth_workspace_bytes": (_sz, [_i64, _i64]),
    "nerfb200_visualize_depth": (_i32, [_vp, _i64, _i64, _i64, _i64, _vp, _sz, _vp, _vp]),
    # training batches from the views
    "nerfb200_view_batch": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _f32, _f32, _f32, _i32, _vp, _i64, _vp, _vp,
                                   _vp]),
    # rendering with empty samples skipped
    "nerfb200_samples_workspace_bytes": (_sz, [_i64, _i32, _i32]),
    "nerfb200_render_samples": (_i32, [_SA, _vp, _sz, POINTER(_i64), _vp]),
    # the training step with empty samples skipped
    "nerfb200_train_samples_workspace_bytes": (_sz, [_i64, _i32, _i32]),
    "nerfb200_train_samples_forward": (_i32, [_TA, _vp, _sz, POINTER(_i64), _vp]),
    "nerfb200_train_samples_forward_dev": (_i32, [_TA, _vp, _sz, POINTER(_i64), _vp]),
    "nerfb200_train_samples_backward": (_i32, [_TA, _vp, _sz, POINTER(_i64), _vp, _P, _P, _P, _P, _vp]),
    "nerfb200_train_samples_backward_dev": (_i32, [_TA, _vp, _sz, _vp, _P, _P, _P, _P, _vp]),
    # the density grid
    "nerfb200_density_workspace_bytes": (_sz, [_i64, _i64]),
    "nerfb200_density_points": (_i32, [_i64, POINTER(_f64), _vp, _i64, _i64, _vp, _vp]),
    "nerfb200_density_update": (_i32, [_vp, _i64, POINTER(_f64), _f64, _f32, _i32, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
    # grids through an occupancy grid
    "nerfb200_masked_grid_workspace_bytes": (_sz, [_i64]),
    "nerfb200_sigma_grid_masked": (_i32, [_vp, _i64, POINTER(_f64), _vp, _i64, POINTER(_f64), _i64, _vp, _sz, _vp,
                                          POINTER(_i64), _vp]),
    "nerfb200_rgb_sigma_grid_masked": (_i32, [_vp, _i64, POINTER(_f64), _vp, _i64, POINTER(_f64), _i64, _vp, _sz, _vp,
                                              POINTER(_i64), _vp]),
}
EXPORTS = tuple(SIGNATURES)     # tests check the library exports all of them

# Every entry include/nerf_pl_b200_sparse_mc.h declares, in header order, as SIGNATURES.
SPARSE_MC_SIGNATURES = {
    "nerfb200_sparse_mc_plan_workspace_bytes": (_sz, [_i64]),
    "nerfb200_sparse_mc_plan": (_i32, [_i64, POINTER(_f64), _vp, _i64, POINTER(_f64), _vp, _sz, POINTER(_i64), _vp]),
    "nerfb200_sparse_mc_workspace_bytes": (_sz, [_i64, _i64, _i64]),
    "nerfb200_sparse_mc_count": (_i32, [_vp, _i64, POINTER(_f64), _vp, _i64, POINTER(_f64), _f64, _vp, _sz,
                                        POINTER(_i64), _vp, _sz, POINTER(_i64), _vp]),
    "nerfb200_sparse_mc_emit_workspace_bytes": (_sz, [_i64, _i64]),
    "nerfb200_sparse_mc_emit": (_i32, [_i64, _f64, _vp, _sz, POINTER(_i64), _vp, _sz, POINTER(_i64), _vp, _sz, _vp,
                                       _vp, _vp]),
}

# Every entry include/nerf_pl_b200_baked.h declares, in header order, as SIGNATURES.
BAKED_SIGNATURES = {
    "nerfb200_baked_bytes": (_sz, [_i64, _i64]),
    "nerfb200_baked_workspace_bytes": (_sz, [_i64, _i64, _i64]),
    "nerfb200_baked_bake": (_i32, [_vp, _i64, POINTER(_f64), _vp, _i64, POINTER(_f64), _vp, _sz, POINTER(_i64), _vp, _sz,
                                   _vp, _sz, _vp]),
    "nerfb200_baked_from_grid_count": (_i32, [_vp, _i64, _vp, _sz, POINTER(_i64), _vp]),
    "nerfb200_baked_from_grid": (_i32, [_vp, _i64, _vp, _sz, _i64, _vp, _sz, _vp]),
    "nerfb200_baked_to_dense": (_i32, [_vp, _sz, _i64, _i64, _vp, _vp]),
    "nerfb200_baked_render": (_i32, [_vp, _sz, _i64, POINTER(_f64), _i64, _vp, _i64, _f64, _i32, _f64, _vp, _vp, _vp,
                                     _vp]),
}

# Every entry include/nerf_pl_b200_baked_sh.h declares, in header order, as SIGNATURES.
BAKED_SH_SIGNATURES = {
    "nerfb200_baked_sh_bytes": (_sz, [_i64, _i64]),
    "nerfb200_baked_sh_workspace_bytes": (_sz, [_i64, _i64, _i64]),
    "nerfb200_baked_sh_bake": (_i32, [_vp, _i64, POINTER(_f64), _vp, _i64, POINTER(_f64), _vp, _sz, POINTER(_i64), _vp,
                                      _sz, _vp, _sz, _vp]),
    "nerfb200_baked_sh_from_grid_count": (_i32, [_vp, _i64, _vp, _sz, POINTER(_i64), _vp]),
    "nerfb200_baked_sh_from_grid": (_i32, [_vp, _i64, _vp, _sz, _i64, _vp, _sz, _vp]),
    "nerfb200_baked_sh_to_dense": (_i32, [_vp, _sz, _i64, _i64, _vp, _vp]),
    "nerfb200_baked_sh_render": (_i32, [_vp, _sz, _i64, POINTER(_f64), _i64, _vp, _i64, _f64, _i32, _f64, _vp, _vp,
                                        _vp, _vp]),
    "nerfb200_query_rgb_sh_workspace_bytes": (_sz, []),
    "nerfb200_query_rgb_sh": (_i32, [_vp, _i64, _i64, _vp, _vp, _sz, _vp, _vp]),
    "nerfb200_sh_fit_host": (_i32, [POINTER(_f32), POINTER(_f32)]),
}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS]
    deps += [os.path.join(_HERE, "..", "include", f) for f in INCLUDES + [SPARSE_MC_INCLUDE, BAKED_INCLUDE, BAKED_SH_INCLUDE]]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile the CUDA library for sm_90a (cross-compiles without a GPU)."""
    if not force and not needs_build():
        return LIB_PATH
    cmd = [_nvcc(), *NVCC_FLAGS, "-o", LIB_PATH] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    if verbose:
        print(proc.stderr)
    return LIB_PATH


_lib = None
_lock = threading.Lock()


def load() -> ctypes.CDLL:
    """Load the library (never builds implicitly: build() is the explicit step)."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(
                    f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                    "(nerf_pl_b200 has no CPU fallback)")
            lib = ctypes.CDLL(LIB_PATH)
            for name, (restype, argtypes) in {**SIGNATURES, **SPARSE_MC_SIGNATURES, **BAKED_SIGNATURES, **BAKED_SH_SIGNATURES}.items():
                fn = getattr(lib, name)
                fn.restype, fn.argtypes = restype, argtypes
            if lib.nerfb200_abi_version() != ABI_VERSION:
                raise RuntimeError("libnerf_pl_b200.so ABI version mismatch")
            _lib = lib
    return _lib


class NerfB200Error(RuntimeError):
    pass


def check(rc: int, what: str) -> None:
    """Map the C-ABI return code to the Python exceptions the reference raises
    (asserts / Exception in searchsorted.py:23-45, RuntimeError from AT_ASSERTM)."""
    if rc == 0:
        return
    msg = load().nerfb200_last_error().decode("utf-8", "replace")
    if rc in (-1, -2):
        raise ValueError(f"{what}: {msg}")
    raise NerfB200Error(f"{what}: {msg} (code {rc})")


def _stream_ptr() -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def call(name: str, device, *args) -> None:
    """Call the stream-taking entry ``name`` with ``args`` and the current stream of ``device`` appended, and raise
    what ``check`` raises for its return code.  ``device`` is made current for the call unless it already is; None,
    or a device without an index, means the current device."""
    fn = getattr(load(), name)
    if device is None or device.index is None or device.index == torch.cuda.current_device():
        rc = fn(*args, _stream_ptr())
    else:
        with torch.cuda.device(device):
            rc = fn(*args, _stream_ptr())
    check(rc, name)


def workspace(nbytes: int, device) -> torch.Tensor:
    """Scratch of ``nbytes`` bytes (a *_workspace_bytes entry's answer) on ``device``; at least one byte, so that the
    entries always see a non-NULL pointer."""
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


def grid_n(N: int, levels: int = 1) -> int:
    """The grid size argument of the occupancy, culling, density and masked-grid entries (NERFB200_GRID_N): N points
    per axis in the low 32 bits and ``levels - 1`` above them; ``N`` itself for one level."""
    return int(N) + (int(levels) - 1) * (1 << 32)


def ranges_host(x_range, y_range, z_range):
    """The ``ranges_host`` argument of the grid entries: {xmin, xmax, ymin, ymax, zmin, zmax} as 6 host doubles."""
    vals = [float(v) for r in (x_range, y_range, z_range) for v in r]
    if len(vals) != 6:
        raise ValueError("x_range, y_range and z_range must each be (min, max)")
    return (c_double * 6)(*vals)
