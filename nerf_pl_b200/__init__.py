"""nerf_pl_b200 — H100-native (sm_90a) implementation of the volumetric-rendering hot path of
kwea123/nerf_pl: ``render_rays`` + ``Embedding`` / ``NeRF`` behind the reference's own Python
signatures, executed by hand-written wgmma (sm_90a) CUDA kernels through a C-ABI library
(``include/nerf_pl_b200.h``).  See DESIGN.md and INTEGRATION.md."""
from .nerf import (Embedding, NeRF, invalidate_packed, nerf_forward_fused, nerf_forward_torch, nerf_parameters,
                   packed_weights)
from .culling import (OccupancyGrid, cull_rays, level_ranges, occupancy_cascade, occupancy_grid, pack_occupancy,
                      render_rays_culled, scatter_results)
from .baked import BakedVolume, bake_volume, render_baked
from .data import DeviceRayBatches, DeviceViewBatches
from .density_grid import DensityGrid
from .inference import batched_inference, generate_rays, mse_psnr, query_sigma, render_image, to_uint8
from .mesh import (extract_mesh, fuse_vertex_colors, marching_cubes, normal_rays, normal_vertex_colors, pack_volume,
                   sparse_marching_cubes,
                   query_rgb_sh, query_rgb_sigma, rgb_sigma_grid, sigma_grid, vertex_normals, write_ply, write_vol)
from .metrics import ssim, visualize_depth
from .optim import FusedAdam
from .rendering import render_rays, render_rays_host, render_rays_loss, sample_pdf, searchsorted, volume_render
from .training import CapturedTrainStep, nerf_forward_train
from .views import Views, read_blender_views, read_llff_views

__all__ = [
    "Embedding", "NeRF", "render_rays", "render_rays_loss", "render_rays_host", "FusedAdam", "invalidate_packed", "sample_pdf", "searchsorted", "volume_render",
    "nerf_forward_fused", "nerf_forward_torch", "nerf_forward_train", "nerf_parameters", "packed_weights",
    "batched_inference", "generate_rays", "render_image", "to_uint8", "query_sigma", "mse_psnr",
    "sigma_grid", "marching_cubes", "sparse_marching_cubes", "extract_mesh", "fuse_vertex_colors", "write_ply",
    "query_rgb_sigma", "query_rgb_sh", "rgb_sigma_grid", "pack_volume", "write_vol", "DeviceRayBatches", "CapturedTrainStep",
    "vertex_normals", "normal_rays", "normal_vertex_colors",
    "OccupancyGrid", "occupancy_grid", "pack_occupancy", "cull_rays", "scatter_results", "render_rays_culled",
    "level_ranges", "occupancy_cascade",
    "BakedVolume", "bake_volume", "render_baked",
    "DensityGrid",
    "ssim", "visualize_depth",
    "DeviceViewBatches", "Views", "read_blender_views", "read_llff_views",
]
__version__ = "0.1.0"
