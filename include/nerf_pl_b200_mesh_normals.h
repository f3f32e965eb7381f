/* nerf_pl_b200 — C ABI, coloured mesh extraction: the vertex-normal colouring method.
 *
 * Replaces: extract_color_mesh.py:187-203 and 280-284 (--use_vertex_normal): open3d's
 * mesh.compute_vertex_normals(), the rays built from the normals, and the uint8 colours.  The render itself is
 * nerfb200_render_rays (both networks, test_time = 1, perturb 0, noise 0) on these rays, and the colours are
 * nerfb200_to_uint8 of its rgb_fine, which equals (rgb * 255.0).astype(uint8) for every rgb in [0, 1].
 * Conventions of nerf_pl_b200.h (which includes this header): device pointers unless `_host`, `stream` last,
 * 0 = ok, negative = invalid argument.  Adding these entries changed no struct: NERFB200_ABI_VERSION stays 3.
 * Definitions and provenance: DESIGN.md section 9, "Vertex-normal colours".
 */
#ifndef NERF_PL_B200_MESH_NORMALS_H_
#define NERF_PL_B200_MESH_NORMALS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* :189 mesh.compute_vertex_normals() (open3d TriangleMesh::ComputeVertexNormals, normalized, on a mesh
 * without normals): normals (n_verts, 3) fp64 of fp32 vertices (n_verts, 3) and int32 triangles
 * (n_tris, 3).  Triangle normal (v1 - v0) x (v2 - v0) in fp64; each vertex sums the normals of its
 * triangles in increasing triangle index; then s = (x^2 + y^2) + z^2, each component divided by sqrt(s)
 * when s > 0, and (0, 0, 1) when x is NaN.  Bit for bit, whatever the launch shape.  The workspace is
 * the caller's (0 bytes: unsupported size).  Synchronises `stream`: an index outside [0, n_verts)
 * returns NERFB200_EINVAL, and the normals are then undefined. */
size_t nerfb200_vertex_normals_workspace_bytes(int64_t n_verts, int64_t n_tris);
int nerfb200_vertex_normals(const float* vertices, int64_t n_verts, const int32_t* triangles, int64_t n_tris, void* ws,
                            size_t bytes, double* normals, void* stream);

/* :190-193 and the torch.cat of :200: rays (n, 8) fp32 [v - (d * near) * near_t, d, near, far] with
 * d = float32(normal), each operation in fp32 as torch does it on the CPU; near, far and near_t are the
 * fp32 roundings of the host values (dataset.bounds.min(), .max(), args.near_t). */
int nerfb200_normal_rays(const float* vertices, const double* normals, int64_t n, float near, float far, float near_t,
                         float* rays, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERF_PL_B200_MESH_NORMALS_H_ */
