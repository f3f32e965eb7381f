"""numpy restatement of the vertex-normal colouring method of extract_color_mesh.py (``--use_vertex_normal``,
:187-203): open3d's ``TriangleMesh::ComputeVertexNormals()`` on a mesh without normals, and the ray expression.

open3d (as published), in float64:
- triangle normal ``n_t = (v1 - v0) x (v2 - v0)`` with Eigen's component formula
  ``(a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0)``;
- vertex normals start at zero; the triangles are visited in index order and each adds ``n_t`` to its corners
  v0, v1, v2: every vertex sums its triangles' normals in increasing triangle index (area-weighted);
- ``normalize()``: ``s = (x^2 + y^2) + z^2``, each component divided by ``sqrt(s)`` when ``s > 0``; then a NaN
  x component makes the normal (0, 0, 1).
numpy's elementwise float64 operations round each step, as the definition does (no contraction).
"""
import numpy as np
import torch


def triangle_normals(vertices, triangles) -> np.ndarray:
    v = np.asarray(vertices, np.float64)
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    with np.errstate(all="ignore"):
        a = v[t[:, 1]] - v[t[:, 0]]
        b = v[t[:, 2]] - v[t[:, 0]]
        return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1],
                         a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                         a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def normalize(s3: np.ndarray) -> np.ndarray:
    """Eigen ``normalize()`` per row, then open3d's NaN rule."""
    out = np.array(s3, np.float64, copy=True)
    with np.errstate(all="ignore"):
        sq = (out[:, 0] * out[:, 0] + out[:, 1] * out[:, 1]) + out[:, 2] * out[:, 2]
        pos = sq > 0
        out[pos] = out[pos] / np.sqrt(sq[pos])[:, None]
    out[np.isnan(out[:, 0])] = (0.0, 0.0, 1.0)
    return out


def vertex_sums(n_verts: int, triangles, tri_n) -> np.ndarray:
    """Per vertex, the sum of its corners' triangle normals in corner order (triangle, then v0 v1 v2), added one at a
    time from zero.  Vectorised over vertices: the k-th step adds every vertex's k-th corner."""
    t = np.asarray(triangles, np.int64).reshape(-1)
    out = np.zeros((n_verts, 3), np.float64)
    if t.size == 0:
        return out
    order = np.argsort(t, kind="stable")
    vert, tri = t[order], order // 3
    start = np.searchsorted(vert, np.arange(n_verts))
    deg = np.bincount(vert, minlength=n_verts)
    with np.errstate(all="ignore"):
        for k in range(int(deg.max())):
            sel = np.nonzero(deg > k)[0]
            out[sel] += tri_n[tri[start[sel] + k]]
    return out


def vertex_normals(vertices, triangles) -> np.ndarray:
    """``np.asarray(mesh.compute_vertex_normals().vertex_normals)`` (V, 3) float64."""
    v = np.asarray(vertices, np.float64)
    return normalize(vertex_sums(len(v), triangles, triangle_normals(v, triangles)))


def vertex_normals_loop(vertices, triangles) -> np.ndarray:
    """The same, written as open3d's loop (slow; for small meshes)."""
    v = np.asarray(vertices, np.float64)
    tn = triangle_normals(v, triangles)
    out = np.zeros((len(v), 3), np.float64)
    with np.errstate(all="ignore"):
        for i, tri in enumerate(np.asarray(triangles, np.int64).reshape(-1, 3)):
            for c in range(3):
                out[tri[c]] += tn[i]
    return normalize(out)


def normal_rays_torch(vertices, normals, bounds, near_t=1.0) -> np.ndarray:
    """extract_color_mesh.py:190-193 as the reference runs it on the CPU (``dataset.bounds`` is ``bounds``), with the
    ``torch.cat`` of :200: (V, 8) float32."""
    bounds = np.asarray(bounds)
    rays_d = torch.FloatTensor(np.asarray(normals))
    near = bounds.min() * torch.ones_like(rays_d[:, :1])
    far = bounds.max() * torch.ones_like(rays_d[:, :1])
    rays_o = torch.FloatTensor(np.asarray(vertices, np.float32)) - rays_d * near * near_t
    return torch.cat([rays_o, rays_d, near, far], 1).numpy()


def hand_meshes():
    """name -> (vertices (V, 3) float32, triangles (T, 3) int32, expected normals or None)."""
    s3 = 1 / np.sqrt(3.0)
    out = {}
    out["one_triangle"] = (np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0]]), np.int32([[0, 1, 2]]),
                           np.float64([[0, 0, 1]] * 3))
    # closed tetrahedron, faces wound outwards
    tv = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    tt = np.int32([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    out["tetrahedron"] = (tv, tt, np.float64([[-s3, -s3, -s3], [1, 0, 0], [0, 1, 0], [0, 0, 1]]))
    # unit cube, two outward triangles per face
    cv = np.float32([[(i >> 0) & 1, (i >> 1) & 1, (i >> 2) & 1] for i in range(8)])
    faces = [(0, [0, 4, 6, 2], -1), (0, [1, 3, 7, 5], 1), (1, [0, 1, 5, 4], -1), (1, [2, 6, 7, 3], 1),
             (2, [0, 2, 3, 1], -1), (2, [4, 5, 7, 6], 1)]
    ct, exp = [], np.zeros((8, 3))
    for axis, (a, b, c, d), sgn in faces:
        for tri in ([a, b, c], [a, c, d]):
            ct.append(tri)
            for k in tri:
                exp[k, axis] += sgn
    out["cube"] = (cv, np.int32(ct), exp / np.linalg.norm(exp, axis=1, keepdims=True))
    # degenerate (collinear) triangle, an isolated vertex, two opposite copies of one triangle
    out["degenerate_isolated_cancelling"] = (
        np.float32([[0, 0, 0], [1, 1, 1], [2, 2, 2], [5, 5, 5], [0, 0, 3], [1, 0, 3], [0, 1, 3]]),
        np.int32([[0, 1, 2], [4, 5, 6], [4, 6, 5]]),
        np.zeros((7, 3)))
    # non-finite coordinates: a NaN or inf y makes x NaN, so vertices 0-3 become (0, 0, 1); vertex 4 touches nothing;
    # an inf x gives the normal (0, NaN, inf), whose finite x keeps it as it is (only component 0 is tested)
    out["non_finite"] = (
        np.float32([[0, 0, 0], [0, np.nan, 0], [0, 1, 0], [0, np.inf, 0], [1, 2, 3], [0, 0, 5], [np.inf, 0, 5],
                    [0, 1, 5]]),
        np.int32([[0, 1, 2], [0, 3, 2], [5, 6, 7]]),
        np.float64([[0, 0, 1]] * 4 + [[0, 0, 0]] + [[0, np.nan, np.inf]] * 3))
    out["order"] = order_mesh()
    return out


def order_mesh():
    """Vertex 0 gets x contributions +1, +2^-60 (as corner v1 of triangles 0 and 1) and -1 (as corner v0 of triangle
    2), and y +1 (corner v0 of triangle 3).  In triangle order x is (1 + 2^-60) - 1 = 0; summed column by column
    (corner v0 of every triangle first, as ``np.add.at`` per column does) it is (-1 + 1) + 2^-60 = 2^-60."""
    e = 2.0 ** -60
    v = np.float32([[0, 0, 0], [0, 1, 0], [0, 0, 1], [0, e, 0], [0, 0, 1], [0, 0, 1], [1, 0, 0]])
    t = np.int32([[2, 0, 1], [4, 0, 3], [0, 2, 1], [0, 5, 6]])
    return v, t, None


def same_bits(a, b) -> bool:
    """Equal float64 arrays bit for bit, with every NaN counted equal (NaN payloads and signs are not part of the
    definition, and differ between CPUs and GPUs)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb_ = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb_) and np.array_equal(a[~na].view(np.uint64), b[~nb_].view(np.uint64)))


def vertex_normals_column_order(vertices, triangles) -> np.ndarray:
    """The order open3d does NOT use: every triangle's corner v0 first, then v1, then v2."""
    v = np.asarray(vertices, np.float64)
    t = np.asarray(triangles, np.int64)
    tn = triangle_normals(v, t)
    out = np.zeros((len(v), 3))
    for c in range(3):
        np.add.at(out, t[:, c], tn)
    return normalize(out)
