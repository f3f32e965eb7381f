"""Write tests/golden/vertex_normal_colors.part*.npz: the vertex-normal colours of extract_color_mesh.py
(``--use_vertex_normal``, :187-203 and :280-284), by the UNMODIFIED reference on the CPU.

The mesh: the reference's ``models.nerf`` NeRF with the trained fine weights gives the sigma grid of :113-140
(N_grid 40 over [-1.5, 1.5]^3); marching cubes (threshold 20), the index -> world transform and the largest-cluster
filter are oracle/mesh_oracle.py's.  The code under test is the reference's own source, parsed with ``ast`` (importing
the script would pull in open3d, mcubes and plyfile): its ``f`` and the ``if args.use_vertex_normal:`` branch of
:187-204, then :280-284, with every ``.cuda()`` removed.  They run in a namespace holding the reference's NeRF,
Embedding and render_rays, the trained coarse and fine weights (through a ``load_ckpt`` stand-in), a ``dataset``
with ``bounds`` and ``white_back``, and a ``mesh`` stand-in whose ``compute_vertex_normals`` is the restatement of
open3d's (tests/normals_ref.py; open3d cannot run here).  Stored: the mesh, and per case the normals (float64), the
rays, ``rgb_fine`` and the uint8 colours.

    NERF_PL_REFERENCE=/path/to/nerf_pl python tests/golden/make_vertex_normal_golden.py
"""
import ast
import json
import os
import sys
import types
from collections import defaultdict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import make_golden  # noqa: E402
from oracle import mesh_oracle as mo  # noqa: E402
from tests import normals_ref, npz_parts  # noqa: E402

NAME = "vertex_normal_colors"      # tests/golden/vertex_normal_colors.part<i>.npz
N_GRID, RANGE, THRESHOLD = 40, (-1.5, 1.5), 20.0
CHUNK = 1024 * 32                  # the script's default --chunk
# name: (dataset.bounds, white_back, N_samples, N_importance, near_t)
CASES = {
    "blender": ((2.0, 6.0), True, 64, 64, 1.0),
    # bounds and near_t that float32 cannot hold, no white background, 128 fine samples
    "inexact": ((1.7, 6.1), False, 64, 128, 1.1),
}


class _StripCuda(ast.NodeTransformer):
    """``x.cuda()`` -> ``x``: the reference runs these lines on a GPU; here they run on the CPU."""

    def visit_Call(self, node):
        self.generic_visit(node)
        if isinstance(node.func, ast.Attribute) and node.func.attr == "cuda" and not node.args:
            return node.func.value
        return node


def _is_use_vertex_normal(node):
    return isinstance(node, ast.If) and ast.unparse(node.test) == "args.use_vertex_normal"


def reference_source():
    """(the ``f`` definition, the body of :187-204's branch, :280-284) as code objects, ``.cuda()`` removed."""
    tree = ast.parse(open(os.path.join(make_golden.REF, "extract_color_mesh.py")).read())
    f_def = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "f")
    main = next(n for n in tree.body if isinstance(n, ast.If) and "__main__" in ast.unparse(n.test))
    branches = [n for n in main.body if _is_use_vertex_normal(n)]
    assert len(branches) == 2, "expected the :187 and :280 branches"
    colors = branches[1]
    after = main.body[main.body.index(colors) + 1]
    assert ast.unparse(after) == "v_colors = v_colors.astype(np.uint8)", ast.unparse(after)

    def code(nodes, what):
        mod = ast.fix_missing_locations(_StripCuda().visit(ast.Module(body=list(nodes), type_ignores=[])))
        return compile(mod, f"extract_color_mesh.py[{what}]", "exec")
    return (code([f_def], "f"), code(branches[0].body, "187-204"),
            code(colors.body + [after], "280-284"))


class MeshStandIn:
    """The open3d TriangleMesh of :163-174 (read from the PLY: float64 vertices holding float32 values, no normals)."""

    def __init__(self, vertices, triangles):
        self.vertices = np.asarray(vertices, np.float64)
        self.triangles = np.asarray(triangles, np.int32)
        self.vertex_normals = np.zeros((0, 3))

    def compute_vertex_normals(self):
        self.vertex_normals = normals_ref.vertex_normals(self.vertices, self.triangles)
        return self


def reference_mesh(Embedding, NeRF, fine_w):
    nerf_fine = make_golden.ref_model(NeRF, fine_w)
    emb_xyz, emb_dir = Embedding(3, 10), Embedding(3, 4)
    xyz_ = torch.from_numpy(mo.grid_positions(N_GRID, RANGE, RANGE, RANGE))
    with torch.no_grad():
        sigma = nerf_fine(torch.cat([emb_xyz(xyz_), emb_dir(torch.zeros_like(xyz_))], 1))[:, -1].numpy()
    sigma = np.maximum(sigma, 0).reshape(N_GRID, N_GRID, N_GRID)
    vi, t = mo.marching_cubes(sigma, THRESHOLD)
    vw = mo.to_world(vi, N_GRID, RANGE, RANGE, RANGE)
    return mo.keep_largest_cluster(vw, t)


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    Embedding, NeRF, render_rays, _ = make_golden.import_reference()
    coarse_w, fine_w = make_golden.load_trained_weights()
    vertices_, triangles = reference_mesh(Embedding, NeRF, fine_w)
    f_code, normal_code, colors_code = reference_source()
    arrays = {"vertices": vertices_, "triangles": triangles}
    meta = {"torch": torch.__version__, "N_grid": N_GRID, "range": list(RANGE), "threshold": THRESHOLD, "cases": {}}
    for name, (bounds, white_back, S, K, near_t) in CASES.items():
        nerf_fine = make_golden.ref_model(NeRF, fine_w)
        weights = {"nerf_coarse": coarse_w, "nerf_fine": fine_w}

        def load_ckpt(model, ckpt_path, model_name):
            model.load_state_dict({k: torch.from_numpy(v) for k, v in weights[model_name].items()})
        ns = {"torch": torch, "np": np, "defaultdict": defaultdict, "render_rays": render_rays, "NeRF": NeRF,
              "load_ckpt": load_ckpt, "nerf_fine": nerf_fine, "embeddings": [Embedding(3, 10), Embedding(3, 4)],
              "vertices_": vertices_.copy(), "triangles": triangles,
              "mesh": MeshStandIn(vertices_, triangles),
              "dataset": types.SimpleNamespace(bounds=np.array(bounds), white_back=white_back),
              "args": types.SimpleNamespace(use_vertex_normal=True, near_t=near_t, N_samples=S, N_importance=K,
                                            chunk=CHUNK, ckpt_path=None)}
        exec(f_code, ns)
        exec(normal_code, ns)
        exec(colors_code, ns)
        rays = torch.cat([ns["rays_o"], ns["rays_d"], ns["near"], ns["far"]], 1).numpy()
        arrays[f"{name}.normals"] = np.asarray(ns["mesh"].vertex_normals, np.float64)
        arrays[f"{name}.rays"] = rays
        arrays[f"{name}.rgb_fine"] = ns["results"]["rgb_fine"].numpy()
        arrays[f"{name}.colors"] = ns["v_colors"]
        meta["cases"][name] = {"bounds": list(bounds), "white_back": white_back, "N_samples": S, "N_importance": K,
                               "near_t": near_t}
        print(f"{name}: {len(vertices_)} vertices, {len(triangles)} triangles, colours {ns['v_colors'].dtype} "
              f"{ns['v_colors'].shape}")
    arrays["meta"] = np.array(json.dumps(meta))
    n = npz_parts.save(HERE, NAME, arrays)
    sizes = [os.path.getsize(os.path.join(HERE, f"{NAME}.part{i}.npz")) for i in range(n)]
    print(f"wrote {NAME}.part0..{n - 1}.npz ({sizes} bytes), torch {torch.__version__}")


if __name__ == "__main__":
    main()
