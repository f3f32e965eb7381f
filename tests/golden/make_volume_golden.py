"""Write tests/golden/volume_unity.part*.npz: the Unity volume (.vol) of extract_mesh.ipynb, by the UNMODIFIED
reference.

For each case, the reference's ``models.nerf`` Embedding / NeRF with the trained fine weights compute ``rgbsigma``
of the notebook's grid on the CPU (its "Search for tight bounds" cell, with the CUDA transfers left out). Then the
literal source of the notebook cell "Generate .vol file for volume rendering in Unity" runs in a temporary directory,
without its ``assert N==512`` guard. The cell's ``sigma`` comes from the literal ``sigma = ...`` lines of the bounds
cell. Stored per case: rgbsigma (N^3, 4), the cell's float32 ``a`` before it is filtered, and the file's bytes.

    NERF_PL_REFERENCE=/path/to/nerf_pl python tests/golden/make_volume_golden.py
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import make_golden  # noqa: E402
from tests import npz_parts, volume_ref  # noqa: E402

NAME = "volume_unity"      # tests/golden/volume_unity.part<i>.npz
# name: (N, x_range, y_range, z_range)
CASES = {
    "cube48": (48, (-1.5, 1.5), (-1.5, 1.5), (-1.5, 1.5)),
    "unequal33": (33, (-1.5, 1.5), (-1.2, 1.4), (-1.5, 1.3)),
}
CHUNK = 1024 * 32     # the notebook's chunk


def notebook_cells():
    nb = json.load(open(os.path.join(make_golden.REF, "extract_mesh.ipynb")))
    src = ["".join(c["source"]) for c in nb["cells"] if c["cell_type"] == "code"]
    bounds = next(s for s in src if "rgbsigma = torch.cat(out_chunks, 0)" in s)
    vol = next(s for s in src if ".vol" in s)
    return bounds, vol


def without_assert(cell: str) -> str:
    """The cell minus its ``assert N==512, \\`` statement (two lines)."""
    lines, out, skip = cell.split("\n"), [], False
    for ln in lines:
        if skip:
            skip = ln.rstrip().endswith("\\")
            continue
        if ln.lstrip().startswith("assert N==512"):
            skip = ln.rstrip().endswith("\\")
            continue
        out.append(ln)
    return "\n".join(out)


def reference_rgbsigma(Embedding, NeRF, weights, N, xr, yr, zr):
    nerf_fine = make_golden.ref_model(NeRF, weights)
    embedding_xyz, embedding_dir = Embedding(3, 10), Embedding(3, 4)
    x, y, z = np.linspace(*xr, N), np.linspace(*yr, N), np.linspace(*zr, N)
    xyz_ = torch.FloatTensor(np.stack(np.meshgrid(x, y, z), -1).reshape(-1, 3))
    dir_ = torch.zeros_like(xyz_)
    out_chunks = []
    with torch.no_grad():
        for i in range(0, xyz_.shape[0], CHUNK):
            emb = torch.cat([embedding_xyz(xyz_[i:i + CHUNK]), embedding_dir(dir_[i:i + CHUNK])], 1)
            out_chunks += [nerf_fine(emb)]
    return torch.cat(out_chunks, 0)


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    Embedding, NeRF, _, _ = make_golden.import_reference()
    weights = make_golden.load_trained_weights()[1]
    bounds_cell, vol_cell = notebook_cells()
    sigma_lines = "\n".join(ln for ln in bounds_cell.split("\n") if ln.startswith("sigma = "))
    vol_cell = without_assert(vol_cell)
    a_lines = vol_cell.split("a = a.flatten()")[0] + "a = a.flatten()\n"
    arrays, meta = {}, {"numpy": np.__version__, "torch": torch.__version__, "simd": volume_ref.numpy_simd(),
                        "cases": {}}
    for name, (N, xr, yr, zr) in CASES.items():
        rgbsigma = reference_rgbsigma(Embedding, NeRF, weights, N, xr, yr, zr)
        ns = {"np": np, "torch": torch, "rgbsigma": rgbsigma, "N": N, "xmin": xr[0], "xmax": xr[1], "ymin": yr[0],
              "ymax": yr[1], "zmin": zr[0], "zmax": zr[1], "scene_name": name}
        exec(sigma_lines, ns)
        ns_a = dict(ns)
        exec(a_lines, ns_a)
        cwd = os.getcwd()
        with tempfile.TemporaryDirectory() as d:
            os.chdir(d)
            try:
                exec(vol_cell, ns)
                vol = open(f"{name}.vol", "rb").read()
            finally:
                os.chdir(cwd)
        # one array per channel, so that the parts of the archive stay under 1 MB each
        for ch in range(4):
            arrays[f"{name}.rgbsigma{ch}"] = rgbsigma.numpy()[:, ch].astype(np.float32)
        arrays[f"{name}.a"] = np.asarray(ns_a["a"], np.float32)
        arrays[f"{name}.vol"] = np.frombuffer(vol, np.uint8)
        meta["cases"][name] = {"N": N, "ranges": [list(xr), list(yr), list(zr)], "M": len(vol) // 8}
        print(f"{name}: N {N}, {len(vol) // 8} voxels with a > 0")
    arrays["meta"] = np.array(json.dumps(meta))
    n = npz_parts.save(HERE, NAME, arrays)
    sizes = [os.path.getsize(os.path.join(HERE, f"{NAME}.part{i}.npz")) for i in range(n)]
    print(f"wrote {NAME}.part0..{n - 1}.npz ({sizes} bytes), numpy {np.__version__}, SIMD {meta['simd']}")


if __name__ == "__main__":
    main()
