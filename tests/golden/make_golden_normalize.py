"""Generate tests/golden/normalize_ref.npz with the REFERENCE's own get_normalize_mesh
(preprocessing/create_point_sdf_grid.py:169-198), imported through make_golden.py's module stubs.

Run in the build container only (the GPU machine has no reference tree):
    python tests/golden/make_golden_normalize.py
trimesh and pymesh are absent, so their four calls are stubbed:
  * trimesh.load_mesh returns one stub mesh per part, whose area_faces are the twin's float64 face areas;
  * trimesh.sample.sample_surface returns the twin's samples of that part (oracle/mesh_norm_oracle.py, draws from
    np.random in sample_surface's order) and records the amount the reference asked for;
  * pymesh.load_mesh returns the float32 vertices widened to float64, and save_mesh_raw captures what is written.
This pins the reference's logic around the sampler: the int32 amounts, the concatenation, the float64 mean centroid, the
max norm and (v - c) / m.  Only the data is committed.
"""
import contextlib
import io
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import make_golden  # noqa: E402
from disn_b200.create_point_sdf_grid import surface_draws  # noqa: E402
from oracle import mc_oracle  # noqa: E402
from oracle import mesh_norm_oracle as no  # noqa: E402


def field_mesh(kind, R, centre=(0, 0, 0), scale=1.0):
    ax = np.linspace(-1, 1, R)
    z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
    x, y, z = x - centre[0], y - centre[1], z - centre[2]
    if kind == "sphere":
        f = np.sqrt(x * x + y * y + z * z) - 0.45
    else:
        f = np.sqrt((np.sqrt(x * x + y * y) - 0.4) ** 2 + z * z) - 0.15
    v, fc = mc_oracle.marching_cubes(f.astype(np.float32), [-1, -1, -1, 1, 1, 1], 0.0)
    return (v * np.float32(scale)).astype(np.float32), fc.astype(np.int32)


def cases():
    sv, sf = field_mesh("sphere", 17)
    tv, tf = field_mesh("torus", 21, centre=(0.2, -0.1, 0.05), scale=7.0)
    # two parts (two materials), the second interleaved with the first in face order
    av, af = field_mesh("sphere", 13, centre=(-0.3, 0, 0))
    bv, bf = field_mesh("torus", 17, centre=(0.3, 0.1, 0))
    v2 = np.concatenate([av, bv])
    f2 = np.concatenate([af, bf + len(av)]).astype(np.int32)
    p2 = np.concatenate([np.zeros(len(af), np.int32), np.ones(len(bf), np.int32)])
    perm = np.random.default_rng(3).permutation(len(f2))
    three = np.concatenate([f2[perm], [[0, 1, 2]]]).astype(np.int32)          # + a small third part
    p3 = np.concatenate([p2[perm], [2]]).astype(np.int32)
    return [("sphere", sv, sf, np.zeros(len(sf), np.int32), 1, 11),
            ("torus_x7_offcentre", tv, tf, np.zeros(len(tf), np.int32), 1, 12),
            ("three_parts", v2, three, p3, 3, 13)]


def main():
    argv, sys.argv = sys.argv, [sys.argv[0]]       # the reference module parses its flags at import
    try:
        _, ref = make_golden.import_reference()
    finally:
        sys.argv = argv
    out = {}
    for name, v, f, pid, P, seed in cases():
        scan = no.part_scan(v, f, pid, P)
        amts = no.amounts(scan["q"])
        np.random.seed(seed)
        draws = surface_draws(amts)
        pts, _ = no.sample(v, f, scan, amts, draws)
        offs = np.concatenate([[0], np.cumsum(amts)])
        asked, saved = [], {}

        class Part:
            def __init__(self, p):
                self.p = p
                self.faces = f[pid == p]
                self.area_faces = scan["areas"][pid == p]

        sys.modules["trimesh"].load_mesh = lambda path, process=True: [Part(p) for p in range(P)]

        def sample_surface(mesh, count):
            asked.append(int(count))
            return pts[offs[mesh.p]:offs[mesh.p + 1]], None

        sys.modules["trimesh"].sample = types.SimpleNamespace(sample_surface=sample_surface)
        sys.modules["pymesh"].load_mesh = lambda path: types.SimpleNamespace(vertices=v.astype(np.float64), faces=f)
        sys.modules["pymesh"].save_mesh_raw = lambda path, verts, faces: saved.update(verts=verts, faces=faces)
        # amounts away from integer boundaries: the reference's float product and the twin's integers agree
        area = np.array([scan["areas"][pid == p].sum() for p in range(P)])
        prod = area * 16384 / area.sum()
        assert P == 1 or np.all(np.abs(prod - np.rint(prod)) > 1e-6), prod     # one part: exactly 16384 both ways
        with tempfile.TemporaryDirectory() as td, contextlib.redirect_stdout(io.StringIO()):
            _, centroid, m = ref.get_normalize_mesh("model.obj", td)
        assert asked == amts, (asked, amts)
        out[name + "_verts"] = v
        out[name + "_faces"] = f
        out[name + "_part_ids"] = pid
        out[name + "_meta"] = np.array([P, seed], np.int64)
        out[name + "_amounts"] = np.array(asked, np.int64)
        out[name + "_centroid"] = np.asarray(centroid, np.float64)
        out[name + "_m"] = np.float64(m)
        out[name + "_out_verts"] = np.asarray(saved["verts"], np.float64)
        print(name, len(f), "faces, amounts", asked, "centroid", centroid, "m", m)
    np.savez_compressed(os.path.join(HERE, "normalize_ref.npz"), **out)


if __name__ == "__main__":
    main()
