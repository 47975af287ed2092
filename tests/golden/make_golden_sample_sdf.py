"""Generate tests/golden/sample_sdf.npz with the REFERENCE's own sample_sdf / check_insideout
(preprocessing/create_point_sdf_grid.py:74-137), imported through make_golden.py's module stubs.

Run in the build container only (the GPU machine has no reference tree):
    python tests/golden/make_golden_sample_sdf.py
The field is analytic (two spheres, one shifted so the origin is outside), seeded with np.random.seed; only the data is
committed.
"""
import contextlib
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden  # noqa: E402

CASES = [  # (name, centre, radius, cat_id, num_sample, bandwidth, iso, seed)
    ("centred_plane", (0.0, 0.0, 0.0), 0.6, "02691156", 4000, 0.1, 0.0, 3),
    ("shifted_car", (0.5, 0.4, 0.3), 0.35, "02958343", 3001, 0.1, 0.0, 4),
    ("chair_iso", (0.0, 0.1, 0.0), 0.5, "03001627", 2000, 0.05, 0.01, 5),
    ("short_band", (0.0, 0.0, 0.0), 0.05, "04530566", 1000, 0.3, 0.0, 6),   # the inner bands run short
]
RES = 20
PARAM = [-1.0, -0.9, -1.1, 1.0, 1.1, 0.9]


def field(centre, radius):
    ax = [np.linspace(PARAM[a], PARAM[3 + a], RES + 1) for a in range(3)]
    z, y, x = np.meshgrid(ax[2], ax[1], ax[0], indexing="ij")
    return (np.sqrt((x - centre[0]) ** 2 + (y - centre[1]) ** 2 + (z - centre[2]) ** 2) - radius).astype(np.float32)


def main():
    argv, sys.argv = sys.argv, [sys.argv[0]]       # the reference module parses its flags at import
    try:
        _, ref = make_golden.import_reference()
    finally:
        sys.argv = argv
    out = {"res": RES, "param": np.float32(PARAM)}
    for name, centre, radius, cat, n, bw, iso, seed in CASES:
        val = field(centre, radius)
        np.random.seed(seed)
        with contextlib.redirect_stdout(io.StringIO()):
            pts, flag = ref.sample_sdf(cat, n, bw, iso, {"param": np.float32(PARAM), "value": val}, RES)
        out[name + "_value"] = val
        out[name + "_samples"] = pts
        out[name + "_insideout"] = np.bool_(flag)
        print(name, pts.shape, bool(flag))
    np.savez(os.path.join(HERE, "sample_sdf.npz"), **out)


if __name__ == "__main__":
    main()
