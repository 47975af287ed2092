"""Coarse-to-fine mesh benchmark (DESIGN.md §4.10): the demo image, the demo camera and synthetic He weights in f16f8.

For each resolution (default 256, 512, 1024, 2048) and two iso values -- the median of the 65^3 grid and its 0.95
quantile (a smaller surface) -- after one warm-up call of disn_mesh_grid_adaptive:
  * the points evaluated by the coarse lattice and by each level;
  * device-event milliseconds of its phases (levels, candidate cells, mesh) and the whole call;
  * the bytes its buffers hold, against the dense path's ~10 B per grid point (grid 4, marks 1, marching-cubes codes 1
    and vertex bases 4);
  * where the dense path runs (sdf_res <= 1024 here), eval_grid_adaptive + marching cubes timed the same way, and
    whether both meshes are equal bit for bit.
Prints one JSON line per row and a final line with the GPU name and power limit read in the same run; with --out DIR
also writes it to DIR/adaptive_mesh_bench.json.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from disn_b200 import _lib, synth  # noqa: E402
from disn_b200.engine import Engine  # noqa: E402
from tools.adaptive_bench import BOX, gpu_info, timed  # noqa: E402


def diag(fn, *args):
    lib = _lib.load_test()
    if getattr(lib, fn)(*args):
        raise RuntimeError(lib.disn_last_error().decode())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512, 1024, 2048])
    ap.add_argument("--dense-max", type=int, default=1024, help="largest sdf_res also run through the dense path")
    ap.add_argument("--out", default=None, metavar="DIR")
    a = ap.parse_args()
    info = gpu_info()
    img = np.load(os.path.join(ROOT, "tests", "golden", "demo_input.npz"))["img_u8"].astype(np.float32) / np.float32(255.)
    eng = Engine(device=0, precision="f16f8")
    eng.load_weights(synth.make_weights(seed=7, init="he"))
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)
    eng.encode(img[None])
    tm = synth.DEMO_TRANS_MAT[0]
    g65 = eng.eval_grid(BOX, synth.DEMO_TRANS_MAT, 64)
    isos = {"median": float(np.median(g65)), "q95": float(np.quantile(g65, 0.95))}
    rows = []
    for res in a.res:
        R = res + 1
        for iso_name, iso in isos.items():
            eng.mesh_grid_adaptive(BOX, tm, res, iso=iso, fetch=False)              # warm-up
            ((nv, nf), counts), wall = timed(lambda: eng.mesh_grid_adaptive(BOX, tm, res, iso=iso, fetch=False), stream)
            ms = np.zeros(3, np.float32)
            diag("disn_mesh_adaptive_phase_ms", eng._h, ms.ctypes.data_as(C.c_void_p))
            held = C.c_int64(0)
            diag("disn_mesh_adaptive_bytes", eng._h, C.byref(held))
            row = {"res": res, "iso": iso_name, "R3": R ** 3, "counts": counts, "evaluated": sum(counts),
                   "phase_ms": dict(zip(["levels", "candidates", "mesh"], [round(float(m), 3) for m in ms])),
                   "call_ms": wall, "verts": nv, "faces": nf, "bytes_held": held.value,
                   "bytes_per_evaluated_point": round(held.value / sum(counts), 2), "dense_bytes_est": 10 * R ** 3}
            if res <= a.dense_max:
                v1, f1 = eng.fetch_mesh()
                eng.eval_grid_adaptive(BOX, tm, res, iso=iso)                       # warm-up
                (ptr, _), dense_eval = timed(lambda: eng.eval_grid_adaptive(BOX, tm, res, iso=iso), stream)
                (dnv, dnf), dense_mc = timed(lambda: eng.marching_cubes(None, BOX, iso, device_ptr=ptr, R=R, fetch=False),
                                             stream)
                v2, f2 = eng.fetch_mesh()
                row.update(dense_eval_ms=dense_eval, dense_mc_ms=dense_mc, dense_total_ms=round(dense_eval + dense_mc, 3),
                           equal=bool(np.array_equal(v1.view(np.uint32), v2.view(np.uint32)) and np.array_equal(f1, f2)))
            rows.append(row)
            print(json.dumps(row), flush=True)
    eng.close()
    result = {"gpu": info, "precision": "f16f8", "isos": isos, "weights": "synthetic He (seed 7)", "image": "demo",
              "band": 1.0, "rows": rows}
    print(json.dumps(result))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "adaptive_mesh_bench.json"), "w") as f:
            json.dump(result, f)


if __name__ == "__main__":
    main()
