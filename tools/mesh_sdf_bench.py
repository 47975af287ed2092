"""Time the signed distance field of a mesh (Engine.mesh_sdf, mesh_sdf.cu) phase by phase.

    python tools/mesh_sdf_bench.py [--reps 5] [--res 128 256] [--out DIR]

Meshes:
  * the marching-cubes mesh of the config-1 predicted 257^3 grid (synthetic He-scaled network on the demo image and
    camera, iso = median of the field);
  * a closed analytic torus meshed from a 129^3 field;
  * the mesh of a 129^3 standard-normal field (millions of faces in tens of thousands of components).
For each mesh and resolution: the call's wall time (it ends in a host synchronisation) and the four phases from CUDA
events inside the call (BVH build, distance, edge rasterisation, flood fill and sign), the median over --reps after one
warm-up call, and the kernel launches per call.  Prints one JSON line with the GPU name and power limit read in the same
run; also writes it to DIR/mesh_sdf_bench.json.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        o = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=20).stdout.splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in o.split(",")]))
    except Exception as e:          # the timing below still needs the GPU; the label is best effort
        return {"error": str(e)}


def meshes(eng):
    from disn_b200 import synth
    from oracle import mc_oracle
    box = [-1, -1, -1, 1, 1, 1]
    eng.load_weights(synth.make_weights(seed=7, init="he"))
    eng.encode(synth.synthetic_images(1))
    ptr = eng.eval_grid_resident(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 256)
    iso = float(np.median(eng.fetch(ptr, (257, 257, 257))))
    yield "predicted_257_mc", eng.marching_cubes(None, box, iso, device_ptr=ptr, R=257)
    ax = np.linspace(-1, 1, 129)
    z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
    torus = (np.sqrt((np.sqrt(x * x + y * y) - 0.5) ** 2 + z * z) - 0.22).astype(np.float32)
    yield "torus_129_closed", mc_oracle.marching_cubes(torus, box, 0.0)
    noise = np.random.default_rng(129).standard_normal((129, 129, 129)).astype(np.float32)
    yield "noise_129_mc", eng.marching_cubes(noise, box, 0.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from disn_b200.engine import Engine
    if not torch.cuda.is_available():
        raise SystemExit("mesh_sdf_bench needs a GPU")
    eng = Engine(device=0, precision="f16f8")
    rows = []
    for name, (v, f) in meshes(eng):
        for res in args.res:
            eng.load_mesh(v, f)
            eng.mesh_sdf(res)                          # warm-up: arena growth, module load
            wall, phases, launches = [], [], []
            for _ in range(args.reps):
                n0 = eng.launch_count
                t0 = time.perf_counter()
                grid, _ = eng.mesh_sdf(res)
                wall.append((time.perf_counter() - t0) * 1e3)
                launches.append(eng.launch_count - n0)
                phases.append(eng.mesh_sdf_phase_ms())
            med = {k: float(np.median([p[k] for p in phases])) for k in phases[0]}
            rows.append(dict(mesh=name, faces=int(len(f)), res=res, wall_ms=float(np.median(wall)),
                             phases_ms={k: round(x, 3) for k, x in med.items()}, launches=launches[0],
                             negative_fraction=float((grid < 0).mean())))
            print(json.dumps(rows[-1]), file=sys.stderr)
    eng.close()
    out = dict(gpu=gpu_info(), reps=args.reps, rows=rows)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "mesh_sdf_bench.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
