"""Time the small-part cleaning (Engine.clean_mesh, mesh_clean.cu) against marching cubes on the meshes it runs on.

    python tools/clean_bench.py [--reps 20] [--out DIR]

Workloads (CUDA events after warm-up, median of --reps):
  * the 257^3 and 513^3 grids of the synthetic He-scaled network on the demo image and camera, iso = median of the
    field, meshed on the device: marching cubes alone, and marching cubes followed by cleaning (the mesh never leaves HBM);
  * a 129^3 standard-normal field: the many-components worst case for the union-find and the per-component atomics.
Prints one JSON line with the GPU name and power limit read in the same run, the mesh sizes, component counts and the
CPU twin's (oracle/mesh_clean_oracle.py) time on the same mesh for context; also writes it to DIR/clean_bench.json.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from disn_b200 import synth
    from disn_b200.engine import Engine
    from oracle import mesh_clean_oracle as mco

    if not torch.cuda.is_available():
        raise SystemExit("clean_bench needs a GPU")
    eng = Engine(device=0, precision="f16f8")
    eng.load_weights(synth.make_weights(seed=7, init="he"))
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)         # the engine's work on a stream the events below are recorded on

    def timed(fn):
        """median and min ms of fn() between CUDA events, after 2 warm-up calls; both calls end in a host
        synchronisation (they size their outputs), which the interval includes"""
        fn()
        fn()
        ts = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            b.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.median(ts)), float(np.min(ts))

    BOX = [-1, -1, -1, 1, 1, 1]
    rows = []

    def run(name, ptr, R, iso):
        mc = lambda: eng.marching_cubes(None, BOX, iso, device_ptr=ptr, R=R, fetch=False)
        nv, nf = mc()
        v, f = eng.marching_cubes(None, BOX, iso, device_ptr=ptr, R=R)
        t0 = time.perf_counter()
        ref = mco.clean(v, f)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        mc_ms, mc_min = timed(mc)
        both_ms, both_min = timed(lambda: (mc(), eng.clean_mesh(fetch=False)))
        eng.marching_cubes(None, BOX, iso, device_ptr=ptr, R=R, fetch=False)
        launches = eng.launch_count
        c = eng.clean_mesh(fetch=False)
        launches = eng.launch_count - launches
        assert (c.n_components, c.n_kept, c.n_verts, c.n_faces) == (ref["n_components"], ref["n_kept"], len(ref["verts"]),
                                                                    len(ref["faces"])), name
        rows.append(dict(workload=name, R=R, iso=iso, verts=nv, faces=nf, components=c.n_components, kept=c.n_kept,
                         verts_out=c.n_verts, faces_out=c.n_faces, mc_ms=mc_ms, mc_plus_clean_ms=both_ms,
                         clean_ms=both_ms - mc_ms, clean_over_mc=(both_ms - mc_ms) / mc_ms, mc_min_ms=mc_min,
                         mc_plus_clean_min_ms=both_min, clean_launches=launches, cpu_twin_ms=cpu_ms))
        print(json.dumps(rows[-1]), file=sys.stderr)

    eng.encode(synth.synthetic_images(1))
    for res in (256, 512):
        R = res + 1
        ptr = eng.eval_grid_resident(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, res)
        grid = torch.from_numpy(eng.fetch(ptr, (R, R, R)))
        iso = float(grid.median().item())
        del grid
        run("predicted_%d^3" % R, ptr, R, iso)
    R = 129
    noise = torch.from_numpy(np.random.default_rng(129).standard_normal((R, R, R)).astype(np.float32)).cuda()
    torch.cuda.synchronize()
    run("normal_noise_%d^3" % R, noise.data_ptr(), R, 0.0)
    eng.close()
    out = {"gpu": gpu_info(), "reps": args.reps, "precision": "f16f8",
           "timing": "CUDA events on the engine's stream around each call (incl. its host synchronisation); median (and min) "
                     "of reps after 2 warm-ups; clean_ms = (mc + clean) - mc",
           "rows": rows}
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "clean_bench.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
