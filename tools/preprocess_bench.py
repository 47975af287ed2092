"""Time the per-object preprocessing chain (create_point_sdf_grid.create_sdf_obj's steps) phase by phase.

    python tools/preprocess_bench.py [--reps 3] [--res 128 256] [--meshes torus predicted noise] [--out DIR]

Meshes (written once as raw OBJs with two materials, in a temporary directory):
  * torus: a closed analytic torus meshed from a 129^3 field, scaled x7 and moved off the origin;
  * predicted: the marching-cubes mesh of the config-1 predicted 257^3 grid (~8.3e5 faces);
  * noise: the mesh of a 129^3 standard-normal field (~6.7e6 faces).
Phases: OBJ parse (host, once per mesh), upload, part areas, normalise (amounts, host draws and the device call),
field (disn_mesh_sdf into the resident field buffer), isosurface (marching cubes at 0.003), band sampling (32768
samples), and the writes (pc_norm.obj, isosurf.obj, ori_sample.npz; once per mesh and resolution).  The chain phases
(`call_wall_ms`) are host wall times of each call: every library call ends in a synchronisation of the context's stream,
so the time spans the device work it launched, and it also holds the call's host work (part areas and normalise: the
counting sort of the part ids and the uploads; normalise also the np.random draws; band sampling: the randint draws).
Only the field's internal phases (`field_phases_ms`) are device times, from the CUDA events of disn_mesh_sdf_phase_ms.
For comparison the same run fetches the field to the host and times the host sample_sdf on it.  Medians over --reps after one warm-up pass.  Prints one JSON line
with the GPU name and power limit read in the same run; also writes it to DIR/preprocess_bench.json.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def raw_meshes(eng, names):
    from disn_b200 import synth
    from oracle import mc_oracle
    box = [-1, -1, -1, 1, 1, 1]
    if "torus" in names:
        ax = np.linspace(-1, 1, 129)
        z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
        torus = (np.sqrt((np.sqrt(x * x + y * y) - 0.5) ** 2 + z * z) - 0.22).astype(np.float32)
        v, f = mc_oracle.marching_cubes(torus, box, 0.0)
        yield "torus_129_x7", (v * np.float32(7) + np.float32([3.5, -2.0, 1.25])).astype(np.float32), f
    if "predicted" in names:
        eng.load_weights(synth.make_weights(seed=7, init="he"))
        eng.encode(synth.synthetic_images(1))
        ptr = eng.eval_grid_resident(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 256)
        iso = float(np.median(eng.fetch(ptr, (257, 257, 257))))
        yield ("predicted_257_mc",) + tuple(eng.marching_cubes(None, box, iso, device_ptr=ptr, R=257))
    if "noise" in names:
        noise = np.random.default_rng(129).standard_normal((129, 129, 129)).astype(np.float32)
        yield ("noise_129_mc",) + tuple(eng.marching_cubes(noise, box, 0.0))


def write_raw(path, v, f):
    """Two materials, alternating in blocks of 1000 faces."""
    with open(path, "w") as fh:
        np.savetxt(fh, v, fmt="v %.9g %.9g %.9g")
        for i in range(0, len(f), 1000):
            fh.write("usemtl m%d\n" % ((i // 1000) % 2))
            np.savetxt(fh, f[i:i + 1000] + 1, fmt="f %d %d %d")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--res", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--meshes", nargs="+", default=["torus", "predicted", "noise"])
    ap.add_argument("--num_sample", type=int, default=32768)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from disn_b200 import create_point_sdf_grid as cpsg
    from disn_b200.create_sdf import read_obj_parts
    from disn_b200.engine import Engine
    from mesh_sdf_bench import gpu_info
    if not torch.cuda.is_available():
        raise SystemExit("preprocess_bench needs a GPU")
    eng = Engine(device=0, precision="f16f8")
    rows = []
    with tempfile.TemporaryDirectory() as td:
        for name, v, f in raw_meshes(eng, args.meshes):
            path = os.path.join(td, name + ".obj")
            write_raw(path, v, f)
            t0 = time.perf_counter()
            mesh = read_obj_parts(path)
            parse_ms = (time.perf_counter() - t0) * 1e3
            verts, faces, pid, names = mesh
            P = len(names)
            for res in args.res:
                R = res + 1
                ph = {k: [] for k in ("upload", "part_areas", "normalise", "field", "isosurface", "band_sampling")}
                for rep in range(args.reps + 1):
                    np.random.seed(rep)
                    t = [time.perf_counter()]
                    eng.load_mesh(verts, faces)
                    t.append(time.perf_counter())
                    q, _ = eng.part_areas(pid, P)
                    t.append(time.perf_counter())
                    amts = cpsg.surface_amounts(q)
                    c, m = eng.normalize_mesh(pid, P, amts, cpsg.surface_draws(amts))
                    t.append(time.perf_counter())
                    ptr = eng.field_buffer(R)
                    _, bbox = eng.mesh_sdf(res, device_ptr=ptr)
                    t.append(time.perf_counter())
                    nv, nf = eng.marching_cubes(None, bbox, 0.003, device_ptr=ptr, R=R, fetch=False)
                    t.append(time.perf_counter())
                    smp = eng.band_samples(args.num_sample, 0.1, 0.003, np.float32(bbox), res, device_ptr=ptr)
                    t.append(time.perf_counter())
                    if rep:
                        for k, a, b in zip(ph, t[:-1], t[1:]):
                            ph[k].append((b - a) * 1e3)
                field_phases = eng.mesh_sdf_phase_ms()
                # writes: the chain's three files, once
                t0 = time.perf_counter()
                eng.write_mesh_obj(os.path.join(td, "isosurf.obj"))
                eng.load_mesh(verts, faces)
                eng.normalize_mesh(given=[c[0], c[1], c[2], m])
                cpsg.write_obj_exact(os.path.join(td, "pc_norm.obj"), *eng.fetch_mesh())
                cpsg.write_sample_file(os.path.join(td, "ori_sample.npz"), os.path.join(td, "flag.txt"), smp, False, c, m,
                                       np.float32(bbox))
                writes_ms = (time.perf_counter() - t0) * 1e3
                # host sample_sdf on the same field, after fetching it
                t0 = time.perf_counter()
                field = eng.fetch(ptr, (R, R, R))
                t1 = time.perf_counter()
                np.random.seed(0)
                cpsg.sample_sdf("", args.num_sample, 0.1, 0.003, {"param": np.float32(bbox), "value": field}, res)
                t2 = time.perf_counter()
                med = {k: round(float(np.median(x)), 3) for k, x in ph.items()}
                rows.append(dict(mesh=name, faces=int(len(faces)), parts=P, res=res, obj_parse_ms=round(parse_ms, 1),
                                 call_wall_ms=med, field_phases_ms={k: round(x, 3) for k, x in field_phases.items()},
                                 writes_ms=round(writes_ms, 1), iso_faces=int(nf),
                                 host_sample_sdf_ms=round((t2 - t1) * 1e3, 1), host_fetch_field_ms=round((t1 - t0) * 1e3, 1),
                                 band_counts=eng.last_band_counts.tolist()))
                print(json.dumps(rows[-1]), file=sys.stderr)
    eng.close()
    out = dict(gpu=gpu_info(), reps=args.reps, num_sample=args.num_sample, rows=rows)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "preprocess_bench.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
