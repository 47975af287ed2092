"""Time the device OBJ reader (Engine.read_obj) against the Python reader (create_sdf.read_obj / read_obj_parts).

    python tools/obj_read_bench.py [--reps 3] [--meshes eval torus noise] [--out DIR]

Meshes: `eval`, the evaluation benchmark's object (tools/eval_bench.py: the 829 K-face marching-cubes ground truth of the
synthetic network's 257^3 grid and its 24 views of the 65^3 grid, summed per object); `torus`, the preprocessing
benchmark's 52 K-face two-material torus (tools/preprocess_bench.py, read with parts); `noise`, the 6.7 M-face mesh of a
129^3 standard-normal field.  Each is written in disn_write_obj's %g, write_obj_exact's %.9g and np.savetxt's %.18e.
Per file: bytes, host wall-clock ms of both readers (the file read, the copies, and a synchronise and fetch at the end;
median of --reps after one warm-up), the device phase times from CUDA events, and the coordinates converted on the host.
Both readers' results are checked equal bit for bit.  Prints one JSON line with the GPU name and power limit read in the
same run; also writes it to DIR/obj_read_bench.json.
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


def median_ms(fn, reps):
    r = fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), r


def meshes(eng, names):
    from disn_b200 import synth
    box = [-1, -1, -1, 1, 1, 1]
    if "eval" in names:
        e = type(eng)(device=0, precision="f16f8")
        e.load_weights(synth.make_weights(seed=7, init="he"))
        e.encode(synth.synthetic_images(1))
        g = e.eval_grid(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 256)[0]
        iso = float(np.median(g))
        gt = e.marching_cubes(g, box, iso)
        g64 = e.eval_grid(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 64)[0]
        spread = float(np.std(g64))
        views = [e.marching_cubes(g64, box, iso + spread * (k - 12) / 96) for k in range(24)]
        e.close()
        yield "eval_object", [gt] + views, None
    if "torus" in names:
        from preprocess_bench import raw_meshes
        (_, v, f), = list(raw_meshes(eng, ["torus"]))
        pid = (np.arange(len(f)) // 1000 % 2).astype(np.int32)
        yield "torus_two_material", [(v, f)], pid
    if "noise" in names:
        noise = np.random.default_rng(129).standard_normal((129, 129, 129)).astype(np.float32)
        yield "noise_129_mc", [eng.marching_cubes(noise, box, 0.0)], None


def write(path, fmt, v, f, pid):
    from disn_b200.create_sdf import write_obj
    if fmt == "%g" and pid is None:
        write_obj(path, v, f)
        return
    with open(path, "w") as fh:
        np.savetxt(fh, v, fmt="v {0} {0} {0}".format(fmt))
        if pid is None:
            np.savetxt(fh, np.asarray(f, np.int64) + 1, fmt="f %d %d %d")
        else:
            for i in range(0, len(f), 1000):
                fh.write("usemtl m%d\n" % pid[i])
                np.savetxt(fh, np.asarray(f[i:i + 1000], np.int64) + 1, fmt="f %d %d %d")


def same(a, b):
    for x, y in zip(a, b):
        if isinstance(x, np.ndarray):
            assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
        else:
            assert x == y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--meshes", nargs="+", default=["eval", "torus", "noise"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from eval_bench import gpu_info
    from disn_b200.create_sdf import read_obj, read_obj_parts
    from disn_b200.engine import Engine

    eng = Engine(device=0, precision="fp32")
    rows = []
    with tempfile.TemporaryDirectory() as td:
        for name, parts_list, pid in meshes(eng, args.meshes):
            parts = pid is not None
            for fmt in ("%g", "%.9g", "%.18e"):
                paths = []
                for k, (v, f) in enumerate(parts_list):
                    paths.append(os.path.join(td, "%s_%d.obj" % (name, k)))
                    write(paths[-1], fmt, v, f, pid)
                py = read_obj_parts if parts else read_obj
                py_ms, want = median_ms(lambda: [py(p) for p in paths], args.reps)
                dev_ms, got = median_ms(lambda: [eng.read_obj(p, parts=parts) for p in paths], args.reps)
                for a, b in zip(got, want):
                    same(a, b)
                phases, host_tokens = {}, 0
                for p in paths:                 # per-file statistics, summed over the object's files
                    eng.read_obj(p, parts=parts)
                    st = eng.obj_read_stats()
                    host_tokens += st["host_tokens"]
                    for k, t in st["phase_ms"].items():
                        phases[k] = phases.get(k, 0.0) + t
                row = dict(mesh=name, format=fmt, files=len(paths), parts=parts,
                                 bytes=int(sum(os.path.getsize(p) for p in paths)),
                                 faces=int(sum(len(f) for _, f in parts_list)), python_ms=py_ms, device_ms=dev_ms,
                                 speedup=py_ms / dev_ms, phase_ms=phases, host_tokens=host_tokens)
                rows.append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
                for p in paths:
                    os.remove(p)
    assert eng.obj_fallbacks == 0
    eng.close()
    out = {"gpu": gpu_info(), "reps": args.reps,
           "timing": "host wall clock per object, median of reps after one warm-up; includes the file read and ends in a "
                     "synchronise and fetch", "rows": rows}
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "obj_read_bench.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
