"""Time the evaluation drivers (disn_b200/eval_cd_emd.py, eval_f_score.py, eval_iou.py) on one synthetic object, and
Engine.iou_views against one Engine.iou call per view.

    python tools/eval_bench.py [--reps 5] [--out DIR]

The object: the ground truth is the marching-cubes mesh of the 257^3 grid of the synthetic He-scaled network on the demo
image and camera at the median of its field; the 24 views are the meshes of its 65^3 grid at 24 isovalues around that
median.  The meshes are written as OBJ files and read back as the drivers read them.  Per driver and object, host
wall-clock (time.perf_counter; every GPU call ends in a synchronise) of: OBJ parsing as the drivers do it
(Engine.read_obj; the Python reader's time is reported beside it as python_parse_ms) / point-file parsing, sampling, and
the GPU metric calls, median of --reps.  iou_views and 24 x iou first check that their counts are equal.  Prints one JSON
line with the GPU name and power limit read in the same run; also writes it to DIR/eval_bench.json.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
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


def timed(fn, reps):
    """fn() once to warm up, then median ms of reps calls (and the last result)."""
    r = fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from disn_b200 import eval_f_score, synth
    from disn_b200.create_sdf import read_obj, write_obj
    from disn_b200.engine import Engine

    V, N, DIM = 24, 2048, 110
    eng = Engine(device=0, precision="f16f8")
    eng.load_weights(synth.make_weights(seed=7, init="he"))
    eng.encode(synth.synthetic_images(1))
    BOX = [-1, -1, -1, 1, 1, 1]
    g = eng.eval_grid(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 256)[0]
    iso = float(np.median(g))
    gt = eng.marching_cubes(g, BOX, iso)
    g64 = eng.eval_grid(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 64)[0]
    spread = float(np.std(g64))
    views = [eng.marching_cubes(g64, BOX, iso + spread * (k - V / 2) / (4 * V)) for k in range(V)]
    eng.close()
    eng = Engine(device=0, precision="fp32")
    eval_f_score._ENGINE = eng
    rows = {}
    with tempfile.TemporaryDirectory() as td:
        gt_path = os.path.join(td, "isosurf.obj")
        write_obj(gt_path, *gt)
        paths = [os.path.join(td, "03001627_obj_%02d.obj" % k) for k in range(V)]
        for p, (v, f) in zip(paths, views):
            write_obj(p, v, f)
        read_all = lambda: [read_obj(gt_path)] + [read_obj(p) for p in paths]
        python_parse_ms, py_meshes = timed(read_all, args.reps)
        parse_ms, meshes = timed(lambda: [eng.read_obj(gt_path)] + [eng.read_obj(p) for p in paths], args.reps)
        assert eng.obj_fallbacks == 0 and all(a.tobytes() == b.tobytes() for m, n in zip(meshes, py_meshes)
                                              for a, b in zip(m, n)), "Engine.read_obj != read_obj"

        def sample():
            np.random.seed(0)
            b = np.zeros((V + 1, N, 3), np.float32)
            for i, (v, _) in enumerate(meshes):
                b[i] = v[np.random.randint(v.shape[0], size=N)]
            return b
        sample_ms, batch = timed(sample, args.reps)
        pl_ms, _ = timed(lambda: eng.points_loss(batch), args.reps)
        rows["cd_emd"] = dict(parse_ms=parse_ms, sample_ms=sample_ms, gpu_ms=pl_ms)

        pnt = [os.path.join(td, "pnt_%02d.txt" % i) for i in range(V + 1)]
        for p, b in zip(pnt, batch):
            np.savetxt(p, b, delimiter=",")

        def load_pnt():
            b = np.zeros((V + 1, N, 3), np.float32)
            for i, p in enumerate(pnt):
                b[i] = np.loadtxt(p, dtype=float, delimiter=",")
            return b
        fparse_ms, fb = timed(load_pnt, args.reps)
        fd_ms, _ = timed(lambda: eval_f_score.get_points_distance(fb), args.reps)
        rows["f_score"] = dict(parse_ms=fparse_ms, sample_ms=0.0, gpu_ms=fd_ms)

        (rv, rf), vs = meshes[0], meshes[1:]
        iv_ms, (_, inter, uni) = timed(lambda: eng.iou_views(rv, rf, vs, dim=DIM), args.reps)
        pairs = lambda: [eng.iou(rv, rf, v, f, dim=DIM, want_grids=True)[1:3] for v, f in vs]
        pair_ms, pr = timed(pairs, args.reps)
        assert [(int(a), int(b)) for a, b in zip(inter, uni)] == [tuple(p) for p in pr], "iou_views != 24 x iou"
        rows["iou"] = dict(parse_ms=parse_ms, sample_ms=0.0, gpu_ms=iv_ms, gpu_ms_24_separate_iou=pair_ms)
    for k, r in rows.items():
        r["total_ms"] = r["parse_ms"] + r["sample_ms"] + r["gpu_ms"]
        r["parse_share"] = r["parse_ms"] / r["total_ms"]
        if k != "f_score":
            r["python_parse_ms"] = python_parse_ms
    eng.close()
    out = {"gpu": gpu_info(), "reps": args.reps, "views": V, "num_sample_points": N, "dim": DIM,
           "gt_mesh": {"grid": "257^3", "verts": int(len(gt[0])), "faces": int(len(gt[1]))},
           "view_faces": {"min": int(min(len(f) for _, f in views)), "max": int(max(len(f) for _, f in views))},
           "timing": "host wall clock per object, median of reps after one warm-up; GPU calls end in a synchronise",
           "drivers": rows, "iou_views_speedup": rows["iou"]["gpu_ms_24_separate_iou"] / rows["iou"]["gpu_ms"]}
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "eval_bench.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
