"""Coarse-to-fine grid benchmark (DESIGN.md §4.9): the demo image, the demo camera and synthetic He weights in f16f8.

For each resolution (default 256, 512, 1024), after one warm-up call:
  * the points evaluated by the coarse lattice and by each level, and their total against R^3;
  * device-event milliseconds per phase (coarse evaluation, each level, fill) and of marching cubes on the result;
  * how many sign-changing edges of the dense grid the adaptive grid missed (an end point interpolated, not evaluated),
    at band 1 and band 2.
The dense evaluation plus marching cubes is timed once per resolution (its kernels are already warm).  The synthetic
network need not cross 0, so the iso value is the median of its 65^3 grid, as in bench.py.  Prints one JSON line with
the GPU name and power limit read in the same run; with --out DIR also writes it to DIR/adaptive_bench.json.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from disn_b200 import _lib, synth  # noqa: E402
from disn_b200.engine import Engine  # noqa: E402

BOX = [-1.0, -1.0, -1.0, 1.0, 1.0, 1.0]


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        o = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=20).stdout.splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in o.split(",")]))
    except Exception as e:          # the timing below still needs the GPU; the label is best effort
        return {"error": repr(e)}


def phase_ms(eng):
    ms, n = (C.c_float * 8)(), C.c_int32(0)
    lib = _lib.load_test()
    if lib.disn_adaptive_phase_ms(eng._h, ms, C.byref(n)):
        raise RuntimeError(lib.disn_last_error().decode())
    return [round(float(v), 3) for v in ms[:n.value]]


def timed(fn, stream):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    out = fn()
    b.record(stream)
    b.synchronize()
    return out, round(a.elapsed_time(b), 3)


def missed_edges(eng, dense_ptr, R, iso, slab=32):
    """sign-changing edges of the dense grid with an end point the last adaptive call did not evaluate"""
    lib = _lib.load_test()
    missed = crossing = 0
    for z0 in range(0, R, slab):
        z1 = min(R, z0 + slab)                  # this slab's planes; one more is read for its z edges
        ze = min(R, z1 + 1)
        d = eng.fetch(dense_ptr + z0 * R * R * 4, (ze - z0, R, R)) < np.float32(iso)
        m = np.empty((ze - z0) * R * R, np.uint8)
        if lib.disn_adaptive_mask(eng._h, z0 * R * R, m.size, m.ctypes.data_as(C.c_void_p)):
            raise RuntimeError(lib.disn_last_error().decode())
        m = m.reshape(ze - z0, R, R).astype(bool)
        own, nz = slice(0, z1 - z0), ze - z0
        for lo, hi in (((own, slice(None), slice(0, -1)), (own, slice(None), slice(1, None))),
                       ((own, slice(0, -1)), (own, slice(1, None))),
                       ((slice(0, nz - 1),), (slice(1, nz),))):
            cross = d[lo] != d[hi]
            crossing += int(cross.sum())
            missed += int((cross & ~(m[lo] & m[hi])).sum())
    return missed, crossing


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512, 1024])
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
    # the synthetic network need not cross 0: mesh at the median of its 65^3 grid, as bench.py does
    iso = float(np.median(eng.eval_grid(BOX, synth.DEMO_TRANS_MAT, 64)))
    rows = []
    for res in a.res:
        R = res + 1
        eng.eval_grid_adaptive(BOX, tm, res, iso=iso)                 # warm-up
        (ptr, counts), wall = timed(lambda: eng.eval_grid_adaptive(BOX, tm, res, iso=iso), stream)
        phases = phase_ms(eng)
        (nv, nf), mc_ms = timed(lambda: eng.marching_cubes(None, BOX, iso, device_ptr=ptr, R=R, fetch=False), stream)
        row = {"res": res, "R3": R ** 3, "counts": counts, "evaluated": sum(counts),
               "fraction": round(sum(counts) / R ** 3, 5), "phase_ms": dict(zip(
                   ["coarse"] + ["level%d" % (16 >> i) for i in range(len(phases) - 2)] + ["fill"], phases)),
               "adaptive_call_ms": wall, "mc_ms": mc_ms, "verts": nv, "faces": nf}
        dense_ptr, dense_ms = timed(lambda: eng.eval_grid_resident(BOX, synth.DEMO_TRANS_MAT, res), stream)
        (dnv, dnf), dense_mc = timed(lambda: eng.marching_cubes(None, BOX, iso, device_ptr=dense_ptr, R=R, fetch=False),
                                     stream)
        row.update(dense_eval_ms=dense_ms, dense_mc_ms=dense_mc, dense_verts=dnv, dense_faces=dnf)
        for band in (1.0, 2.0):
            _, cnt = eng.eval_grid_adaptive(BOX, tm, res, iso=iso, band=band)
            miss, cross = missed_edges(eng, dense_ptr, R, iso)
            row["band%g" % band] = {"evaluated": sum(cnt), "missed_edges": miss, "dense_crossing_edges": cross}
        rows.append(row)
        print(json.dumps(row), flush=True)
    eng.close()
    result = {"gpu": info, "precision": "f16f8", "iso": iso, "weights": "synthetic He (seed 7)", "image": "demo", "rows": rows}
    print(json.dumps(result))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "adaptive_bench.json"), "w") as f:
            json.dump(result, f)


if __name__ == "__main__":
    main()
