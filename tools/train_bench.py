"""Decoder training step time on the GPU: Engine.train_step at B images x N points (the reference's recommended 20 x 2048
by default) on synthetic data.  The step time is host wall time around the call, which ends in a device synchronise;
the phases (encode, gather, forward, loss, backward, Adam) are the device events the step records (train_phase_ms),
their medians over the timed steps.

    python tools/train_bench.py [--B 20] [--N 2048] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from disn_b200 import synth  # noqa: E402
from disn_b200.engine import Engine  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=20)
    ap.add_argument("--N", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="fp32", choices=("fp32", "bf16x3", "f16f8"))
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    imgs = synth.synthetic_images(a.B)
    tm = synth.synthetic_trans_mats(a.B).astype(np.float32)
    pts = rng.uniform(-0.5, 0.5, size=(a.B, a.N, 3)).astype(np.float32)
    gt = (np.linalg.norm(pts, axis=2) - 0.303).astype(np.float32)
    eng = Engine(device=0, precision=a.precision, max_batch=8)
    try:
        eng.load_weights(synth.make_weights(seed=7))
        eng.train_begin()

        def timed(fn, n):
            ts = []
            for _ in range(n):
                t0 = time.perf_counter()
                fn()
                ts.append(time.perf_counter() - t0)
            return ts

        step = lambda: eng.train_step(imgs, pts, pts, tm, gt, 1e-4)
        timed(step, a.warmup)
        t_step, phases = [], []
        for _ in range(a.steps):
            t_step += timed(step, 1)
            phases.append(eng.train_phase_ms())
    finally:
        eng.close()
    ms = lambda ts: 1e3 * float(np.median(ts))
    res = {"gpu": gpu_info(), "B": a.B, "N": a.N, "precision": a.precision, "step_ms": ms(t_step),
           "step_ms_p10_p90": [1e3 * float(np.percentile(t_step, 10)), 1e3 * float(np.percentile(t_step, 90))],
           "phase_ms": {k: float(np.median([p[k] for p in phases])) for k in phases[0]},
           "steps_per_s": 1e3 / ms(t_step)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
