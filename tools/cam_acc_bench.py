"""Throughput of the camera checkpoint score (Engine.cam_metrics, the work of train_sdf_cam --test per batch).

Times Engine.cam_metrics on synthetic in-memory views at --batch images (scored in encodes of 8, as the driver does)
and --points samples per view, after a warm-up, with a host clock around calls that end in a device synchronisation.
A separate torch.profiler pass gives cam_acc_kernel's share of the device time of a call.  Prints one JSON line with the
card's name and power limit.

    python tools/cam_acc_bench.py --batch 32 --points 2048 --iters 300 [--out results/cam_acc_bench.json]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--points", type=int, default=2048)
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--precision", default="f16f8", choices=("fp32", "bf16x3", "f16f8"))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from disn_b200 import synth, train_sdf_cam
    from disn_b200.engine import Engine
    from tests.test_gpu_cam import make_cam_weights
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU")
    B, N = args.batch, args.points
    rng = np.random.default_rng(0)
    batch = {"img": synth.synthetic_images(B, seed=1), "sdf_pt": rng.uniform(-0.5, 0.5, (B, N, 3)).astype(np.float32),
             "RT": (np.tile(np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [0, 0, 1.4]]), (B, 1, 1))
                    + 0.1 * rng.standard_normal((B, 4, 3))).astype(np.float32)}
    K = np.array([[149.84375, 0., 68.5], [0., 149.84375, 68.5], [0., 0., 1.]])
    batch["trans_mat"] = (batch["RT"].astype(np.float64) @ K.T).astype(np.float32)
    eng = Engine(device=0, precision=args.precision, max_batch=min(B, train_sdf_cam.ENGINE_BATCH))
    try:
        eng.load_weights_raw(make_cam_weights(synth.make_weights(seed=7, init="he")))
        for _ in range(args.warmup):
            train_sdf_cam.batch_metrics(eng, batch)
        times = []
        for _ in range(args.iters):
            t0 = time.perf_counter()
            train_sdf_cam.batch_metrics(eng, batch)       # every call ends in a stream synchronisation
            times.append(time.perf_counter() - t0)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                train_sdf_cam.batch_metrics(eng, batch)
        kern = {e.key: e.device_time_total for e in prof.key_averages()}
        total = sum(v for k, v in kern.items() if not k.startswith("Memcpy") and not k.startswith("Memset"))
        acc = sum(v for k, v in kern.items() if "cam_acc_kernel" in k)
    finally:
        eng.close()
    t = np.array(times)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip().splitlines()
    res = {"metric": "cam_metrics_views_per_s", "batch": B, "points": N, "precision": args.precision,
           "iters": args.iters, "median_ms": float(np.median(t) * 1e3), "p10_ms": float(np.percentile(t, 10) * 1e3),
           "p90_ms": float(np.percentile(t, 90) * 1e3), "views_per_s": float(B / np.median(t)),
           "cam_acc_kernel_share_of_device_kernel_time": float(acc / total) if total else None,
           "device": torch.cuda.get_device_name(0), "power_limit": power[0] if power else None}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
