"""Same-GPU, same-process A/B of the fused point kernel under different environment switches.

    python tools/kbench.py [--res 256] [--precision f16f8] [--reps 5] [--rounds 2] "DISN_TC_CORR=0xFF" "DISN_TC_CORR=0xDF" ...

The C library reads its switches with getenv() at launch time, so one process (weights loaded once, image encoded once) can
interleave all configurations.  Prints the mean kernel time per configuration and round (CUDA events on the launching stream).
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--precision", default="f16f8")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("configs", nargs="+")
    a = ap.parse_args()
    import torch
    from disn_b200 import synth
    from disn_b200.engine import Engine
    dev = torch.device("cuda", 0)
    eng = Engine(device=0, precision=a.precision, max_batch=1)
    eng.load_weights(synth.make_weights(seed=7, init="he"))
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    eng.set_stream(stream.cuda_stream)
    img = torch.from_numpy(synth.synthetic_images(1)).to(dev)
    tm = torch.from_numpy(synth.DEMO_TRANS_MAT.copy()).to(dev)
    R = a.res + 1
    out = torch.empty((R, R, R), dtype=torch.float32, device=dev)
    eng.encode_device(img.data_ptr(), 1, 137, 137, 3)
    keys = set()
    for c in a.configs:
        keys.update(kv.split("=")[0] for kv in c.split(",") if kv)
    for rnd in range(a.rounds):
        for c in a.configs:
            for k in keys:
                os.environ.pop(k, None)
            for kv in c.split(","):
                if kv:
                    k, v = kv.split("=")
                    os.environ[k] = v
            for _ in range(2):
                eng.eval_grid_device(synth.DEMO_SDF_PARAMS, tm.data_ptr(), a.res, 0, R, out.data_ptr())
            torch.cuda.synchronize(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.reps):
                eng.eval_grid_device(synth.DEMO_SDF_PARAMS, tm.data_ptr(), a.res, 0, R, out.data_ptr())
            e1.record(stream)
            torch.cuda.synchronize(dev)
            ms = e0.elapsed_time(e1) / a.reps
            chk = float(out.double().abs().sum().item())
            print("round %d  %-44s %8.3f ms   %.4g pts/s   checksum %.6e" % (rnd, c, ms, R ** 3 / ms * 1e3, chk), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
