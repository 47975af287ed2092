"""Max |sdf - oracle64| of the tensor-core point kernel per precision mode on N random points per image (2 images).
    python tests/err_report.py [N]
Test infrastructure (it calls the oracle as the checker), hence under tests/."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from disn_b200 import synth
from disn_b200.engine import Engine
from oracle import disn_oracle as orc

N = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 20000
W = synth.make_weights(seed=7, init="he")
imgs = synth.synthetic_images(2, seed=1234)
enc = orc.encode(imgs, W, dtype=np.float64)
tm = np.concatenate([synth.DEMO_TRANS_MAT, synth.synthetic_trans_mats(1)], axis=0)
pts = np.random.default_rng(5).uniform(-1, 1, size=(2, N, 3)).astype(np.float32)
ref = orc.decode(enc, pts, pts, tm, W, dtype=np.float64)["pred_sdf"]


def report(tag, eng):
    e = np.abs(eng.eval_points(pts, tm) - ref) / 10.0
    print("%-14s max %.3e  rms %.3e  p99.99 %.3e" % (tag, e.max(), np.sqrt((e ** 2).mean()), np.quantile(e, 0.9999)), flush=True)


eng = Engine(device=0, precision="bf16x3", max_batch=2)
eng.load_weights(W)
eng.encode(imgs)
report("bf16x3", eng)
eng.set_precision("f16f8")
report("f16f8", eng)
eng.close()
