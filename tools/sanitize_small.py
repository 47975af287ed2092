"""Tiny end-to-end run for compute-sanitizer (memcheck / racecheck): every entry point that owns device memory, on one
context per precision.  The decoder calls run before and after a first, larger nn_distance, so a scratch buffer that one
call releases while another still uses it shows up as an invalid access."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from disn_b200 import synth
from disn_b200.engine import Engine
from oracle import disn_oracle as orc

BOX = [-1, -1, -1, 1, 1, 1]
W = synth.make_weights(seed=7, init="he")
rng = np.random.default_rng(3)
for name, shp in orc.cam_head_shapes().items():
    W[name] = (rng.standard_normal(shp) * (0.02 if name.endswith("biases") else np.sqrt(2.0 / shp[0]))).astype(np.float32)
for prec in (sys.argv[1:] or ["fp32", "bf16x3", "f16f8"]):
    eng = Engine(device=0, precision=prec)
    eng.load_weights(W)
    imgs = synth.synthetic_images(1)
    tm = synth.DEMO_TRANS_MAT
    eng.encode(imgs)
    pts = np.random.default_rng(0).uniform(-1, 1, (1, 300, 3)).astype(np.float32)   # 3 pair-tiles: ring wrap-around, tail tile
    out = eng.eval_points(pts, tm)
    gfeat = rng.standard_normal((1, 1024)).astype(np.float32)
    pfeat = rng.standard_normal((1, 300, 1472)).astype(np.float32)
    for _ in range(2):       # the decoder scratch before and after the nn scratch grows
        eng.eval_points_ex(pts, tm)
        eng.point_img_feat(pts, tm)
        eng.eval_features(pts, gfeat, pfeat)
        eng.nn_distance(rng.uniform(-1, 1, (2, 512, 3)), rng.uniform(-1, 1, (2, 384, 3)))
    g = eng.eval_grid(synth.DEMO_SDF_PARAMS, tm, 8)
    gd = eng.fetch(eng.eval_grid_resident(synth.DEMO_SDF_PARAMS, tm, 8), (1, 9, 9, 9))
    v, f = eng.marching_cubes(g[0], BOX, float(np.median(g)))
    eng.load_mesh(v, f)
    cv, cf = eng.clean_mesh(0.5, 0.0)
    eng.iou(v, f, v, f, dim=32)
    a, b = rng.uniform(-1, 1, (1, 64, 3)), rng.uniform(-1, 1, (1, 48, 3))
    match, cost = eng.approx_match(a, b, cost=True)
    eng.match_cost(a, b, match)
    eng.cam_estimate(imgs)
    print(prec, float(out.mean()), g.shape, bool(np.array_equal(g, gd)), v.shape, f.shape, cf.shape, float(cost[0]))
    eng.close()
