"""Shape sweeps of the kernels around the fused point kernel, against exact references:
  A. the encoder GEMMs (fp32 CUDA-core gemm_f32_kernel + splitk_reduce_kernel, bf16x3 wgmma conv_tc_kernel) through the
     disn_debug_gemm harness, element-wise against float64 with bounds relative to S = |A| @ |W| + |b|;
  B. the explicit-feature decoder (get_decoder) on both sides of its 23-way split-K projection;
  C. IoU at dims above the former fixed voxel window;
  D. marching cubes and small-part cleaning at sizes where their scans recurse.
The float64 references and split rules live in tests/test_shapes_cpu.py."""
import ctypes as C
import itertools
import time
import zlib

import numpy as np
import pytest

from disn_b200 import synth
from oracle import disn_oracle as orc
from oracle import mc_oracle
from oracle import mesh_clean_oracle as mco
from oracle import metrics_oracle as mo
from tests.test_gpu_surface import _icosphere
from tests.test_shapes_cpu import (FP32_BOUND, TC_BOUND, as_matrix, edge_triangles, far_triangle, fp32_splits, gemm_ref,
                                   make_case, ratio, tc_splits, unwindowed, within)

pytestmark = pytest.mark.gpu

BOX = [-1, -1, -1, 1, 1, 1]


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ----------------------------------------------------------------------------------------------------------------------
# A. encoder GEMM sweep
# ----------------------------------------------------------------------------------------------------------------------
# Plain GEMMs, every (M, N, K) of the grid; (relu, bias) cycle through all four combinations along the grid.  With
# 132 SMs the grid reaches (fp32 splits, tensor-core splits):
#   K = 64             -> (1, 1): a single K slice, nothing to split
#   K = 1472, M <= 256 -> (23, 23) for N = 512: 23 slices, a prime, split 23 ways by both kernels
#   K = 1472, M = 514  -> (8, 1) for N = 512: the fp32 kernel splits along K/8, the tensor cores cannot split 23 slices
#   K = 4608, M = 3001 -> (4, 3) for N = 512: both split, the m-tiles end in a partial one of 57 rows
# and M = 4225 (33 full m-tiles and one row) at N = 512 has 136 tiles: no split in either kernel with a long K.
PLAIN = [dict(shape=m, N=n, K=k) for m, n, k in itertools.product((1, 127, 128, 129, 514, 3001), (64, 192, 512),
                                                                   (64, 1472, 4608))]
PLAIN.append(dict(shape=4225, N=512, K=1472))
for i, c in enumerate(PLAIN):
    c.update(relu=i % 2, bias=(i // 2) % 2, positive=i % 3 == 1)
# im2col: (B, H, W, Cin) -> Cout.  A 1x1 image (every tap but the centre is padding), H != W with border-only rows
# (3 x 17), m-tiles that span images (7 x 5 = 35 pixels per image), and the VGG sizes 14/28/56; each once with ReLU and
# bias, once linear without bias on strictly positive activations.
IM2COL = [((1, 1, 1, 64), 64), ((1, 3, 17, 64), 128), ((2, 7, 5, 128), 64), ((3, 14, 14, 512), 512),
          ((1, 28, 28, 256), 512), ((2, 56, 56, 128), 128)]
CONV = [dict(shape=s, N=n, K=9 * s[3], relu=r, bias=r, positive=True) for s, n in IM2COL for r in (1, 0)]
CASES = PLAIN + CONV


def _case_id(c):
    geo = ("M%d" % c["shape"]) if np.isscalar(c["shape"]) else "x".join(map(str, c["shape"]))
    return "%s_N%d_K%d_r%d_b%d%s" % (geo, c["N"], c["K"], c["relu"], c["bias"], "_pos" if c["positive"] else "")


def _rows(c):
    s = c["shape"]
    return s if np.isscalar(s) else s[0] * s[1] * s[2]


@pytest.fixture(scope="module")
def dbg():
    """a context of the diagnostics library (it carries its own copy of the code: handles do not cross libraries)"""
    from disn_b200 import _lib
    lib = _lib.load_test()
    cfg = _lib.DisnConfig()
    lib.disn_default_config(C.byref(cfg))
    cfg.device, cfg.precision = 0, _lib.PREC_FP32
    h = C.c_void_p()
    if lib.disn_create(C.byref(cfg), C.byref(h)):
        raise RuntimeError(lib.disn_last_error().decode())
    yield lib, h
    lib.disn_destroy(h)


def _debug_gemm(dbg, c, A, Wt, b):
    lib, h = dbg
    M, N, K = _rows(c), c["N"], c["K"]
    H, Wd, Cin = (0, 0, 0) if A.ndim == 2 else A.shape[1:]
    o32, otc = np.empty((M, N), np.float32), np.empty((M, N), np.float32)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    l0 = lib.disn_launch_count(h)
    if lib.disn_debug_gemm(h, p(A), p(Wt), p(b), M, N, K, H, Wd, Cin, c["relu"], p(o32), p(otc)):
        raise RuntimeError(lib.disn_last_error().decode())
    return o32, otc, lib.disn_launch_count(h) - l0


def test_gemm_sweep_reaches_every_split_case():
    """no split, split-K in the fp32 kernel, split-K in the wgmma kernel, and the 23-way split (per-case launch counts
    confirm the modelled split decisions)"""
    sms = _sms()
    got = [(fp32_splits(_rows(c), c["N"], c["K"], sms), tc_splits(_rows(c), c["N"], c["K"], sms)) for c in CASES]
    print("split cases on %d SMs:" % sms, sorted(set(got)))
    assert any(f == 1 and t == 1 and c["K"] > 64 for (f, t), c in zip(got, CASES))
    assert any(f > 1 for f, _ in got) and any(t > 1 for _, t in got)
    assert any(f > 1 and t == 1 for f, t in got)
    assert any(f == 23 for f, _ in got) and any(t == 23 for _, t in got)


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_encoder_gemm_matches_float64(dbg, case):
    c = case
    A, Wt, b = make_case(c["shape"], c["N"], c["K"], c["relu"], c["bias"], c["positive"], seed=zlib.crc32(_case_id(c).encode()))
    M, N, K = _rows(c), c["N"], c["K"]
    sms = _sms()
    fs, ts = fp32_splits(M, N, K, sms), tc_splits(M, N, K, sms)
    o32, otc, launches = _debug_gemm(dbg, c, A, Wt, b)
    assert launches == 2 + (fs > 1) + (ts > 1), (launches, fs, ts)
    r32, rtc, _ = _debug_gemm(dbg, c, A, Wt, b)
    np.testing.assert_array_equal(o32, r32)                        # fixed reduction order: bitwise repeatable
    np.testing.assert_array_equal(otc, rtc)
    ref, S = gemm_ref(as_matrix(A) if A.ndim == 4 else A, Wt, b, c["relu"])
    assert np.isfinite(o32).all() and np.isfinite(otc).all()      # the harness fills the output with NaN first
    e32, etc = ratio(o32, ref, S), ratio(otc, ref, S)
    print("gemm %-34s fp32 split %2d  worst err/S %.3e (2^%.1f) | bf16x3 split %2d  worst err/S %.3e (2^%.1f)"
          % (_case_id(c), fs, e32, np.log2(max(e32, 1e-300)), ts, etc, np.log2(max(etc, 1e-300))))
    assert within(o32, ref, S, FP32_BOUND, 1e-30), e32
    assert within(otc, ref, S, TC_BOUND), etc
    if c["relu"]:
        pos = float((ref > 0).mean())
        assert 0.05 < pos < 0.6, pos                              # negative-mean data, but not all clipped


# ----------------------------------------------------------------------------------------------------------------------
# B. explicit-feature decoder at its split shapes
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def feature_scale(he_weights):
    """embedding mean/std and per-channel RMS of point features from a real encode of the synthetic network"""
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="fp32")
    try:
        eng.load_weights(he_weights)
        eng.encode(synth.synthetic_images(1, seed=17))
        emb = eng.get_encoded(0).astype(np.float64)
        pts = np.random.default_rng(18).uniform(-1, 1, (1, 4000, 3)).astype(np.float32)
        feat = eng.point_img_feat(pts, synth.DEMO_TRANS_MAT)[0].reshape(-1, 1472).astype(np.float64)
    finally:
        eng.close()
    return float(emb.mean()), float(emb.std()), np.sqrt((feat ** 2).mean(axis=0))


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "f16f8"])
def test_feature_decoder_split_shapes(he_weights, feature_scale, precision):
    """(B, N) on both sides of the 23-way split of the K = 1472 projection: up to B*N = 256 rows the tensor cores split it
    23 ways, at 257 rows not at all; the fp32 kernel splits 23 ways up to 384 rows; 8 x 4099 rows fill the GPU unsplit.
    pred, global and local each against the float64 oracle heads.  The context is fresh: get_decoder needs no encode (its
    first call used to write the global stream's GEMV partial sums through the not yet allocated encoder buffer)."""
    from disn_b200.engine import Engine
    emb_mean, emb_std, feat_rms = feature_scale
    bar = 1e-5 if precision == "fp32" else 1e-4
    sms = _sms()
    eng = Engine(device=0, precision=precision, max_batch=8)
    try:
        eng.load_weights(he_weights)
        launches = {}
        for B, N in ((1, 1), (1, 63), (1, 256), (2, 128), (1, 257), (8, 4099)):
            rng = np.random.default_rng(B * 10007 + N)
            rot = rng.uniform(-1, 1, (B, N, 3)).astype(np.float32)
            g = (emb_mean + emb_std * rng.standard_normal((B, 1024))).astype(np.float32)
            pf = (np.abs(rng.standard_normal((B, N, 1472))) * feat_rms).astype(np.float32)
            l0 = eng.launch_count
            pred, og, ol = eng.eval_features(rot, g.reshape(B, 1, 1, 1024), pf.reshape(B, N, 1, 1472))
            launches[(B, N)] = eng.launch_count - l0
            chunks = range(0, N, 1024)           # the heads are per point: chunked to bound the float64 temporaries
            rg = np.concatenate([orc.get_sdf_basic2(rot[:, i:i + 1024], g, he_weights, dtype=np.float64)
                                 for i in chunks], axis=1)
            rl = np.concatenate([orc.get_sdf_basic2_imgfeat_twostream(rot[:, i:i + 1024], pf[:, i:i + 1024], he_weights,
                                                                      dtype=np.float64) for i in chunks], axis=1)
            errs = [float(np.abs(got - ref).max()) / orc.SDF_WEIGHT for got, ref in ((pred, rg + rl), (og, rg), (ol, rl))]
            print("eval_features %-6s B=%d N=%-5d rows %-6d splits fp32 %2d / tc %2d: max |err|/10 pred %.2e global %.2e "
                  "local %.2e (|local| max %.2f)" % (precision, B, N, B * N, fp32_splits(B * N, 512, 1472, sms),
                                                     tc_splits(B * N, 512, 1472, sms), *errs, float(np.abs(rl).max())))
            assert max(errs) <= bar, errs
        # the projection's split-K reduce is the only launch that differs between 256 and 257 rows
        split_at = lambda m: (tc_splits if precision != "fp32" else fp32_splits)(m, 512, 1472, sms) > 1
        assert launches[(1, 256)] - launches[(1, 257)] == int(split_at(256)) - int(split_at(257)), launches
    finally:
        eng.close()


# ----------------------------------------------------------------------------------------------------------------------
# C. IoU above the former fixed voxel window
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [110, 128, 256, 512])
def test_iou_window_matches_oracle(dim):
    """occupancy grids and counts == the CPU twin, and the twin == an unwindowed voxelisation, for a sphere of radius
    0.97 and triangles straddling both binning edges on every axis; two far-away triangles (+-1e9) contribute nothing and
    must not overflow the cell-range cast.  The former fixed window kept 0 of the sphere's bins at dim 512.  At dim 512 the
    two CPU voxelisations take about 80 s together; the size is the point of the test, so it stays."""
    from disn_b200.engine import Engine
    sphere = _icosphere(0.97, (0.0, 0.0, 0.0), sub=3)
    assert (np.abs(sphere[0]).max(axis=0) > 0.95).all()
    ev, ef = edge_triangles()
    fv, ff = far_triangle()
    near = (np.concatenate([ev, fv]), np.concatenate([ef, ff + len(ev)]))
    out = np.array([[1e9, 1e9, 1e9], [1.1e9, 1e9, 1e9], [1e9, 1.1e9, 1e9]], np.float32)
    edges = (np.concatenate([near[0], out, -out]), np.concatenate([near[1], np.array([[0, 1, 2], [3, 4, 5]]) + len(near[0])]))
    eng = Engine(device=0, precision="fp32")
    try:
        t0 = time.perf_counter()
        iou, inter, uni, o1, o2 = eng.iou(*sphere, *edges, dim=dim, want_grids=True)
        t_gpu = time.perf_counter() - t0
        t0 = time.perf_counter()
        r1, r2 = mo.voxel_occupancy(*sphere, dim), mo.voxel_occupancy(*edges, dim)
        t_cpu = time.perf_counter() - t0
        np.testing.assert_array_equal(o1, r1)
        np.testing.assert_array_equal(o2, r2)
        np.testing.assert_array_equal(r1, unwindowed(*sphere, dim))
        np.testing.assert_array_equal(r2, unwindowed(*near, dim))     # the far triangles are outside any useful window
        assert (inter, uni) == (int(np.logical_and(r1, r2).sum()), int(np.logical_or(r1, r2).sum()))
        for axis in range(3):                    # the sphere reaches |x| = 0.95 on every axis, the triangles both edges
            p1 = r1.any(axis=tuple(a for a in range(3) if a != axis))
            assert p1[int((-0.95 + 1.1) / 2.4 * dim)] and p1[int((0.95 + 1.1) / 2.4 * dim)]
            p2 = r2.any(axis=tuple(a for a in range(3) if a != axis))
            assert p2[0] and p2[dim - 1]
        s = eng.iou(*sphere, *sphere, dim=dim)
        assert s == 1.0
        print("iou dim %d: %d + %d occupied bins, inter %d, union %d; GPU %.2f s, CPU twin %.2f s"
              % (dim, int(r1.sum()), int(r2.sum()), inter, uni, t_gpu, t_cpu))
    finally:
        eng.close()


# ----------------------------------------------------------------------------------------------------------------------
# D. marching cubes and cleaning where their scans recurse
# ----------------------------------------------------------------------------------------------------------------------
def test_marching_cubes_257_predicted_grid_bit_exact(engine):
    """The 257^3 grid of the synthetic network (demo image and camera, iso = median): 8288 chunks of 2048 points, so the
    chunk-total scan recurses; faces and vertices bit-identical to the CPU oracle."""
    engine.encode(synth.synthetic_images(1))
    grid = engine.eval_grid(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 256)[0]
    iso = float(np.median(grid))
    t0 = time.perf_counter()
    v, f = engine.marching_cubes(grid, BOX, iso)
    t_gpu = time.perf_counter() - t0
    t0 = time.perf_counter()
    rv, rf = mc_oracle.marching_cubes(grid, BOX, iso)
    t_cpu = time.perf_counter() - t0
    print("marching cubes 257^3: %d verts, %d faces; GPU %.2f s, CPU oracle %.1f s" % (len(v), len(f), t_gpu, t_cpu))
    assert len(f) > 10 ** 5
    np.testing.assert_array_equal(f, rf)
    np.testing.assert_array_equal(v, rv)


def test_mesh_clean_three_level_scan_bit_exact(engine):
    """The 129^3 standard-normal field meshes to ~6.7 M faces: above 2048^2, so the cleaning's face scans recurse three
    levels.  Faces, vertices, labels and counts bit-identical to the CPU twin."""
    R = 129
    noise = np.random.default_rng(129).standard_normal((R, R, R)).astype(np.float32)
    v, f = engine.marching_cubes(noise, BOX, 0.0)
    assert len(f) > 2048 ** 2
    t0 = time.perf_counter()
    out_v, out_f, labels = engine.clean_mesh(0.5, 0.3, want_labels=True)
    t_gpu = time.perf_counter() - t0
    cnt = engine.last_clean
    t0 = time.perf_counter()
    want = mco.clean(v, f, 0.5, 0.3)
    t_cpu = time.perf_counter() - t0
    print("clean 129^3 noise: %d verts, %d faces, %d components, %d kept; GPU %.2f s, CPU twin %.1f s"
          % (len(v), len(f), cnt.n_components, cnt.n_kept, t_gpu, t_cpu))
    np.testing.assert_array_equal(out_f, want["faces"])
    np.testing.assert_array_equal(out_v, want["verts"])
    np.testing.assert_array_equal(labels, want["labels"])
    assert (cnt.n_components, cnt.n_kept, cnt.n_verts, cnt.n_faces) == (want["n_components"], want["n_kept"],
                                                                        len(want["verts"]), len(want["faces"]))
