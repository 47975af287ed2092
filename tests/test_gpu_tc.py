"""GPU tests of the warpgroup-MMA building blocks and the tensor-core point and encoder kernels."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _bf16_round(x):
    """round-to-nearest-even to bfloat16, returned as float32"""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32)


@pytest.mark.parametrize("passes", [1, 2])
def test_wgmma_gemm_layout(passes):
    """D = A.B^T through m64n128 warpgroup MMAs on SW128 K-major tiles (A written by threads, B by the bulk-copy engine),
    read back through the accumulator fragment layout the kernels assume: D_out[c, 64h + r, j] = D[64c + r, 128h + j]."""
    from disn_b200 import _lib
    lib = _lib.load_test()
    rng = np.random.default_rng(42)
    A = rng.standard_normal((128, 64)).astype(np.float32)
    B = rng.standard_normal((256, 64)).astype(np.float32)
    D = np.empty((2, 128, 128), np.float32)
    _lib.check(lib.disn_tc_selftest(0, A.ctypes.data_as(C.c_void_p), B.ctypes.data_as(C.c_void_p), passes,
                                    D.ctypes.data_as(C.c_void_p)))
    ref = passes * (_bf16_round(A).astype(np.float64) @ _bf16_round(B).astype(np.float64).T)   # [128,256]
    got = np.empty((128, 256), np.float64)
    for c in range(2):
        for h in range(2):
            got[c * 64:(c + 1) * 64, h * 128:(h + 1) * 128] = D[c, h * 64:(h + 1) * 64, :]
    assert np.isfinite(got).all()
    assert np.abs(got - ref).max() < 1e-3 * np.abs(ref).max()


@pytest.fixture(scope="module")
def tc_engine(he_weights):
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="bf16x3", max_batch=2)
    eng.load_weights(he_weights)
    yield eng
    eng.close()


@pytest.mark.parametrize("n", [1, 64, 127, 128, 129, 1000, 20000])
def test_tc_eval_points_matches_oracle(tc_engine, he_weights, n):
    """bf16x3 tensor-core path vs the fp64 oracle: |sdf - ref| <= 1e-4 (north_star tolerance)."""
    from disn_b200 import synth
    from oracle import disn_oracle as orc
    imgs = synth.synthetic_images(2, seed=1234)
    tc_engine.encode(imgs)
    enc = orc.encode(imgs, he_weights, dtype=np.float64)
    rng = np.random.default_rng(200 + n)
    pts = rng.uniform(-1, 1, size=(2, n, 3)).astype(np.float32)
    tm = np.concatenate([synth.DEMO_TRANS_MAT, synth.synthetic_trans_mats(1)], axis=0)
    pred, uv = tc_engine.eval_points(pts, tm, want_uv=True)
    nref = min(n, 3000)      # keep the CPU oracle in seconds
    ref = orc.decode(enc, pts[:, :nref], pts[:, :nref], tm, he_weights, dtype=np.float64)
    np.testing.assert_allclose(uv[:, :nref], ref["sample_img_points"], rtol=0, atol=2e-4)
    err = np.abs(pred[:, :nref] - ref["pred_sdf"]).max() / orc.SDF_WEIGHT
    assert err <= 1e-4, err
    if n > nref:     # the rest against the fp32 CUDA-core path
        tc_engine.set_precision("fp32")
        p32 = tc_engine.eval_points(pts, tm)
        tc_engine.set_precision("bf16x3")
        assert np.abs(pred - p32).max() / orc.SDF_WEIGHT <= 1e-4


def test_tc_grid_matches_fp32_path_and_slabs(tc_engine):
    from disn_b200 import synth
    from oracle import disn_oracle as orc
    imgs = synth.synthetic_images(1, seed=5)
    tc_engine.encode(imgs)
    tm = synth.DEMO_TRANS_MAT
    sp = np.array([[-1.0, -0.9, -0.8, 1.0, 0.7, 0.9]])
    g_tc = tc_engine.eval_grid(sp, tm, 40)
    tc_engine.set_precision("fp32")
    g_32 = tc_engine.eval_grid(sp, tm, 40)
    tc_engine.set_precision("bf16x3")
    assert g_tc.shape == (1, 41, 41, 41)
    err = np.abs(g_tc - g_32).max()
    rms = np.sqrt(np.mean(g_32.astype(np.float64) ** 2))
    assert err <= 1e-4, (err, rms)
    assert rms > 0.02          # the field is O(0.1): the bar is not vacuous
    a = tc_engine.eval_grid(sp, tm, 40, z0=0, z1=17)
    b = tc_engine.eval_grid(sp, tm, 40, z0=17, z1=41)
    np.testing.assert_array_equal(np.concatenate([a, b], axis=1), g_tc)   # deterministic, slab-invariant


def test_full_size_grid_properties(tc_engine):
    """BASELINE config 1 at full size (257^3 = 16 974 593 points): size-independent properties instead of the
    CPU oracle -- (i) tensor-core path within 1e-4 of the fp32 CUDA-core path everywhere, (ii) bitwise
    run-to-run determinism, (iii) z-slab sharding (the multi-GPU decomposition) reproduces the single call."""
    from disn_b200 import synth
    imgs = synth.synthetic_images(1)
    tc_engine.encode(imgs)
    tm, sp = synth.DEMO_TRANS_MAT, synth.DEMO_SDF_PARAMS
    g1 = tc_engine.eval_grid(sp, tm, 256)
    assert g1.shape == (1, 257, 257, 257) and np.isfinite(g1).all()
    g2 = tc_engine.eval_grid(sp, tm, 256)
    np.testing.assert_array_equal(g1, g2)
    slabs = [tc_engine.eval_grid(sp, tm, 256, z0=a, z1=b) for a, b in ((0, 32), (32, 129), (129, 257))]
    np.testing.assert_array_equal(np.concatenate(slabs, axis=1), g1)
    tc_engine.set_precision("fp32")
    g32 = tc_engine.eval_grid(sp, tm, 256)
    tc_engine.set_precision("bf16x3")
    err = float(np.abs(g1 - g32).max())
    rms = float(np.sqrt(np.mean(g32.astype(np.float64) ** 2)))
    assert err <= 1e-4, (err, rms)
    assert rms > 0.02


def test_batch_of_eight_images(he_weights):
    """BASELINE config 2 shape: batch = 8 images through one encode + one grid call; spot-check two of them."""
    from disn_b200 import synth
    from disn_b200.engine import Engine
    from oracle import disn_oracle as orc
    eng = Engine(device=0, precision="bf16x3", max_batch=8)
    try:
        eng.load_weights(he_weights)
        imgs = synth.synthetic_images(8, seed=500)
        tms = synth.synthetic_trans_mats(8, seed=600)
        sps = np.tile(synth.DEMO_SDF_PARAMS, (8, 1))
        eng.encode(imgs)
        grid = eng.eval_grid(sps, tms, 10)
        assert grid.shape == (8, 11, 11, 11)
        for b in (0, 7):
            ref = orc.create_sdf_grid(imgs[b:b + 1], tms[b:b + 1], sps[b:b + 1], he_weights, sdf_res=10, dtype=np.float64)
            assert np.abs(grid[b].reshape(-1) - ref.reshape(-1)).max() <= 1e-4
    finally:
        eng.close()


def test_tc_encoder_matches_oracle(tc_engine, he_weights):
    """Encoder GEMMs on the tensor cores (bf16 hi/lo split): taps, embedding and folded products vs the fp64 oracle."""
    from disn_b200 import synth
    from oracle import disn_oracle as orc
    imgs = synth.synthetic_images(2, seed=4321)
    tc_engine.encode(imgs)
    enc = orc.encode(imgs, he_weights, dtype=np.float64)
    for i, tap in enumerate(orc.VGG_TAPS):
        got, ref = tc_engine.get_encoded(1 + i), enc.vgg_end_points[tap]
        assert np.abs(got - ref).max() <= 5e-5 * np.abs(ref).max(), tap
    emb = tc_engine.get_encoded(0)
    assert np.abs(emb - enc.img_embedding).max() <= 5e-5 * np.abs(enc.img_embedding).max()
    Wl = he_weights["sdfprediction_imgfeat/fold2/conv1/weights"].reshape(-1, 512).astype(np.float64)
    off, pmap = 512, 0
    for m, c in zip(enc.maps, orc.TAP_CHANNELS):
        pmap = pmap + m @ Wl[off:off + c]
        off += c
    got = tc_engine.get_encoded(6)
    assert np.abs(got - pmap).max() <= 5e-5 * np.abs(pmap).max()


@pytest.mark.parametrize("mode", [1, 2, 3])
def test_wgmma_f16_e5m2_split_accumulation(mode):
    """fp16 (SW128) and e5m2 (SW64) warpgroup MMAs summed into one fp32 result, as in DISN_PREC_F16F8.  The fp16 part
    accumulates in fp32; Hopper's e5m2 MMAs align each group's products to the largest one and keep ~14 bits, so their part
    is held to 2^-12 of the sum of |products| (the point kernel gives them their own accumulator for that reason)."""
    from disn_b200 import _lib
    lib = _lib.load_test()
    rng = np.random.default_rng(mode)
    A16 = rng.standard_normal((128, 64)).astype(np.float32)
    B16 = rng.standard_normal((256, 64)).astype(np.float32)
    A8 = (rng.standard_normal((128, 64)) * 2.0 ** -6).astype(np.float32)
    B8 = (rng.standard_normal((256, 64)) * 2.0 ** 3).astype(np.float32)
    A8q, B8q = np.empty_like(A8), np.empty_like(B8)
    D = np.empty((2, 128, 128), np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(lib.disn_tc_selftest_mixed(0, p(A16), p(B16), p(A8), p(B8), mode, p(A8q), p(B8q), p(D)))
    assert np.abs(A8q - A8).max() <= 0.125 * np.abs(A8).max() + 2.0 ** -17      # e5m2: 2 mantissa bits
    ref = np.zeros((128, 256))
    if mode & 1:
        ref += A16.astype(np.float16).astype(np.float64) @ B16.astype(np.float16).astype(np.float64).T
    if mode & 2:
        ref += A8q.astype(np.float64) @ B8q.astype(np.float64).T
    got = np.empty((128, 256), np.float64)
    for c in range(2):
        for h in range(2):
            got[c * 64:(c + 1) * 64, h * 128:(h + 1) * 128] = D[c, h * 64:(h + 1) * 64, :]
    assert np.isfinite(got).all()
    bound = 2e-6 * max(1.0, np.abs(ref).max()) * 8
    if mode & 2:
        bound = bound + 2.0 ** -12 * (np.abs(A8q).astype(np.float64) @ np.abs(B8q).astype(np.float64).T)
    assert (np.abs(got - ref) < bound).all()


# ---------------------------------------------------------------------------------------------------------
# DISN_PREC_F16F8: fp16 product + two e5m2 correction products
# ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def f8_engine(he_weights):
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="f16f8", max_batch=2)
    eng.load_weights(he_weights)
    yield eng
    eng.close()


@pytest.mark.parametrize("n", [1, 127, 129, 3000, 20000])
def test_f16f8_eval_points_matches_oracle(f8_engine, he_weights, n):
    """f16f8 path vs the fp64 oracle: |sdf - ref| <= 1e-4 (north_star tolerance)."""
    from disn_b200 import synth
    from oracle import disn_oracle as orc
    imgs = synth.synthetic_images(2, seed=1234)
    f8_engine.encode(imgs)
    enc = orc.encode(imgs, he_weights, dtype=np.float64)
    rng = np.random.default_rng(300 + n)
    pts = rng.uniform(-1, 1, size=(2, n, 3)).astype(np.float32)
    tm = np.concatenate([synth.DEMO_TRANS_MAT, synth.synthetic_trans_mats(1)], axis=0)
    pred = f8_engine.eval_points(pts, tm)
    nref = min(n, 3000)
    ref = orc.decode(enc, pts[:, :nref], pts[:, :nref], tm, he_weights, dtype=np.float64)
    err = np.abs(pred[:, :nref] - ref["pred_sdf"]).max() / orc.SDF_WEIGHT
    print("f16f8 max |sdf - oracle64| =", err)
    assert err <= 1e-4, err
    if n > nref:
        f8_engine.set_precision("fp32")
        p32 = f8_engine.eval_points(pts, tm)
        f8_engine.set_precision("f16f8")
        assert np.abs(pred - p32).max() / orc.SDF_WEIGHT <= 1e-4


def test_f16f8_full_size_grid_properties(f8_engine):
    """257^3 grid: within 1e-4 of the fp32 CUDA-core path everywhere, deterministic, slab-invariant."""
    from disn_b200 import synth
    imgs = synth.synthetic_images(1)
    f8_engine.encode(imgs)
    tm, sp = synth.DEMO_TRANS_MAT, synth.DEMO_SDF_PARAMS
    g1 = f8_engine.eval_grid(sp, tm, 256)
    assert np.isfinite(g1).all()
    np.testing.assert_array_equal(g1, f8_engine.eval_grid(sp, tm, 256))
    slabs = [f8_engine.eval_grid(sp, tm, 256, z0=a, z1=b) for a, b in ((0, 100), (100, 257))]
    np.testing.assert_array_equal(np.concatenate(slabs, axis=1), g1)
    f8_engine.set_precision("fp32")
    g32 = f8_engine.eval_grid(sp, tm, 256)
    f8_engine.set_precision("f16f8")
    err = float(np.abs(g1 - g32).max())
    print("f16f8 257^3 max |sdf - fp32 path| =", err)
    assert err <= 1e-4, err


def test_res512_grid_config4(f8_engine):
    """BASELINE config 4 shape (--sdf_res 512: 513^3 = 135 005 697 points, 540 MB of SDF): finite, identical under a
    different slab decomposition, and within 1e-4 of the fp32 CUDA-core path on sampled planes."""
    from disn_b200 import synth
    imgs = synth.synthetic_images(1)
    f8_engine.encode(imgs)
    tm, sp = synth.DEMO_TRANS_MAT, synth.DEMO_SDF_PARAMS
    R = 513
    g = f8_engine.eval_grid(sp, tm, 512)
    assert g.shape == (1, R, R, R) and np.isfinite(g).all()
    top = f8_engine.eval_grid(sp, tm, 512, z0=0, z1=200)
    np.testing.assert_array_equal(top, g[:, :200])
    del top
    f8_engine.set_precision("fp32")
    try:
        for z in (0, 256, 511):
            ref = f8_engine.eval_grid(sp, tm, 512, z0=z, z1=z + 2)
            assert float(np.abs(ref - g[:, z:z + 2]).max()) <= 1e-4
    finally:
        f8_engine.set_precision("f16f8")


def test_res512_mesh_chamfer_parity(f8_engine):
    """BASELINE config 4: --sdf_res 512 grid -> CUDA marching cubes; the mesh of the tensor-core SDF must coincide with the
    mesh of the fp32 CUDA-core SDF: every sampled vertex has a counterpart within a small fraction of the lattice spacing
    (2/512), and the two Chamfer terms (test/test_cd_emd.py:300-301) of 2048-vertex samples against the other mesh vanish."""
    from disn_b200 import synth
    f8_engine.encode(synth.synthetic_images(1))
    tm, sp = synth.DEMO_TRANS_MAT, synth.DEMO_SDF_PARAMS
    bbox = [-1, -1, -1, 1, 1, 1]
    g_tc = f8_engine.eval_grid(sp, tm, 512)[0]
    f8_engine.set_precision("fp32")
    try:
        g_32 = f8_engine.eval_grid(sp, tm, 512)[0]
    finally:
        f8_engine.set_precision("f16f8")
    assert float(np.abs(g_tc - g_32).max()) <= 1e-4
    iso = float(np.median(g_32[::8, ::8, ::8]))
    v_tc, f_tc = f8_engine.marching_cubes(g_tc, bbox, iso)
    v_32, f_32 = f8_engine.marching_cubes(g_32, bbox, iso)
    assert len(f_32) > 10000 and abs(len(f_tc) - len(f_32)) <= 0.01 * len(f_32)
    rng = np.random.default_rng(0)
    a = v_tc[rng.choice(len(v_tc), 2048, replace=False)][None]
    b = v_32[rng.choice(len(v_32), 2048, replace=False)][None]
    d_ab = f8_engine.nn_distance(a, v_32[None])[0]          # sampled tc vertices -> all fp32-path vertices
    d_ba = f8_engine.nn_distance(b, v_tc[None])[0]
    spacing = 2.0 / 512
    cd_x1000 = float((d_ab.mean() + d_ba.mean()) * 1000)
    q99 = float(np.sqrt(max(np.quantile(d_ab, 0.99), np.quantile(d_ba, 0.99))))
    print("res-512 meshes: %d / %d faces, CD x1000 = %.3e, 99%% NN distance = %.3e, max = %.3e (lattice spacing %.3e)"
          % (len(f_tc), len(f_32), cd_x1000, q99, float(np.sqrt(max(d_ab.max(), d_ba.max()))), spacing))
    # where the synthetic field is flat around the iso level a 1e-5 SDF difference moves the crossing by whole cells, so the
    # bar is on the metric the reference reports (mean) and on the bulk of the vertices, not on the single worst one
    assert q99 < 0.25 * spacing
    assert cd_x1000 < 1e-3          # reference CD x1000 values are O(1): parity to three orders below its resolution
