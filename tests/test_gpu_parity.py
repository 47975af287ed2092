"""GPU parity tests (run with -m gpu on an H100): the CUDA path through the C ABI against the CPU oracle
on the same seeded inputs.  Tolerance (BASELINE.json north_star): |sdf_gpu - sdf_ref| <= 1e-4 abs on the
SDF value (= pred/10), i.e. 1e-3 on pred; the fp32 path is held to 10x tighter."""
import numpy as np
import pytest

from disn_b200 import synth
from oracle import disn_oracle as orc

pytestmark = pytest.mark.gpu

SDF_TOL = 1e-4          # on pred / SDF_WEIGHT
FP32_TOL = 1e-5         # fp32 CUDA-core path, same unit


@pytest.fixture(scope="module")
def enc_case(engine, he_weights):
    imgs = synth.synthetic_images(2, seed=1234)
    engine.encode(imgs)
    enc = orc.encode(imgs, he_weights, dtype=np.float64)
    return imgs, enc


def test_encoder_matches_oracle(engine, he_weights, enc_case):
    imgs, enc = enc_case
    rs = engine.get_encoded(8)
    np.testing.assert_allclose(rs, orc.tf_resize_bilinear(imgs, 224, 224), rtol=0, atol=1e-6)
    for i, tap in enumerate(orc.VGG_TAPS):
        got = engine.get_encoded(1 + i)
        ref = enc.vgg_end_points[tap]
        scale = np.abs(ref).max()
        assert np.abs(got - ref).max() <= 2e-5 * scale, tap
    emb = engine.get_encoded(0)
    assert np.abs(emb - enc.img_embedding).max() <= 2e-5 * np.abs(enc.img_embedding).max()
    # folded per-image products
    Wg = he_weights["sdfprediction/fold2/conv1/weights"].reshape(-1, 512).astype(np.float64)
    gb = enc.img_embedding @ Wg[512:] + he_weights["sdfprediction/fold2/conv1/biases"]
    assert np.abs(engine.get_encoded(7) - gb).max() <= 2e-5 * np.abs(gb).max()
    Wl = he_weights["sdfprediction_imgfeat/fold2/conv1/weights"].reshape(-1, 512).astype(np.float64)
    off, pmap = 512, 0
    for m, c in zip(enc.maps, orc.TAP_CHANNELS):
        pmap = pmap + m @ Wl[off:off + c]
        off += c
    got = engine.get_encoded(6)
    assert np.abs(got - pmap).max() <= 3e-5 * np.abs(pmap).max()


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000, 4099])
def test_eval_points_matches_oracle(engine, he_weights, enc_case, n):
    imgs, enc = enc_case
    rng = np.random.default_rng(100 + n)
    pts = rng.uniform(-1, 1, size=(2, n, 3)).astype(np.float32)
    tm = np.concatenate([synth.DEMO_TRANS_MAT, synth.synthetic_trans_mats(1)], axis=0)
    pred, uv = engine.eval_points(pts, tm, want_uv=True)
    ref = orc.decode(enc, pts, pts, tm, he_weights, dtype=np.float64)
    assert pred.shape == (2, n, 1) and uv.shape == (2, n, 2)
    np.testing.assert_allclose(uv, ref["sample_img_points"], rtol=0, atol=2e-4)
    err = np.abs(pred - ref["pred_sdf"]).max() / orc.SDF_WEIGHT
    assert err <= FP32_TOL, err


def test_eval_points_separate_rot_input_and_clamping(engine, he_weights, enc_case):
    imgs, enc = enc_case
    rng = np.random.default_rng(5)
    pts = rng.uniform(-3, 3, size=(2, 777, 3)).astype(np.float32)   # many project outside -> clamped
    rot = rng.uniform(-1, 1, size=(2, 777, 3)).astype(np.float32)
    tm = synth.synthetic_trans_mats(2, seed=99)
    pred, uv = engine.eval_points(pts, tm, pts_rot=rot, want_uv=True)
    ref = orc.decode(enc, pts, rot, tm, he_weights, dtype=np.float64)
    assert ((uv == 0) | (uv == 136)).any()
    finite = np.isfinite(ref["pred_sdf"])
    assert np.abs(pred - ref["pred_sdf"])[finite].max() / orc.SDF_WEIGHT <= FP32_TOL


def test_empty_point_list(engine, enc_case):
    tm = synth.synthetic_trans_mats(2)
    out = engine.eval_points(np.zeros((2, 0, 3), np.float32), tm)
    assert out.shape == (2, 0, 1)


def test_eval_grid_matches_reference_loop(engine, he_weights, golden):
    """disn_eval_grid == the reference's chunked loop (create_sdf.py:241-285) on a res-8 and res-16 grid."""
    imgs = synth.synthetic_images(1)
    engine.encode(imgs)
    tm = synth.DEMO_TRANS_MAT
    got8 = engine.eval_grid(synth.DEMO_SDF_PARAMS, tm, 8)
    np.testing.assert_allclose(got8.reshape(1, -1, 1), golden["oracle_small"]["grid_res8"], rtol=0, atol=FP32_TOL)
    sp = np.array([[-1.0, -0.9, -0.8, 1.0, 0.7, 0.9]])
    ref16 = orc.create_sdf_grid(imgs, tm, sp, he_weights, sdf_res=16, dtype=np.float64)
    got16 = engine.eval_grid(sp, tm, 16)
    assert got16.shape == (1, 17, 17, 17)
    assert np.abs(got16.reshape(1, -1, 1) - ref16).max() <= FP32_TOL
    # z-slab calls tile the same array (multi-GPU sharding contract)
    a = engine.eval_grid(sp, tm, 16, z0=0, z1=9)
    b = engine.eval_grid(sp, tm, 16, z0=9, z1=17)
    np.testing.assert_array_equal(np.concatenate([a, b], axis=1), got16)


def test_grid_equals_explicit_points_bitwise(engine, he_weights):
    """In-kernel grid generation is bit-identical to feeding the reference's host-built float32 grid."""
    imgs = synth.synthetic_images(1, seed=3)
    engine.encode(imgs)
    tm = synth.synthetic_trans_mats(1, seed=8)
    sp = np.array([[-0.93, -1.0, -0.71, 1.0, 0.88, 0.97]])
    res = 12
    pts = orc.grid_points(sp[0], res + 1)[None]
    by_pts = engine.eval_points(pts, tm) / np.float32(orc.SDF_WEIGHT)
    by_grid = engine.eval_grid(sp, tm, res)
    np.testing.assert_array_equal(by_grid.reshape(-1), by_pts.reshape(-1))


def test_xavier_reference_init_and_224_input(engine, he_weights):
    """BASELINE config 0's literal random-init condition (xavier/zero) and a 224x224 input (skips the resize)."""
    from disn_b200.engine import Engine
    W = synth.make_weights(seed=11, init="xavier")
    eng = Engine(device=0, precision="fp32")
    try:
        eng.load_weights(W)
        img224 = np.random.default_rng(1).random((1, 224, 224, 3), dtype=np.float32)
        eng.encode(img224)
        pts = np.random.default_rng(2).uniform(-1, 1, size=(1, 500, 3)).astype(np.float32)
        pred = eng.eval_points(pts, synth.DEMO_TRANS_MAT)
        ref = orc.get_model(img224, pts, pts, synth.DEMO_TRANS_MAT, W, dtype=np.float64)["pred_sdf"]
        scale = max(np.abs(ref).max(), 1e-12)
        assert np.abs(pred - ref).max() <= 1e-4 * scale + 1e-7
    finally:
        eng.close()


def test_errors_are_loud(engine):
    from disn_b200._lib import DisnError
    wrong_b = 1 if engine.batch != 1 else 2
    with pytest.raises(DisnError):      # batch differs from the encoded batch
        engine.eval_points(np.zeros((wrong_b, 4, 3), np.float32), synth.DEMO_TRANS_MAT.repeat(wrong_b, 0))
    with pytest.raises(DisnError):
        engine.eval_grid(synth.DEMO_SDF_PARAMS.repeat(engine.batch, 0),
                         synth.DEMO_TRANS_MAT.repeat(engine.batch, 0), 8, z0=5, z1=20)


def test_camera_pose_net_matches_oracle(he_weights):
    """--cam_est path (demo/demo.py:195-258): VGG embedding -> pose heads -> pred_RT . K^T."""
    from disn_b200.engine import Engine
    rng = np.random.default_rng(3)
    W = {k: v for k, v in he_weights.items() if k.startswith("vgg_16/")}
    for name, shp in orc.cam_head_shapes().items():
        W[name] = (rng.standard_normal(shp) * (0.02 if name.endswith("biases") else np.sqrt(2.0 / shp[0]))).astype(np.float32)
    imgs = synth.synthetic_images(2, seed=77)
    for prec in ("fp32", "bf16x3"):
        eng = Engine(device=0, precision=prec, max_batch=2)
        try:
            eng.load_weights_raw(W)
            tm, rt = eng.cam_estimate(imgs, want_rt=True)
        finally:
            eng.close()
        ref_rt, ref_tm = orc.cam_estimate(imgs, W)
        assert tm.shape == (2, 4, 3) and rt.shape == (2, 4, 3)
        assert np.abs(rt - ref_rt).max() <= 2e-4 * max(1.0, np.abs(ref_rt).max()), prec
        assert np.abs(tm - ref_tm).max() <= 2e-4 * np.abs(ref_tm).max(), prec
        # rotation block is a scaled orthonormal frame
        Rm = rt[:, :3, :]
        s2 = (Rm[:, :, 0] ** 2).sum(1)
        np.testing.assert_allclose(np.einsum("bij,bik->bjk", Rm, Rm), s2[:, None, None] * np.eye(3)[None], atol=1e-3 * s2.max())
