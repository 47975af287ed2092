"""GPU parity tests on the configurations and the operand mode the bench actually runs (BASELINE.json configs 0/1/2,
precision f16f8): the real grid outputs are compared with the float64 oracle at randomly sampled grid indices, the
reference-literal conditions (xavier/zero init, 224x224 input, tanh) run in every precision mode, the activation range
of the f16f8 mode is swept, and the shipped demo image goes through the GPU path.

Oracle cost: the float64 VGG restatement takes ~10 s per image on 8 host cores, so the 8 synthetic images are
encoded once per session (fixture oracle_enc8) and sliced."""
import os
from types import SimpleNamespace

import numpy as np
import pytest

from disn_b200 import synth
from oracle import disn_oracle as orc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-4                      # north_star: |sdf - reference| <= 1e-4 absolute, sdf = pred / 10


@pytest.fixture(scope="session")
def oracle_enc8(he_weights):
    """float64 oracle encoder outputs of synthetic_images(8, seed=1234) (image b uses seed 1234 + b)."""
    imgs = synth.synthetic_images(8, seed=1234)
    return imgs, orc.encode(imgs, he_weights, dtype=np.float64)


def _slice_enc(enc, b0, b1):
    return SimpleNamespace(resized_ref_img=enc.resized_ref_img[b0:b1], img_embedding=enc.img_embedding[b0:b1],
                           maps=[m[b0:b1] for m in enc.maps], vgg_end_points=None)


def _grid_points_at(sdf_params, R, flat_idx):
    """The reference's float32 grid points (create_sdf.py:246-255) at flat (z,y,x) indices, x fastest."""
    x_ = np.linspace(sdf_params[0], sdf_params[3], num=R)
    y_ = np.linspace(sdf_params[1], sdf_params[4], num=R)
    z_ = np.linspace(sdf_params[2], sdf_params[5], num=R)
    ix, iy, iz = flat_idx % R, (flat_idx // R) % R, flat_idx // (R * R)
    return np.stack([x_[ix], y_[iy], z_[iz]], axis=1).astype(np.float32)


def _sampled_grid_error(grid, enc, tm, sdf_params, W, n_per_image, seed):
    """max |grid/1 - oracle64| over n_per_image random grid indices of every image (grid is already pred / 10)."""
    B, R = grid.shape[0], grid.shape[1]
    worst = 0.0
    for b in range(B):
        idx = np.random.default_rng(seed + b).choice(R ** 3, size=min(n_per_image, R ** 3), replace=False)
        pts = _grid_points_at(sdf_params[b], R, idx)[None]
        ref = orc.decode(_slice_enc(enc, b, b + 1), pts, pts, tm[b:b + 1], W, dtype=np.float64)["pred_sdf"]
        got = grid[b].reshape(-1)[idx]
        worst = max(worst, float(np.abs(got - ref.reshape(-1) / orc.SDF_WEIGHT).max()))
    return worst


@pytest.fixture(scope="module")
def eng8(he_weights):
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="f16f8", max_batch=8)
    eng.load_weights(he_weights)
    yield eng
    eng.close()


@pytest.mark.parametrize("precision", ["f16f8", "bf16x3"])
def test_config1_res256_grid_vs_oracle_at_sampled_indices(eng8, he_weights, oracle_enc8, precision):
    """BASELINE config 1 (single image, --sdf_res 256 -> 257^3 = 16 974 593 points): 20 000 random samples of the REAL
    output against the float64 oracle, plus bitwise z-slab invariance (what the multi-GPU sharding relies on)."""
    imgs, enc = oracle_enc8
    eng8.set_precision(precision)
    eng8.encode(imgs[:1])
    tm, sp = synth.DEMO_TRANS_MAT, synth.DEMO_SDF_PARAMS
    grid = eng8.eval_grid(sp, tm, 256)
    assert grid.shape == (1, 257, 257, 257) and np.isfinite(grid).all()
    err = _sampled_grid_error(grid, enc, tm, sp, he_weights, 20000, seed=900)
    assert err <= TOL, err
    slabs = [eng8.eval_grid(sp, tm, 256, z0=a, z1=b) for a, b in ((0, 33), (33, 130), (130, 257))]
    np.testing.assert_array_equal(np.concatenate(slabs, axis=1), grid)


def test_config1_every_point_of_the_grid_vs_the_fp32_path(eng8):
    """The sampled tests above see 20 000 of the 16 974 593 points.  This one compares EVERY point of the 257^3 grid of the
    shipped operand mode with the CUDA-core fp32 path of the same library on the same encoder products (the fp32 path is
    held to the float64 oracle at <= 1e-5 by test_gpu_parity.py (FP32_TOL)), so the maximum over the whole grid is bounded too:
    |f16f8 - oracle| <= |f16f8 - fp32| + |fp32 - oracle| <= 9e-5 + 1e-5."""
    imgs = synth.synthetic_images(1, seed=1234)
    tm, sp = synth.DEMO_TRANS_MAT, synth.DEMO_SDF_PARAMS
    eng8.set_precision("f16f8")
    eng8.encode(imgs)
    g_tc = eng8.eval_grid(sp, tm, 256)
    eng8.set_precision("fp32")
    g_32 = eng8.eval_grid(sp, tm, 256)
    eng8.set_precision("f16f8")
    assert g_tc.shape == g_32.shape == (1, 257, 257, 257)
    d = np.abs(g_tc.astype(np.float64) - g_32)
    print("full-grid max |f16f8 - fp32| = %.3e, rms %.3e, max |sdf| %.3f" % (d.max(), np.sqrt((d ** 2).mean()), np.abs(g_32).max()))
    assert d.max() <= 9e-5, float(d.max())


@pytest.mark.parametrize("init", ["he", "xavier"])
def test_config0_res64_grid_vs_oracle(eng8, he_weights, oracle_enc8, init):
    """BASELINE config 0 (demo.py, --sdf_res 64 -> 65^3 = 274 625 points, 2 chunks of 137 313): f16f8 output vs the
    float64 oracle at 20 000 sampled indices.  init='xavier' is the config's literal 'random-init weights' condition
    (xavier-uniform, zero biases: utils/tf_util.py:41,173-174); there |pred| is tiny, so the bound is relative too."""
    from disn_b200.engine import Engine
    imgs, enc = oracle_enc8
    tm, sp = synth.DEMO_TRANS_MAT, synth.DEMO_SDF_PARAMS
    if init == "he":
        eng, W = eng8, he_weights
        eng.set_precision("f16f8")
    else:
        W = synth.make_weights(seed=11, init="xavier")
        eng = Engine(device=0, precision="f16f8", max_batch=1)
        eng.load_weights(W)
        enc = orc.encode(imgs[:1], W, dtype=np.float64)
    try:
        eng.encode(imgs[:1])
        grid = eng.eval_grid(sp, tm, 64)
        assert grid.shape == (1, 65, 65, 65)
        err = _sampled_grid_error(grid, enc, tm, sp, W, 20000, seed=901)
        assert err <= TOL, err
        if init == "xavier":      # the absolute bar is vacuous when |sdf| ~ 1e-3: also hold 1e-3 of the field's scale
            assert err <= 1e-3 * float(np.abs(grid).max()) + 1e-8, (err, float(np.abs(grid).max()))
    finally:
        if init != "he":
            eng.close()


def test_config2_batch8_res128_grid_vs_oracle(eng8, he_weights, oracle_enc8):
    """BASELINE config 2 (batch of 8 renders, --sdf_res 128 -> 8 x 129^3 points, VGG on the tensor cores): every image of the
    batch against the float64 oracle at 2 500 sampled indices (20 000 in total), ShapeNet-style cameras and boxes."""
    imgs, enc = oracle_enc8
    eng8.set_precision("f16f8")
    eng8.encode(imgs)
    # encoder products of the batch (tensor-core conv path) vs the oracle
    emb = eng8.get_encoded(0)
    assert np.abs(emb - enc.img_embedding).max() <= 2e-4 * np.abs(enc.img_embedding).max()   # measured 6e-5 (bf16x3 convs, split-K)
    tm = synth.synthetic_trans_mats(8, seed=4321)
    sp = np.tile(synth.DEMO_SDF_PARAMS, (8, 1)) * np.linspace(0.8, 1.0, 8)[:, None]
    grid = eng8.eval_grid(sp, tm, 128)
    assert grid.shape == (8, 129, 129, 129) and np.isfinite(grid).all()
    err = _sampled_grid_error(grid, enc, tm, sp, he_weights, 2500, seed=902)
    assert err <= TOL, err


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "f16f8"])
def test_xavier_init_224_input_and_tanh_in_every_mode(precision):
    """Reference-literal random init (xavier/zero), a 224x224 input (skips the resize, model_normalization.py:65-72) and
    FLAGS.tanh (model_normalization.py:214-216) in every precision mode."""
    from disn_b200.engine import Engine
    W = synth.make_weights(seed=11, init="xavier")
    img224 = np.random.default_rng(1).random((1, 224, 224, 3), dtype=np.float32)
    pts = np.random.default_rng(2).uniform(-1, 1, size=(1, 700, 3)).astype(np.float32)
    enc = orc.encode(img224, W, dtype=np.float64)
    for tanh in (False, True):
        eng = Engine(device=0, precision=precision, tanh=tanh)
        try:
            eng.load_weights(W)
            eng.encode(img224)
            pred = eng.eval_points(pts, synth.DEMO_TRANS_MAT)
        finally:
            eng.close()
        ref = orc.decode(enc, pts, pts, synth.DEMO_TRANS_MAT, W, FLAGS=orc.default_flags(tanh=tanh),
                         dtype=np.float64)["pred_sdf"]
        scale = max(float(np.abs(ref).max()), 1e-12)
        assert np.abs(pred - ref).max() / orc.SDF_WEIGHT <= TOL
        assert np.abs(pred - ref).max() <= 1e-3 * scale + 1e-8, (precision, tanh)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "f16f8"])
def test_tanh_with_order_one_outputs(he_weights, oracle_enc8, precision):
    """tanh on O(1) predictions (He-scaled weights), where it actually bends the output."""
    from disn_b200.engine import Engine
    imgs, enc = oracle_enc8
    pts = np.random.default_rng(12).uniform(-1, 1, size=(1, 3000, 3)).astype(np.float32)
    eng = Engine(device=0, precision=precision, tanh=True)
    try:
        eng.load_weights(he_weights)
        eng.encode(imgs[:1])
        pred = eng.eval_points(pts, synth.DEMO_TRANS_MAT)
    finally:
        eng.close()
    ref = orc.decode(_slice_enc(enc, 0, 1), pts, pts, synth.DEMO_TRANS_MAT, he_weights,
                     FLAGS=orc.default_flags(tanh=True), dtype=np.float64)["pred_sdf"]
    assert np.abs(ref).max() > 0.3 and np.abs(ref).max() <= 1.0
    assert np.abs(pred - ref).max() / orc.SDF_WEIGHT <= TOL


def _scaled_heads(W, s):
    """Same function, internal activations of both point MLPs scaled by s: W1,b1 and every later bias (and the
    image-feature rows of fold2/conv1) times s, the linear output layer's weights times 1/s."""
    out = dict(W)
    for scope in ("sdfprediction", "sdfprediction_imgfeat"):
        g = lambda n: np.asarray(W["%s/%s" % (scope, n)], np.float64)
        out["%s/fold1/conv1/weights" % scope] = (g("fold1/conv1/weights") * s).astype(np.float32)
        for l in ("fold1/conv1", "fold1/conv2", "fold1/conv3", "fold2/conv1", "fold2/conv2"):
            out["%s/%s/biases" % (scope, l)] = (g(l + "/biases") * s).astype(np.float32)
        w = g("fold2/conv1/weights").copy()
        w[..., 512:, :] *= s                      # rows fed by the (unscaled) image features
        out["%s/fold2/conv1/weights" % scope] = w.astype(np.float32)
        out["%s/fold2/conv5/weights" % scope] = (g("fold2/conv5/weights") / s).astype(np.float32)
    return out


@pytest.mark.parametrize("scale", [1.0 / 64, 1.0, 64.0, 1024.0])
def test_f16f8_activation_range_sweep(he_weights, oracle_enc8, scale):
    """The f16f8 operands use static power-of-two scales chosen from the WEIGHTS (tc_pack_weights).  Sweep the
    activation magnitude over 2^16 with the function itself unchanged: the 1e-4 bar must hold across the range."""
    from disn_b200.engine import Engine
    imgs, enc = oracle_enc8
    W = _scaled_heads(he_weights, scale)
    pts = np.random.default_rng(31).uniform(-1, 1, size=(1, 4000, 3)).astype(np.float32)
    ref = orc.decode(_slice_enc(enc, 0, 1), pts, pts, synth.DEMO_TRANS_MAT, W, dtype=np.float64)["pred_sdf"]
    eng = Engine(device=0, precision="f16f8")
    try:
        eng.load_weights(W)
        eng.encode(imgs[:1])
        pred = eng.eval_points(pts, synth.DEMO_TRANS_MAT)
    finally:
        eng.close()
    assert np.isfinite(pred).all()
    assert np.abs(pred - ref).max() / orc.SDF_WEIGHT <= TOL, scale


def test_f16f8_overflow_is_loud_and_bf16x3_still_works(he_weights, oracle_enc8):
    """Activations beyond fp16's 65504 must raise, not return inf; DISN_PREC_BF16X3 has no such limit."""
    from disn_b200._lib import DisnError
    from disn_b200.engine import Engine
    imgs, enc = oracle_enc8
    W = _scaled_heads(he_weights, 2.0 ** 17)
    pts = np.random.default_rng(32).uniform(-1, 1, size=(1, 1000, 3)).astype(np.float32)
    eng = Engine(device=0, precision="f16f8")
    try:
        eng.load_weights(W)
        eng.encode(imgs[:1])
        with pytest.raises(DisnError, match="fp16 range"):
            eng.eval_points(pts, synth.DEMO_TRANS_MAT)
        with pytest.raises(DisnError, match="fp16 range"):
            eng.eval_grid(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 16)
        eng.set_precision("bf16x3")
        pred = eng.eval_points(pts, synth.DEMO_TRANS_MAT)
        ref = orc.decode(_slice_enc(enc, 0, 1), pts, pts, synth.DEMO_TRANS_MAT, W, dtype=np.float64)["pred_sdf"]
        assert np.abs(pred - ref).max() / orc.SDF_WEIGHT <= TOL
        eng.set_precision("f16f8")           # the error state does not stick to the context
        eng.load_weights(he_weights)
        eng.encode(imgs[:1])
        assert np.isfinite(eng.eval_points(pts, synth.DEMO_TRANS_MAT)).all()
    finally:
        eng.close()


def test_shipped_demo_image_through_the_gpu_path(he_weights, golden):
    """demo/demo.py:261-279: the shipped render (tests/golden/demo_input.npz = the PNG decoded by the reference's own
    loader steps, see make_golden_demo.py) + the demo trans_mat, --sdf_res 64 (BASELINE config 0), f16f8; parity vs the
    float64 oracle at 8 000 sampled grid indices, and the mesh pipeline runs on the real input's field."""
    from disn_b200.engine import Engine
    img = (golden["demo_input"]["img_u8"].astype(np.float32) / np.float32(255.))[None]     # demo.py:264
    assert img.shape == (1, 137, 137, 3) and 0.0 <= img.min() and img.max() <= 1.0
    eng = Engine(device=0, precision="f16f8")
    try:
        eng.load_weights(he_weights)
        eng.encode(img)
        grid = eng.eval_grid(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 64)
        verts, faces = eng.marching_cubes(grid[0], synth.DEMO_SDF_PARAMS[0], iso=float(np.median(grid)))
    finally:
        eng.close()
    enc = orc.encode(img, he_weights, dtype=np.float64)
    err = _sampled_grid_error(grid, enc, synth.DEMO_TRANS_MAT, synth.DEMO_SDF_PARAMS, he_weights, 8000, seed=903)
    assert err <= TOL, err
    assert len(verts) > 100 and len(faces) > 100 and faces.max() < len(verts)
