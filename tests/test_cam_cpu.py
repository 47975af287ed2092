"""oracle.disn_oracle's restatement of the camera-pose heads and geometry (cam_head_outputs / cam_pose / cam_heads)
without a GPU: its two modes agree on ordinary inputs, its float32-op mode gives the hand-derived results at the
degenerate poses, it equals orc.cam_estimate on the same embedding, and every fault in CAM_FAULTS moves the result by at
least three times the bounds tests/test_gpu_cam.py holds the kernel to."""
import numpy as np
import pytest

from oracle import disn_oracle as orc
from tests.test_gpu_cam import BOUND_PATH, K_SKEW, POSES, make_cam_weights

f32 = np.float32


@pytest.fixture(scope="module")
def cam_w(he_weights):
    return make_cam_weights(he_weights)


@pytest.fixture(scope="module")
def emb():
    """Embeddings like the VGG's fc8 output on the suite's images (measured: std 0.56, max 2.3), one scale per image."""
    rng = np.random.default_rng(11)
    return (rng.standard_normal((6, 1024)) * 0.56 * np.linspace(0.5, 2.0, 6)[:, None]).astype(np.float32)


def pose(name, K=orc.CAM_K, mode="float32-ops", fault=None):
    s, x, y, t = POSES[name]
    return orc.cam_pose(f32([s]), f32([list(x) + list(y)]), f32([t]), K=K, mode=mode, fault=fault)


# ---- restatement sanity ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", ["default", "skew"])
def test_modes_agree_on_ordinary_inputs(cam_w, emb, K):
    Km = orc.CAM_K if K == "default" else K_SKEW
    rt64, tm64 = orc.cam_heads(emb, cam_w, K=Km)
    rt32, tm32 = orc.cam_heads(emb, cam_w, K=Km, mode="float32-ops")
    assert rt64.dtype == np.float64 and rt32.dtype == np.float32
    assert np.abs(rt32 - rt64).max() <= 1e-6 * np.abs(rt64).max()
    assert np.abs(tm32 - tm64).max() <= 1e-6 * np.abs(tm64).max()
    # a scaled orthonormal frame
    R = rt64[:, :3]
    s2 = (R[:, :, 0] ** 2).sum(1)
    np.testing.assert_allclose(np.einsum("bij,bik->bjk", R, R), s2[:, None, None] * np.eye(3)[None], atol=1e-12)


def test_float32_ops_at_degenerate_poses_are_the_hand_derived_values():
    off = f32([-0.00193892, 0.00169222, 1.3949631])
    # x_raw = 0: |x| = 0 is clamped to 1e-8, x = 0 / 1e-8 = 0, so z = 0 x y = 0 and y = 0: R = 0; t + offset in float32
    rt, tm = pose("x_raw_zero")
    assert (rt[0, :3] == 0).all() and (tm[0, :3] == 0).all()
    np.testing.assert_array_equal(rt[0, 3], f32([0.1, -0.2, 0.3]) + off)
    assert rt[0, 3, 2] == f32(f32(0.3) + f32(1.3949631)) != f32(0.3 + 1.3949631)
    # the offsets alone, in float32
    rt, _ = pose("x_squared_near_overflow")
    np.testing.assert_array_equal(rt[0, 3], off)
    # |x_raw| = 1e-9 < 1e-8: x = x_raw / 1e-8 has length 0.1, not 1
    rt, _ = pose("x_raw_inside_clamp")
    x = f32([6e-10, 8e-10, 0.0]) / f32(1e-8)
    np.testing.assert_array_equal(rt[0, :3, 0], f32(1.25) * x)
    assert abs(np.linalg.norm(x.astype(np.float64)) - 0.1) < 1e-7
    # y_raw = 3 x_raw with x_raw = (1/2, -1, 1): x = (1/3, -2/3, 2/3) and fl(2/3) = 2 fl(1/3), so every product pair of
    # x cross y_raw rounds to the same value: z = 0 exactly, hence y = 0; only the x column survives
    rt, tm = pose("y_raw_3x_raw")
    third = f32(1) / f32(3)
    np.testing.assert_array_equal(rt[0, :3, 0], f32(0.8) * f32([third, -2 * third, 2 * third]))
    assert (rt[0, :3, 1:] == 0).all()
    # y_raw = 0: z = 0, y = 0
    rt, _ = pose("y_raw_zero")
    assert (rt[0, :3, 1:] == 0).all() and (rt[0, :3, 0] != 0).all()
    # a negative scale negates the rotation block exactly; the translation row keeps its sign
    rt_n, _ = pose("negative_scale")
    s, x, y, t = POSES["negative_scale"]
    rt_p, _ = orc.cam_pose(f32([-s]), f32([list(x) + list(y)]), f32([t]), mode="float32-ops")
    np.testing.assert_array_equal(rt_n[0, :3], -rt_p[0, :3])
    np.testing.assert_array_equal(rt_n[0, 3], rt_p[0, 3])
    # |x_raw|^2 overflows float32: |x| = inf, x = 0, R = 0 (float64 keeps the rotation)
    rt, _ = pose("x_squared_sum_overflows")
    assert (rt[0, :3] == 0).all()
    assert (pose("x_squared_sum_overflows", mode="float64")[0][0, :3, 0] != 0).all()
    # 2.69e38 is still finite: an ordinary frame
    rt, _ = pose("x_squared_near_overflow")
    np.testing.assert_allclose(rt[0, :3, 0], [1.3 / np.hypot(1.3, 1.0), 1.0 / np.hypot(1.3, 1.0), 0], rtol=1e-6)
    # |x cross y_raw|^2 overflows: z = 0, y = 0, x stays
    rt, _ = pose("y_raw_near_overflow")
    assert (rt[0, :3, 1:] == 0).all()
    np.testing.assert_allclose(rt[0, :3, 0], [0.6, 0.0, 0.8], rtol=1e-6)


def test_restatement_equals_cam_estimate(cam_w, emb, monkeypatch):
    """orc.cam_estimate (its own heads and rotation_from_ortho6d) on an embedding handed over in place of the VGG's."""
    monkeypatch.setattr(orc, "vgg_16", lambda img, W, dtype: (emb.astype(dtype).reshape(-1, 1, 1, 1024), None))
    for K in (orc.CAM_K, K_SKEW):
        rt, tm = orc.cam_estimate(np.zeros((emb.shape[0], 224, 224, 3), np.float32), cam_w, K=K)
        rt2, tm2 = orc.cam_heads(emb, cam_w, K=K)
        np.testing.assert_allclose(rt2, rt, rtol=0, atol=1e-14)
        np.testing.assert_allclose(tm2, tm, rtol=0, atol=1e-12)


# ---- every fault is visible ------------------------------------------------------------------------------------------------
def _shift(a, b):
    """Relative move of b from a (inf where a fault makes values non-finite)."""
    d = np.abs(np.asarray(b, np.float64) - a)
    return np.inf if not np.isfinite(d).all() else d.max() / np.abs(a).max()


@pytest.mark.parametrize("fault", orc.CAM_FAULTS)
def test_every_fault_moves_the_result_three_bounds(cam_w, emb, fault):
    """Each fault, on the ordinary embeddings and at the pose inside the clamp (where the clamp acts), moves pred_RT or
    pred_trans_mat by at least 3x the largest whole-path bound of any precision."""
    b_rt = max(b[0] for b in BOUND_PATH.values())
    b_tm = max(b[1] for b in BOUND_PATH.values())
    worst = 0.0
    for K in (orc.CAM_K, K_SKEW):
        ref = orc.cam_heads(emb, cam_w, K=K)
        bad = orc.cam_heads(emb, cam_w, K=K, fault=fault)
        worst = max(worst, _shift(ref[0], bad[0]) / b_rt, _shift(ref[1], bad[1]) / b_tm)
        ref = pose("x_raw_inside_clamp", K=K, mode="float64")
        bad = pose("x_raw_inside_clamp", K=K, mode="float64", fault=fault)
        worst = max(worst, _shift(ref[0], bad[0]) / b_rt, _shift(ref[1], bad[1]) / b_tm)
    print("%-24s moves the result by %.3g bounds" % (fault, worst))
    assert worst >= 3, fault
