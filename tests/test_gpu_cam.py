"""The estimated-camera path (disn_cam_estimate, csrc/cam.cu; demo/demo.py:195-258, cam_est/model_cam.py:47-109,
models/posenet.py:13-36,91-124) against oracle.disn_oracle's float64 and float32-op restatements, on synthetic camera
weights (the He-scaled vgg_16/* of the suite plus random pose heads).

- Heads on the device's embedding (disn_debug_cam_heads): every entry of pred_RT and pred_trans_mat within its own
  error-analysis bound of the float64 restatement on the same float32 embedding -- C_HEADS * 2^-24 * M per raw head
  output (M: the sum of the magnitudes of every term the three layers add), carried through the pose by the float64
  Jacobian of the pose, plus the pose's own float32 rounding (C_GEOM ulps of |scale|) and the 3 roundings of RT . K^T.
- Whole path in each precision at B = 1, 3, 8 on 137x137 (resized) and 224x224 (not resized) inputs:
  max |got - ref| / max |ref| of pred_RT and of pred_trans_mat against orc.cam_estimate in float64 within BOUND_PATH.
- Degenerate poses (fc3 weights zeroed, the head outputs set by the biases): pred_RT bit for bit the float32-op
  restatement, pred_trans_mat within 1.5 ulp of the exact product of that RT with K^T (see test_degenerate_poses).
- State and errors, and the demo's --cam_est flow.

Measured on an H100 80GB HBM3 (700 W); each bound is about twice the worst value measured.
    heads, B = 1, 3, 8, default and skewed K: max |err| 2.6e-6 on pred_RT, 4.1e-4 on pred_trans_mat (entries up to ~200);
        worst err / bound with C_HEADS = C_GEOM = 1: 0.009 (pred_RT), 0.007 (pred_trans_mat).  M adds magnitudes with
        no cancellation while the roundings of a 1024-term fmaf chain largely cancel, hence C_HEADS = 0.02.
    whole path, worst over B = 1, 3, 8 and both input sizes, max |got - ref| / max |ref|   (bound)
        fp32    pred_RT 5.3e-6, pred_trans_mat 4.4e-6                                  (1e-5, 1e-5)
        bf16x3  pred_RT 7.5e-5, pred_trans_mat 7.0e-5                                  (1.5e-4, 1.5e-4)
        f16f8   the bf16x3 values bit for bit: the encoder's GEMMs have no f16f8 mode  (1.5e-4, 1.5e-4)
    degenerate poses: pred_RT bit for bit, pred_trans_mat within the 1.5 ulp the kernel is held to.
"""
import os

import numpy as np
import pytest

from disn_b200 import synth
from oracle import disn_oracle as orc

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                  # float32 unit roundoff
MAX_B = 8                       # the encoder's batch limit (GEMV_MAXB)
# whole path, max |got - ref| / max |ref| per precision: (pred_RT, pred_trans_mat)
BOUND_PATH = {"fp32": (1e-5, 1e-5), "bf16x3": (1.5e-4, 1.5e-4), "f16f8": (1.5e-4, 1.5e-4)}
C_HEADS = 0.02                  # multiple of 2^-24 * M for each raw head output
C_GEOM = 4.0                    # float32 ulps (of |scale|) of the rotation block's own rounding
# a non-default intrinsics matrix, exact in float32, with skew and unequal focal lengths (K != K^T in every sense)
K_SKEW = np.array([[160.25, 1.5, 70.0], [0.0, 140.5, 66.25], [0.0, 0.0, 1.0]])


def make_cam_weights(he_weights, seed=3):
    """A camera checkpoint's variables: the suite's He-scaled vgg_16/* and random He-scaled pose heads."""
    rng = np.random.default_rng(seed)
    W = {k: v for k, v in he_weights.items() if k.startswith("vgg_16/")}
    for name, shp in orc.cam_head_shapes().items():
        W[name] = (rng.standard_normal(shp) * (0.02 if name.endswith("biases") else np.sqrt(2.0 / shp[0]))).astype(np.float32)
    return W


def rel_err(got, ref):
    e = np.abs(np.asarray(got, np.float64) - ref)
    s = np.abs(ref).max()
    return e.max() / s, np.sqrt((e ** 2).mean()) / s


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---- fixtures -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cam_w(he_weights):
    return make_cam_weights(he_weights)


@pytest.fixture(scope="module")
def cam_engines(cam_w):
    """One camera context per precision, max_batch 8."""
    from disn_b200.engine import Engine
    engs = {}
    for prec in ("fp32", "bf16x3", "f16f8"):
        engs[prec] = Engine(device=0, precision=prec, max_batch=MAX_B)
        engs[prec].load_weights_raw(cam_w)
    yield engs
    for e in engs.values():
        e.close()


@pytest.fixture(scope="module")
def images():
    """8 images per input size: 137x137 renders (resized to 224 by the encoder) and 224x224 ones (not resized)."""
    return {137: synth.synthetic_images(MAX_B, seed=77),
            224: np.random.default_rng(224).random((MAX_B, 224, 224, 3), dtype=np.float32)}


@pytest.fixture(scope="module")
def path_ref(images, cam_w):
    """orc.cam_estimate in float64 on each size's 8 images (images are independent: B < 8 uses the first B)."""
    return {hw: orc.cam_estimate(imgs, cam_w, dtype=np.float64) for hw, imgs in images.items()}


@pytest.fixture(scope="module")
def shared(he_weights, cam_w):
    """fp32 context holding the SDF network and the camera heads on one shared vgg_16/*."""
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="fp32", max_batch=MAX_B)
    eng.load_weights(dict(he_weights, **{k: v for k, v in cam_w.items() if k.startswith("cameraprediction/")}))
    yield eng
    eng.close()


# ---- heads on the device's embedding ------------------------------------------------------------------------------------
def debug_cam_heads(eng, emb, K=None):
    import ctypes as C
    from disn_b200 import _lib
    lib = _lib.load_test()
    e = np.ascontiguousarray(emb, np.float32)
    B = e.shape[0]
    rt, tm = np.empty((B, 4, 3), np.float32), np.empty((B, 4, 3), np.float32)
    kk = None if K is None else np.ascontiguousarray(K, np.float32).reshape(9)
    _lib.check(lib.disn_debug_cam_heads(eng._h, e.ctypes.data_as(C.c_void_p), B,
                                        None if kk is None else kk.ctypes.data_as(C.c_void_p),
                                        rt.ctypes.data_as(C.c_void_p), tm.ctypes.data_as(C.c_void_p)))
    return rt, tm


def heads_bound(emb, W, K=orc.CAM_K, c_heads=C_HEADS, c_geom=C_GEOM):
    """Per-entry bound on |float32 heads + pose - float64| for embeddings emb [B, n] (see the module docstring)."""
    emb = np.asarray(emb, np.float64)
    K = np.asarray(K, np.float64)
    B = emb.shape[0]

    def magnitude(name):
        m = np.abs(emb)
        for i in (1, 2, 3):
            m = m @ np.abs(np.asarray(W["cameraprediction/%s/fc%d/weights" % (name, i)], np.float64)) + \
                np.abs(np.asarray(W["cameraprediction/%s/fc%d/biases" % (name, i)], np.float64))
        return m

    d = c_heads * U * np.concatenate([magnitude(n) for n in ("scale", "ortho6d", "translation")], axis=1)   # [B,10]
    s, r6, t = orc.cam_head_outputs(emb, W)
    p = np.concatenate([s[:, None], r6, t], axis=1)

    def pose(q):
        rt, tm = orc.cam_pose(q[:, 0], q[:, 1:7], q[:, 7:10], K)
        return np.concatenate([rt, tm], axis=1)

    J = np.empty((B, 8, 3, 10))
    for k in range(10):
        h = 1e-6 * np.maximum(1.0, np.abs(p[:, k]))
        e = np.zeros_like(p)
        e[:, k] = h
        J[..., k] = (pose(p + e) - pose(p - e)) / (2 * h)[:, None, None]
    prop = np.einsum("bijk,bk->bij", np.abs(J), d)
    rt = pose(p)[:, :4]
    own = np.empty((B, 4, 3))
    own[:, :3] = c_geom * U * np.abs(s)[:, None, None]
    own[:, 3] = U * (np.abs(rt[:, 3]) + np.abs(orc.CAM_T_OFFSET))      # the add, and the offset's float32 rounding
    b_rt = prop[:, :4] + own
    b_tm = prop[:, 4:] + own @ np.abs(K).T + 3 * U * (np.abs(rt) @ np.abs(K).T)
    return b_rt, b_tm


def _report(tag, got, ref, bound):
    e = np.abs(np.asarray(got, np.float64) - ref)
    print("%-28s max %.3e  rms %.3e  max err/bound %.3f" % (tag, e.max(), np.sqrt((e ** 2).mean()), (e / bound).max()),
          flush=True)
    return (e / bound).max()


@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("K", ["default", "skew"])
def test_heads_on_device_embedding(shared, cam_w, images, B, K):
    """The heads on the VGG embedding the device computes, each image scaled differently (the per-image indexing),
    against the float64 restatement on that exact float32 embedding; each image also alone, bit for bit."""
    Km = None if K == "default" else K_SKEW
    shared.encode(images[137][:B])
    scales = np.linspace(0.6, 1.7, B, dtype=np.float32)
    emb = shared.get_encoded(0) * scales[:, None]
    rt, tm = debug_cam_heads(shared, emb, Km)
    Kr = orc.CAM_K if Km is None else Km
    ref_rt, ref_tm = orc.cam_heads(emb, cam_w, K=Kr)
    b_rt, b_tm = heads_bound(emb, cam_w, Kr, c_heads=1.0, c_geom=1.0)
    r_rt = _report("heads RT  B=%d K=%s" % (B, K), rt, ref_rt, b_rt)
    r_tm = _report("heads TM  B=%d K=%s" % (B, K), tm, ref_tm, b_tm)
    b_rt, b_tm = heads_bound(emb, cam_w, Kr)
    assert (np.abs(rt - ref_rt) <= b_rt).all(), r_rt
    assert (np.abs(tm - ref_tm) <= b_tm).all(), r_tm
    for b in range(B):
        rt1, tm1 = debug_cam_heads(shared, emb[b:b + 1], Km)
        np.testing.assert_array_equal(bits(rt1[0]), bits(rt[b]))
        np.testing.assert_array_equal(bits(tm1[0]), bits(tm[b]))


# ---- whole path -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw", [137, 224])
@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "f16f8"])
def test_whole_path(cam_engines, images, path_ref, prec, hw):
    """Image -> VGG embedding -> heads -> pose at B = 1, 3, 8; three calls (eager, graph capture, graph replay) bit for
    bit equal, the last one without out_rt."""
    eng = cam_engines[prec]
    ref_rt, ref_tm = path_ref[hw]
    worst = [0.0, 0.0]
    for B in (1, 3, MAX_B):
        tm, rt = eng.cam_estimate(images[hw][:B], want_rt=True)
        tm2, rt2 = eng.cam_estimate(images[hw][:B], want_rt=True)
        tm3 = eng.cam_estimate(images[hw][:B])
        np.testing.assert_array_equal(bits(rt2), bits(rt))
        np.testing.assert_array_equal(bits(tm2), bits(tm))
        np.testing.assert_array_equal(bits(tm3), bits(tm))
        e_rt, s_rt = rel_err(rt, ref_rt[:B])
        e_tm, s_tm = rel_err(tm, ref_tm[:B])
        print("path %-6s %dx%d B=%d  RT max %.3e rms %.3e   TM max %.3e rms %.3e"
              % (prec, hw, hw, B, e_rt, s_rt, e_tm, s_tm), flush=True)
        worst = [max(worst[0], e_rt), max(worst[1], e_tm)]
    assert worst[0] <= BOUND_PATH[prec][0] and worst[1] <= BOUND_PATH[prec][1], (prec, worst)


@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "f16f8"])
def test_batch_images_are_independent(cam_engines, images, prec):
    """Image 1 of a batch of 3 gives the same bits whatever images 0 and 2 are."""
    eng = cam_engines[prec]
    a = images[137][:3]
    b = a.copy()
    b[0], b[2] = images[137][3], images[137][4]
    tm_a, rt_a = eng.cam_estimate(a, want_rt=True)
    tm_b, rt_b = eng.cam_estimate(b, want_rt=True)
    np.testing.assert_array_equal(bits(rt_b[1]), bits(rt_a[1]))
    np.testing.assert_array_equal(bits(tm_b[1]), bits(tm_a[1]))
    assert not np.array_equal(rt_b[0], rt_a[0]) and not np.array_equal(rt_b[2], rt_a[2])


def test_non_default_intrinsics_are_transposed(cam_engines, images, path_ref):
    """pred_trans_mat = pred_RT . K^T for a K with skew and unequal focal lengths: RT is unchanged by K, trans_mat is
    within 3 float32 roundings of RT . K^T and far from RT . K, and the whole path stays in its bound."""
    eng = cam_engines["fp32"]
    tm0, rt0 = eng.cam_estimate(images[137][:3], want_rt=True)
    tm, rt = eng.cam_estimate(images[137][:3], K=K_SKEW, want_rt=True)
    np.testing.assert_array_equal(bits(rt), bits(rt0))
    r = rt.astype(np.float64)
    exact = r @ K_SKEW.T
    assert (np.abs(tm - exact) <= 3 * U * (np.abs(r) @ np.abs(K_SKEW).T)).all()
    assert np.abs(tm - r @ K_SKEW).max() > 1.0
    ref_rt = path_ref[137][0][:3]
    e_tm, _ = rel_err(tm, ref_rt @ K_SKEW.T)
    assert e_tm <= BOUND_PATH["fp32"][1], e_tm


# ---- degenerate poses -----------------------------------------------------------------------------------------------------
POSES = {   # name: (scale, x_raw, y_raw, translation before the offset)
    "x_raw_zero": (1.25, (0.0, 0.0, 0.0), (0.3, -0.2, 0.9), (0.1, -0.2, 0.3)),
    "x_raw_inside_clamp": (1.25, (6e-10, 8e-10, 0.0), (0.2, 0.5, -0.4), (0.0, 0.0, 0.0)),
    "y_raw_3x_raw": (0.8, (0.5, -1.0, 1.0), (1.5, -3.0, 3.0), (-0.05, 0.02, 0.4)),
    "y_raw_zero": (1.1, (0.3, 0.4, 1.2), (0.0, 0.0, 0.0), (0.2, 0.1, -0.1)),
    "negative_scale": (-0.75, (0.6, -0.3, 0.2), (0.1, 0.9, -0.4), (0.01, 0.02, 0.03)),
    "x_squared_near_overflow": (1.0, (1.3e19, 1.0e19, 0.0), (1.0, 2.0, -0.5), (0.0, 0.0, 0.0)),
    "x_squared_sum_overflows": (1.0, (1.5e19, 1.5e19, 1.5e19), (1.0, 2.0, -0.5), (0.0, 0.0, 0.0)),
    "y_raw_near_overflow": (1.0, (0.6, 0.0, 0.8), (0.0, 2.0e19, 0.0), (0.0, 0.0, 0.0)),
}


def pose_weights(s, x, y, t):
    """fc3 weights zeroed, biases set: every image's head outputs are exactly (s, x, y, t) in float32."""
    f = lambda v: np.asarray(v, np.float32)
    return {"cameraprediction/scale/fc3/weights": np.zeros((32, 1), np.float32),
            "cameraprediction/scale/fc3/biases": f([s]),
            "cameraprediction/ortho6d/fc3/weights": np.zeros((256, 6), np.float32),
            "cameraprediction/ortho6d/fc3/biases": f(list(x) + list(y)),
            "cameraprediction/translation/fc3/weights": np.zeros((64, 3), np.float32),
            "cameraprediction/translation/fc3/biases": f(t)}


def ulp(v):
    return np.spacing(np.abs(np.asarray(v, np.float32))).astype(np.float64)


@pytest.fixture(scope="module")
def pose_engine(cam_w):
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="fp32", max_batch=2)
    eng.load_weights_raw(cam_w)
    yield eng
    eng.close()


@pytest.mark.parametrize("name", list(POSES))
@pytest.mark.parametrize("K", ["default", "skew"])
def test_degenerate_poses(pose_engine, images, name, K):
    """pred_RT bit for bit the float32-op restatement (the kernel rounds op by op in TF's order; its three-term sums run
    left to right as the restatement's do).  pred_trans_mat: TF's float32 matmul pins no order, so no bit pattern is
    the reference's.  Any order rounds 3 products and 2 sums, each by at most half an ulp of S = sum_k |RT_ik K_jk|
    (every partial sum is at most S): within 2.5 ulp(S) of the exact RT . K^T.  The kernel's fmaf chain rounds three
    times: within 1.5 ulp(S), which is what it is held to; the restatement is held to its 2.5."""
    s, x, y, t = POSES[name]
    Km = orc.CAM_K if K == "default" else K_SKEW
    pose_engine.load_weights_raw(pose_weights(s, x, y, t))
    tm, rt = pose_engine.cam_estimate(images[137][:2], K=None if K == "default" else K_SKEW, want_rt=True)
    f = np.float32
    ref_rt, ref_tm = orc.cam_pose(f([s]), f([list(x) + list(y)]), f([t]), K=Km, mode="float32-ops")
    print("pose %-24s K=%-7s RT %s" % (name, K, np.array2string(rt[0].reshape(-1), precision=6)), flush=True)
    for b in range(2):
        np.testing.assert_array_equal(rt[b], ref_rt[0], err_msg=name)
        assert np.isfinite(rt[b]).all()
        r = rt[b].astype(np.float64)
        exact = r @ Km.T
        S = np.abs(r) @ np.abs(Km).T
        assert (np.abs(tm[b] - exact) <= 1.5 * ulp(S)).all(), (name, tm[b] - exact)
        assert (np.abs(ref_tm[0] - exact) <= 2.5 * ulp(S)).all(), name


# ---- state and errors ------------------------------------------------------------------------------------------------------
def test_refused_calls_leave_the_context_usable(cam_w, cam_engines, images, path_ref):
    """B = max_batch + 1, a missing and a mis-shaped cameraprediction/* variable are refused, the variable by name; the
    context then estimates the bits it estimates without the refusals."""
    from disn_b200._lib import DisnError
    from disn_b200.engine import Engine
    imgs = images[137]
    eng = cam_engines["fp32"]
    with pytest.raises(DisnError, match="max_batch"):
        eng.cam_estimate(np.concatenate([imgs, imgs[:1]]))
    tm, rt = eng.cam_estimate(imgs[:2], want_rt=True)
    assert rel_err(rt, path_ref[137][0][:2])[0] <= BOUND_PATH["fp32"][0]
    assert rel_err(tm, path_ref[137][1][:2])[0] <= BOUND_PATH["fp32"][1]
    missing = "cameraprediction/translation/fc3/biases"
    fresh = Engine(device=0, precision="fp32", max_batch=1)
    try:
        fresh.load_weights_raw({k: v for k, v in cam_w.items() if k != missing})
        with pytest.raises(DisnError, match="missing variable " + missing):
            fresh.cam_estimate(imgs[:1])
        fresh.load_weights_raw({missing: cam_w[missing]})
        tm0, rt0 = fresh.cam_estimate(imgs[:1], want_rt=True)
        assert rel_err(tm0, path_ref[137][1][:1])[0] <= BOUND_PATH["fp32"][1]
        with pytest.raises(DisnError, match="max_batch"):
            fresh.cam_estimate(imgs[:2])
        tm1, rt1 = fresh.cam_estimate(imgs[:1], want_rt=True)
        fresh.load_weights_raw({missing: np.zeros(2, np.float32)})
        with pytest.raises(DisnError, match="mis-shaped variable " + missing):
            fresh.cam_estimate(imgs[:1])
        fresh.load_weights_raw({missing: cam_w[missing]})
        tm2, rt2 = fresh.cam_estimate(imgs[:1], want_rt=True)
    finally:
        fresh.close()
    for got_tm, got_rt in ((tm1, rt1), (tm2, rt2)):
        np.testing.assert_array_equal(bits(got_rt), bits(rt0))
        np.testing.assert_array_equal(bits(got_tm), bits(tm0))


def test_camera_then_sdf_on_one_context(he_weights, cam_w, images, path_ref):
    """A context holding both networks: cam_estimate drops the encoded batch (eval_points refuses until a new encode),
    and cam_estimate then encode + eval_points gives the bits of a context that never ran the camera path."""
    from disn_b200._lib import DisnError
    from disn_b200.engine import Engine
    imgs = images[137][:2]
    pts = np.random.default_rng(9).uniform(-1, 1, (2, 2000, 3)).astype(np.float32)
    tm = synth.synthetic_trans_mats(2, seed=5)
    plain = Engine(device=0, precision="f16f8", max_batch=2)
    both = Engine(device=0, precision="f16f8", max_batch=2)
    try:
        plain.load_weights(he_weights)
        plain.encode(imgs)
        want = plain.eval_points(pts, tm)
        both.load_weights(dict(he_weights, **{k: v for k, v in cam_w.items() if k.startswith("cameraprediction/")}))
        both.encode(imgs)
        np.testing.assert_array_equal(bits(both.eval_points(pts, tm)), bits(want))
        for _ in range(3):          # eager, captured and replayed encoder graphs of both kinds
            cam = both.cam_estimate(imgs)
            with pytest.raises(DisnError, match="disn_encode has not been called"):
                both.eval_points(pts, tm)
            both.encode(imgs)
            np.testing.assert_array_equal(bits(both.eval_points(pts, tm)), bits(want))
        assert rel_err(cam, path_ref[137][1][:2])[0] <= BOUND_PATH["f16f8"][1]
    finally:
        plain.close()
        both.close()


# ---- the demo's --cam_est flow -------------------------------------------------------------------------------------------
def test_demo_cam_est_flow(he_weights, cam_w, golden, tmp_path, monkeypatch):
    """demo.read_img_get_transmat(cam_est=True) on the shipped demo image gives Engine(bf16x3).cam_estimate's bits, and
    demo.create meshes the grid eval_grid computes at that trans_mat."""
    import cv2
    from disn_b200 import create_sdf as drv
    from disn_b200 import demo
    from disn_b200.engine import Engine
    img_u8 = golden["demo_input"]["img_u8"]
    path = str(tmp_path / "demo.png")
    assert cv2.imwrite(path, img_u8)
    monkeypatch.setattr(demo, "CAM_WEIGHTS", cam_w)
    flags = demo.default_flags(log_dir=str(tmp_path / "out"), sdf_res=32, cam_est=True, keep_dist=True)
    drv.configure(flags)
    batch = demo.read_img_get_transmat(path, cam_est=True)
    img = (img_u8.astype(np.float32) / np.float32(255.))[None]
    np.testing.assert_array_equal(batch["img"], img)
    eng = Engine(device=0, precision="bf16x3", max_batch=1)
    try:
        eng.load_weights_raw(cam_w)
        want_tm = eng.cam_estimate(img)
    finally:
        eng.close()
    np.testing.assert_array_equal(bits(batch["trans_mat"]), bits(want_tm))
    (obj,) = demo.create(he_weights, img_file=path, flags=flags)
    assert os.path.basename(obj) == "demo_obj_00.obj" and "camest_" in obj and os.path.getsize(obj) > 0
    res, bbox, grid = drv.read_dist(obj[:-4] + ".dist")
    assert res == 32
    eng = Engine(device=0, precision=flags.precision, max_batch=1)
    try:
        eng.load_weights(he_weights)
        eng.encode(img)
        want = eng.eval_grid(batch["sdf_params"], want_tm, 32)
    finally:
        eng.close()
    np.testing.assert_array_equal(bits(np.asarray(grid).reshape(-1)), bits(want.reshape(-1)))
