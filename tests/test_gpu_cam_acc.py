"""GPU tests of disn_cam_metrics (Engine.cam_metrics), the camera checkpoint score of cam_est/train_sdf_cam.py --test,
and of the --test / --create driver end to end.

The predicted matrices must be disn_cam_estimate's bits; each float64 sum must lie within 2^-40 * sum|term| of the
exactly rounded (math.fsum) sum of cam_metric_terms evaluated on the returned matrices; repeated calls are bitwise equal
and each image's results do not depend on the other images of its batch.
"""
import glob
import math
import os
import random

import numpy as np
import pytest

from disn_b200 import synth
from oracle import disn_oracle as orc
from oracle.cam_acc_oracle import cam_metric_terms
from tests.test_gpu_cam import make_cam_weights

pytestmark = pytest.mark.gpu

MAX_B = 8
KEYS = ("rotpc", "rot2d", "rot3d", "rot2d_dist", "rotmatrix")


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def cam_w(he_weights):
    return make_cam_weights(he_weights)


@pytest.fixture(scope="module")
def engines(cam_w):
    from disn_b200.engine import Engine
    engs = {}
    for prec in ("fp32", "bf16x3"):
        engs[prec] = Engine(device=0, precision=prec, max_batch=MAX_B)
        engs[prec].load_weights_raw(cam_w)
    yield engs
    for e in engs.values():
        e.close()


@pytest.fixture(scope="module")
def images():
    return {137: synth.synthetic_images(MAX_B, seed=78),
            224: np.random.default_rng(225).random((MAX_B, 224, 224, 3), dtype=np.float32)}


def ground_truth(B, N, seed):
    """Points and ground-truth poses in front of the camera: RT [B,4,3] near [I; (0, 0, 1.4)], trans_mat = RT . K^T."""
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-0.5, 0.5, (B, N, 3)).astype(np.float32)
    RT = np.tile(np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [0, 0, 1.4]], np.float64), (B, 1, 1))
    RT = (RT + 0.15 * rng.standard_normal((B, 4, 3))).astype(np.float32)
    tm = (RT.astype(np.float64) @ orc.CAM_K.T).astype(np.float32)
    pts.reshape(-1)[5::97] = np.float32(0.49)             # projections beyond the [0, 136] clamp on some axes
    return pts, tm, RT


def check_sums(sums, pts, tm, RT, pred_tm, pred_rt):
    terms = cam_metric_terms(pts, tm, RT, pred_tm, pred_rt)
    for b in range(len(sums)):
        for k, key in enumerate(KEYS):
            t = terms[key][b].astype(np.float64).ravel()
            exact = math.fsum(t)
            assert abs(sums[b, k] - exact) <= 2.0 ** -40 * math.fsum(np.abs(t)), (b, key, sums[b, k], exact)


@pytest.mark.parametrize("hw", [137, 224])
@pytest.mark.parametrize("prec", ["fp32", "bf16x3"])
@pytest.mark.parametrize("N", [1, 2048, 4099])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_cam_metrics(engines, images, prec, hw, B, N):
    eng = engines[prec]
    imgs = images[hw][:B]
    pts, tm, RT = ground_truth(B, N, 100 * B + N % 13 + hw)
    want_tm, want_rt = eng.cam_estimate(imgs, want_rt=True)
    pred_tm, pred_rt, sums = eng.cam_metrics(imgs, pts, tm, RT)
    np.testing.assert_array_equal(bits(pred_tm), bits(want_tm))
    np.testing.assert_array_equal(bits(pred_rt), bits(want_rt))
    assert sums.shape == (B, 5) and np.isfinite(sums).all()
    check_sums(sums, pts, tm, RT, pred_tm, pred_rt)
    again = eng.cam_metrics(imgs, pts, tm, RT)
    for a, b in zip(again, (pred_tm, pred_rt, sums)):
        assert a.tobytes() == b.tobytes()
    if B > 1:       # image 1's results do not depend on the other images (and points) of the batch
        imgs2, pts2, tm2, RT2 = imgs.copy(), pts.copy(), tm.copy(), RT.copy()
        others = [b for b in range(B) if b != 1]
        imgs2[others] = images[hw][::-1][:B][others]
        pts2[others] = ground_truth(B, N, 7)[0][others]
        tm2[others], RT2[others] = tm[::-1][others], RT[::-1][others]
        got = eng.cam_metrics(imgs2, pts2, tm2, RT2)
        for a, b in zip(got, (pred_tm, pred_rt, sums)):
            assert a[1].tobytes() == b[1].tobytes()
        assert not np.array_equal(got[2][0], sums[0])


def test_refusals_leave_the_context_usable(cam_w, engines, images):
    import ctypes as C
    from disn_b200._lib import DisnError
    from disn_b200.engine import Engine
    eng = engines["fp32"]
    imgs = images[137]
    pts, tm, RT = ground_truth(MAX_B + 1, 16, 3)
    before = eng.cam_estimate(imgs[:2], want_rt=True)
    with pytest.raises(DisnError, match="max_batch"):
        eng.cam_metrics(np.concatenate([imgs, imgs[:1]]), pts, tm, RT)
    with pytest.raises(DisnError, match="N >= 1"):
        eng.cam_metrics(imgs[:2], pts[:2, :0], tm[:2], RT[:2])
    sums = np.zeros((2, 5))
    a = np.ascontiguousarray(imgs[:2])
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    for args in ((p(a), p(pts), None), (None, p(pts), p(RT)), (p(a), None, p(RT))):
        rc = eng.lib.disn_cam_metrics(eng._h, args[0], 2, 137, 137, 3, None, args[1], 16, p(tm), args[2], None, None,
                                      p(sums))
        assert rc != 0 and b"null argument" in eng.lib.disn_last_error()
    rc = eng.lib.disn_cam_metrics(eng._h, p(a), 0, 137, 137, 3, None, p(pts), 16, p(tm), p(RT), None, None, p(sums))
    assert rc != 0 and b"max_batch" in eng.lib.disn_last_error()
    after = eng.cam_estimate(imgs[:2], want_rt=True)
    for x, y in zip(after, before):
        np.testing.assert_array_equal(bits(x), bits(y))
    missing = "cameraprediction/ortho6d/fc2/biases"
    fresh = Engine(device=0, precision="fp32", max_batch=2)
    try:
        fresh.load_weights_raw({k: v for k, v in cam_w.items() if k != missing})
        with pytest.raises(DisnError, match="missing variable " + missing):
            fresh.cam_metrics(imgs[:2], pts[:2], tm[:2], RT[:2])
        fresh.load_weights_raw({missing: np.zeros(3, np.float32)})
        with pytest.raises(DisnError, match="mis-shaped variable " + missing):
            fresh.cam_metrics(imgs[:2], pts[:2], tm[:2], RT[:2])
        fresh.load_weights_raw({missing: cam_w[missing]})
        got = fresh.cam_metrics(imgs[:2], pts[:2], tm[:2], RT[:2])
        np.testing.assert_array_equal(bits(got[0]), bits(fresh.cam_estimate(imgs[:2])))
    finally:
        fresh.close()


def _driver(root, log_dir, est_dir, bs, cam_w):
    from disn_b200 import train_sdf_cam
    np.random.seed(11)
    random.seed(11)
    return train_sdf_cam.main(["--test", "--create", "--view_dir", str(root / "views"), "--sdf_dir", str(root / "sdf"),
                               "--test_lst_dir", str(root / "lst"), "--log_dir", str(log_dir),
                               "--img_h5_dir", str(est_dir), "--batch_size", str(bs), "--verbose_freq", "5",
                               "--precision", "fp32"], weights=cam_w)


def test_driver_creates_view_files_the_sdf_drivers_read(he_weights, cam_w, golden, tmp_path, capsys):
    """--test --create on the golden fixture: at batch 1 every est file's trans_mat is Engine.cam_estimate's bits on its
    image and the rest is the source file bit for bit; batch 12 (encodes of 8 and 4) writes the same views within the
    fp32 path's bound.  create_sdf --cam_est and test_sdf_acc then read the est files."""
    from disn_b200 import create_sdf, test_sdf_acc
    from disn_b200.engine import Engine
    from tests.test_sdf_acc_cpu import write_fixture
    root = write_fixture(golden["sdf_acc_ref"], tmp_path / "tree")
    est1, est12 = tmp_path / "est1", tmp_path / "est12"
    d2, d3 = _driver(root, tmp_path / "log1", est1, 1, cam_w)
    assert len(d2) == len(d3) == 96
    out = capsys.readouterr().out
    assert sum(ln.startswith(" -- ") for ln in out.splitlines()) == 96 // 5 + 1
    assert "avg 2d dist" in out and "avg 3d dist" in out
    _driver(root, tmp_path / "log12", est12, 12, cam_w)
    files = sorted(glob.glob(str(est1 / "*" / "*" / "*.npz")))
    assert len(files) == 96
    eng = Engine(device=0, precision="fp32", max_batch=1)
    try:
        eng.load_weights_raw(cam_w)
        for f in files:
            rel = os.path.relpath(f, est1)
            src = root / "views" / rel
            with np.load(src) as s:     # the loader's image: img_arr[:, :, :4] / 255, fed as RGB
                img = (s["img_arr"][:, :, :4].astype(np.float32) / 255.)[None, :, :, :3]
            want = eng.cam_estimate(img)[0]
            with np.load(f) as z, np.load(src) as s:
                assert sorted(z.files) == sorted(s.files)
                np.testing.assert_array_equal(bits(z["trans_mat"]), bits(want))
                for k in z.files:
                    if k != "trans_mat":
                        assert z[k].dtype == s[k].dtype and z[k].tobytes() == s[k].tobytes(), (rel, k)
            with np.load(est12 / rel) as z12:
                tm12 = z12["trans_mat"]
            assert np.abs(tm12 - want).max() <= 2e-5 * np.abs(want).max(), rel
    finally:
        eng.close()
    random.seed(3)
    written = create_sdf.main(["--view_dir", str(est1), "--sdf_dir", str(root / "sdf"), "--test_lst_dir",
                               str(root / "lst"), "--log_dir", str(tmp_path / "sdflog"), "--sdf_res", "16",
                               "--view_num", "2", "--cam_est"], weights=he_weights)
    objs = sorted(glob.glob(str(tmp_path / "sdflog" / "test_objs" / "camest_17_0.0" / "*" / "*.obj")))
    assert len(objs) == 4 * 2 and sorted(written) == objs
    np.random.seed(5)
    random.seed(5)
    summary = test_sdf_acc.main(["--view_dir", str(est1), "--sdf_dir", str(root / "sdf"), "--test_lst_dir",
                                 str(root / "lst"), "--log_dir", str(tmp_path / "acclog"), "--batch_size", "8",
                                 "--img_feat_twostream"], weights=he_weights)
    assert set(summary) == set(test_sdf_acc.LOSS_KEYS) and all(np.isfinite(v) for v in summary.values())
