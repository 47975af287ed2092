"""CPU tests of the camera checkpoint score and the estimated-camera view files against tests/golden/cam_acc_ref.npz,
made by running the reference's own camera loader, get_img_points / get_loss and train_sdf_cam's eval_one_epoch and
create_img_h5 on the fixture of sdf_acc_ref.npz (tests/golden/make_golden_cam_acc.py): the loader's draws and batches,
the driver's printed lines, .xyz files, err_log.txt and est view files, with a CPU twin engine in place of the GPU one."""
import contextlib
import hashlib
import io
import math
import random
import re
from types import SimpleNamespace

import numpy as np
import pytest

from disn_b200 import data_sdf_h5_queue_mask_imgh5_cammat as cam_data
from disn_b200 import train_sdf_cam
from disn_b200.engine import CAM_LOSS_KEYS, cam_losses
from oracle.cam_acc_oracle import cam_metric_terms
from tests.test_sdf_acc_cpu import write_fixture

K = np.array([[149.84375, 0., 68.5], [0., 149.84375, 68.5], [0., 0., 1.]], dtype=np.float32)


def kmatmul(a, b):
    """The golden's tf.matmul: products summed in k order, one float32 rounding per op."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    r = a[..., :, 0:1] * b[..., 0:1, :]
    for k in range(1, a.shape[-1]):
        r = r + a[..., :, k:k + 1] * b[..., k:k + 1, :]
    return r


def twin_pose(imgs):
    """The golden's stub camera net (make_golden_cam_acc.twin_pose): pred_RT of the fed images."""
    f = np.float32
    imgs = np.asarray(imgs, f)
    m = imgs.reshape(len(imgs), -1, 3).mean(axis=1, dtype=np.float64).astype(f)
    t = f(0.3) * (m[:, 0] - f(0.5))
    den = f(1) + t * t
    c, s = (f(1) - t * t) / den, (f(2) * t) / den
    sc = f(1) + f(0.2) * (m[:, 1] - f(0.5))
    rt = np.zeros((len(imgs), 4, 3), f)
    rt[:, 0, 0], rt[:, 0, 2], rt[:, 1, 1] = sc * c, -(sc * s), sc
    rt[:, 2, 0], rt[:, 2, 2] = sc * s, sc * c
    rt[:, 3, 0], rt[:, 3, 2] = f(0.05) * (m[:, 2] - f(0.5)), f(1.4)
    return rt


def exact_sums(terms):
    """[B,5] float64: each image's terms, exactly summed, in disn_cam_metrics's order."""
    keys = ("rotpc", "rot2d", "rot3d", "rot2d_dist", "rotmatrix")
    B = len(terms["rotmatrix"])
    return np.array([[math.fsum(terms[k][b].astype(np.float64).ravel()) for k in keys] for b in range(B)])


class TwinEngine:
    """Engine.cam_metrics on the host: the stub camera net and cam_metric_terms, exactly summed."""

    def __init__(self):
        self.calls = []

    def cam_metrics(self, imgs, pts, trans_mat, RT, K_=None):
        imgs = np.asarray(imgs, np.float32)
        assert imgs.shape[-1] == 3 and len(imgs) <= train_sdf_cam.ENGINE_BATCH
        self.calls.append(len(imgs))
        rt = twin_pose(imgs)
        tm = kmatmul(rt, np.tile(K.T[None], (len(rt), 1, 1)))
        return tm, rt, exact_sums(cam_metric_terms(pts, trans_mat, RT, tm, rt))


@pytest.fixture(scope="module")
def ref(golden):
    return golden["cam_acc_ref"]


@pytest.fixture(scope="module")
def tree(golden, tmp_path_factory):
    """The fixture tree; the view files hold the matrices the reference's gen_obj_img_h5 wrote (ours are within 1 ulp)."""
    sref = golden["sdf_acc_ref"]
    root = write_fixture(sref, tmp_path_factory.mktemp("cam_acc"))
    for i, vid in enumerate(sref["view_ids"]):
        path = root / "views" / (str(vid) + ".npz")
        with np.load(path) as z:
            d = {k: z[k] for k in z.files}
        for k in d:
            if k != "img_arr":
                d[k] = sref["view_" + k][i].astype(np.float32)
        np.savez(path, **d)
    return root


def _listinfo(tree):
    return train_sdf_cam.build_listinfo(SimpleNamespace(category="all", test_lst_dir=str(tree / "lst")),
                                        train_sdf_cam.CAM_CATS)


def _flags(bs, npts):
    return SimpleNamespace(num_points=1, num_sample_points=npts, batch_size=bs, img_h=137, img_w=137, cat_limit=168000,
                           max_epoch=1)


def _runs(ref):
    return [(int(bs), mode, int(vf)) for bs, mode, vf in ref["runs"]]


@pytest.mark.parametrize("bs", [4, 1])
def test_loader_draws_and_batches_equal_the_reference(ref, tree, bs):
    seed, npts = int(ref["meta"][1]), int(ref["meta"][0])
    np.random.seed(seed)
    random.seed(seed)
    li, limit = _listinfo(tree)
    draws = []
    ri = np.random.randint
    with contextlib.redirect_stdout(io.StringIO()):
        ds = cam_data.Pt_sdf_img(_flags(bs, npts), listinfo=li, cats_limit=limit,
                                 info={"rendered_dir": str(tree / "views"), "sdf_dir": str(tree / "sdf")})
        try:
            np.random.randint = lambda *a, **k: draws.append(ri(*a, **k)) or draws[-1]
            ds.order = ds.refill_data_order()
            batches = [ds.get_batch(i * bs) for i in range(ds.num_batches)]
        finally:
            np.random.randint = ri
    pre = "bs%d_" % bs
    assert np.array_equal(ds.order, ref[pre + "order"])
    assert np.array_equal(np.concatenate([np.ravel(d) for d in draws]), ref[pre + "draws_randint"])
    assert np.array_equal([np.size(d) for d in draws], ref[pre + "draws_randint_len"])
    assert ref[pre + "draws_sample"].size == 0
    for k in ("pc", "sdf_pt", "sdf_val", "sdf_params", "norm_params", "img", "trans_mat", "RT", "shifts"):
        a = np.stack([b[k] for b in batches])
        assert a.dtype == np.float32 and a.shape == tuple(ref[pre + k + "_shape"]), k
        assert hashlib.sha256(a.tobytes()).hexdigest() == str(ref[pre + k + "_sha"]), k
    ids = [["%s/%s/%d" % t for t in zip(b["cat_id"], b["obj_nm"], b["view_id"])] for b in batches]
    assert np.array_equal(np.array(ids), ref[pre + "ids"])


LOSS_LINE = re.compile(r"^ -- \d{3} / \d{3} -- ")
SUMMARY = re.compile(r"^avg (\w+) dist (\S+), max \w+ dist (\S+), min \w+ dist (\S+)$")


def assert_same_summary(lines, want):
    """The summary lines of eval_one_epoch: same text, numbers within 2 float32 ulp."""
    assert len(lines) == len(want) == 2
    for mine, theirs in zip(lines, want):
        m, t = SUMMARY.match(mine), SUMMARY.match(theirs)
        assert m and t and m.group(1) == t.group(1), (mine, theirs)
        for a, b in zip(m.groups()[1:], t.groups()[1:]):
            assert abs(float(a) - float(b)) <= 2 * np.spacing(np.float32(abs(float(b)))), (mine, theirs)


def run_driver(ref, tree, tmp_path, bs, mode, vf, engine, weights=None):
    weights = weights if weights is not None else \
        {str(k)[len("weight/"):]: ref[k] for k in ref.files if k.startswith("weight/")}
    seed = int(ref["meta"][1])
    np.random.seed(seed)
    random.seed(seed)
    log_dir, est_dir = tmp_path / "log", tmp_path / "est"
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        train_sdf_cam.main(["--test", "--create", "--view_dir", str(tree / "views"), "--sdf_dir", str(tree / "sdf"),
                            "--test_lst_dir", str(tree / "lst"), "--log_dir", str(log_dir), "--img_h5_dir", str(est_dir),
                            "--batch_size", str(bs), "--num_sample_points", str(int(ref["meta"][0])), "--loss_mode", mode,
                            "--verbose_freq", str(vf)], weights=weights, engine=engine)
    return out.getvalue().splitlines(), log_dir, est_dir


@pytest.mark.parametrize("run", [0, 1])
def test_driver_writes_the_reference_outputs(ref, tree, tmp_path, run):
    bs, mode, vf = _runs(ref)[run]
    pre = "bs%d_" % bs
    engine = TwinEngine()
    printed, log_dir, est_dir = run_driver(ref, tree, tmp_path, bs, mode, vf, engine)
    assert engine.calls == [bs] * (96 // bs)
    # the loss lines, apart from their time field, and the summary lines
    strip = lambda ln: ln.split("time: ")[0]
    lines = [ln for ln in printed if LOSS_LINE.match(ln)]
    want = [str(x) for x in ref[pre + "lines"]]
    assert len(lines) == len(want) > 0 and [strip(x) for x in lines] == [strip(x) for x in want]
    assert re.search(r"time: \d+\.\d\d, $", lines[0])
    assert_same_summary([ln for ln in printed if ln.startswith("avg ")], [str(x) for x in ref[pre + "summary"]])
    (log,) = log_dir.glob("log_train_*.txt")
    assert [ln for ln in log.read_text().splitlines() if LOSS_LINE.match(ln)] == lines
    # the .xyz files, err_log.txt and one overlay per written image
    (res,) = log_dir.glob("test_results_*")
    names, blob, off = ref[pre + "xyz_names"], ref[pre + "xyz_blob"], ref[pre + "xyz_offsets"]
    assert sorted(p.name for p in res.glob("*.xyz")) == [str(n) for n in names]
    for i, n in enumerate(names):
        assert (res / str(n)).read_bytes() == blob[off[i]:off[i + 1]].tobytes(), n
    assert (res / "err_log.txt").read_text() == str(ref[pre + "err_log"])
    assert len(list(res.glob("*_comp.png"))) == len(names) // 2
    # every est view file equals the one the reference's create_img_h5 wrote
    ids = [str(x) for x in ref[pre + "est_ids"]]
    assert sorted(str(p.relative_to(est_dir))[:-4] for p in est_dir.glob("*/*/*.npz")) == ids
    for i, vid in enumerate(ids):
        with np.load(est_dir / (vid + ".npz")) as z:
            assert sorted(z.files) == [str(k) for k in ref[pre + "est_datasets"]]
            assert z["img_arr"].dtype == np.uint8
            assert hashlib.sha256(z["img_arr"].tobytes()).hexdigest() == str(ref[pre + "est_img_arr_sha"][i])
            for k in z.files:
                if k != "img_arr":
                    want = ref[pre + "est_" + k][i]
                    assert z[k].dtype == want.dtype == np.float32 and z[k].tobytes() == want.tobytes(), (vid, k)


@pytest.mark.parametrize("flags,match", [([], "training"), (["--test", "--shift"], "shift"),
                                         (["--create", "--rotation"], "rotation")])
def test_refused_flags_raise(flags, match, tmp_path):
    with pytest.raises(NotImplementedError, match=match):
        train_sdf_cam.main(flags + ["--view_dir", "v", "--sdf_dir", "s", "--log_dir", str(tmp_path)], weights={})
    with pytest.raises(ValueError, match="img_h5_dir"):
        train_sdf_cam.main(["--create", "--view_dir", "v", "--sdf_dir", "s", "--log_dir", str(tmp_path)], weights={})


def test_regularization_is_the_vgg_kernels_weight_decay_only():
    w = {"vgg_16/fc8/weights": np.full((1, 1, 2, 2), 2.0, np.float32), "vgg_16/fc8/biases": np.ones(2, np.float32),
         "vgg_16/conv1/conv1_1/weights": np.ones((3, 3, 3, 1), np.float32),
         "cameraprediction/scale/fc1/weights": np.ones((4, 4), np.float32),
         "sdfprediction/fold1/conv1/weights": np.ones((1, 1, 3, 4), np.float32)}
    assert train_sdf_cam.regularization(w) == np.float32(2e-3 * (16 + 27) / 2)


def test_cam_losses_follow_the_loss_mode():
    rng = np.random.default_rng(1)
    sums = rng.uniform(0, 50, (3, 5))
    f = np.float32
    reg = f(0.125)
    base, r3, r2 = cam_losses(sums, 7, reg, "3D")
    assert list(base) == list(CAM_LOSS_KEYS) and all(type(v) is np.float32 for v in base.values())
    assert base["rotpc_loss"] == f(sums[:, 0].sum() / 2)
    assert base["rot2d_loss"] == f(sums[:, 1].sum() / 2) / f(10000)
    assert np.array_equal(r3, (sums[:, 2] / 7).astype(f)) and np.array_equal(r2, (sums[:, 3] / 7).astype(f))
    assert base["rot3d_dist"] == f(r3.astype(np.float64).mean()) and base["rot2d_dist"] == f(r2.astype(np.float64).mean())
    assert base["rotmatrix_loss"] == f(sums[:, 4].sum() / 36)
    pc, p2, mat = base["rotpc_loss"], base["rot2d_loss"], base["rotmatrix_loss"]
    for mode, loss in (("3D", pc), ("2D", p2), ("3DM", pc + mat * f(0.3)), ("mix", p2 + pc + mat)):
        v = cam_losses(sums, 7, reg, mode)[0]
        assert v["overall_loss"] == f(loss + reg) and v["regularization"] == reg, mode
