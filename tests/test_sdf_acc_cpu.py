"""CPU tests of the test-set path against tests/golden/sdf_acc_ref.npz, made by running the reference's own
gen_obj_img_h5, Pt_sdf_img and test_sdf_acc.test_one_epoch (with its get_loss) on the fixture stored there
(tests/golden/make_golden_sdf_acc.py): the view files, the loader's draws and batches, and the driver's printed lines
with a CPU twin engine in place of the GPU one."""
import contextlib
import hashlib
import io
import random
import re
from types import SimpleNamespace

import numpy as np
import pytest

from disn_b200 import create_img_h5, data_sdf_h5_queue, test_sdf_acc


def twin_pred(pts, imgs):
    """The golden's stub model (make_golden_sdf_acc.twin_pred): pred_sdf of the fed points and images."""
    pts = np.asarray(pts, np.float32)
    m = np.asarray(imgs, np.float32).reshape(len(pts), -1, 3).mean(axis=1, dtype=np.float64).astype(np.float32)
    c = (m - np.float32(0.5)) * np.float32(0.2)
    r = np.float32(0.35) + np.float32(0.1) * m.mean(axis=1, dtype=np.float32)
    d = np.sqrt(((pts - c[:, None, :]) ** 2).sum(axis=2, dtype=np.float32))
    return (np.float32(10) * (d - r[:, None]))[..., None].astype(np.float32)


class TwinEngine:
    """Engine.encode / sdf_metrics on the host: the twin model and the metric's float32 terms, summed in float64."""

    def encode(self, imgs):
        self.imgs = np.asarray(imgs, np.float32)

    def sdf_metrics(self, pts, trans_mat, sdf_val, iso_offset=0.003, sdf_weight=10.0, mask_weight=4.0):
        p = twin_pred(pts, self.imgs).reshape(len(self.imgs), -1)
        g = np.asarray(sdf_val, np.float32).reshape(p.shape) - np.float32(iso_offset)
        w = (g <= np.float32(0.01)).astype(np.float32) * np.float32(mask_weight) + (g > np.float32(0.01)).astype(np.float32)
        wt = np.abs(g * np.float32(sdf_weight) - p) * w
        rt = np.abs(g - p / np.float32(sdf_weight))
        return (((g > 0) == (p > 0)).sum(axis=1).astype(np.int64), wt.astype(np.float64).sum(axis=1),
                rt.astype(np.float64).sum(axis=1))


@pytest.fixture(scope="module")
def ref(golden):
    return golden["sdf_acc_ref"]


def write_fixture(ref, root):
    """The golden's fixture tree under root, with the view files of create_img_h5 under root/views."""
    blob, off = ref["file_blob"], ref["file_offsets"]
    for i, rel in enumerate(ref["files"]):
        p = root / str(rel)
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(blob[off[i]:off[i + 1]].tobytes())
    views = root / "views"
    with contextlib.redirect_stdout(io.StringIO()):
        for cat_id, obj in _objects(ref):
            create_img_h5.gen_obj_img_h5(str(root / "render"), str(views / cat_id), str(root / "sdf"), cat_id, obj)
    return root


@pytest.fixture(scope="module")
def tree(ref, tmp_path_factory):
    return write_fixture(ref, tmp_path_factory.mktemp("sdf_acc"))


def _objects(ref):
    return sorted({tuple(str(k).split("/")[:2]) for k in ref["view_ids"]})


def _flags(batch_size, npts, **kw):
    d = dict(num_points=1, num_sample_points=npts, batch_size=batch_size, img_h=137, img_w=137,
             cat_limit=168000, max_epoch=1, backcolorwhite=True, mask_weight=4.0)
    d.update(kw)
    return SimpleNamespace(**d)


LINE = re.compile(r"([a-z_]+): (-?[0-9.]+), ")


def score_lines(text):
    return [ln for ln in text.splitlines() if re.match(r"^( -- \d{3} / \d{3} -- |Summary: )", ln)]


def assert_same_lines(lines, want):
    """Same prefix, keys, order and format; accuracy and regularization exact.  The means may differ in the last float32
    bits, because the reference's reduce_mean sums in float32 and sdf_metrics in float64."""
    assert len(lines) == len(want) > 0
    for mine, theirs in zip(lines, want):
        km, kt = LINE.findall(mine), LINE.findall(theirs)
        assert mine.split("accuracy")[0] == theirs.split("accuracy")[0]
        assert [k for k, _ in km] == [k for k, _ in kt] == list(test_sdf_acc.LOSS_KEYS)
        for (k, a), (_, b) in zip(km, kt):
            if k in ("accuracy", "regularization"):
                assert a == b, (k, mine, theirs)
            else:
                assert abs(float(a) - float(b)) <= 4 * np.spacing(np.float32(abs(float(b)))) + 1e-6, (k, mine, theirs)


def _listinfo(ref):
    info, limit = [], {c: 0 for c in test_sdf_acc.CATS.values()}
    objs = _objects(ref)
    for cat_id in test_sdf_acc.CATS.values():
        for c, obj in objs:
            if c == cat_id:
                for v in range(24):
                    limit[cat_id] += 1
                    info.append((cat_id, obj, v))
    return info, limit


def test_view_files_equal_the_reference(ref, tree):
    ids = [str(k) for k in ref["view_ids"]]
    assert len(ids) == 4 * 24
    for i, vid in enumerate(ids):
        with np.load(tree / "views" / (vid + ".npz")) as z:
            assert sorted(z.files) == list(ref["view_datasets"])
            img = z["img_arr"]
            assert img.dtype == np.uint8 and img.shape == tuple(ref["view_img_arr_shape"][i])
            assert hashlib.sha256(img.tobytes()).hexdigest() == str(ref["view_img_arr_sha"][i])
            for k in ("K", "RT", "obj_rot_mat", "regress_mat", "trans_mat"):
                want = ref["view_" + k][i]
                assert z[k].dtype == np.float32 and z[k].shape == want.shape, k
                np.testing.assert_array_max_ulp(z[k], want.astype(np.float32), maxulp=1)
    # an existing view file is kept as it is
    f = tree / "views" / _objects(ref)[0][0] / _objects(ref)[0][1] / "00.npz"
    before = f.stat().st_mtime_ns
    with contextlib.redirect_stdout(io.StringIO()) as out:
        assert create_img_h5.gen_obj_img_h5(str(tree / "render"), str(tree / "views" / _objects(ref)[0][0]),
                                            str(tree / "sdf"), *_objects(ref)[0]) == []
    assert "exist!" in out.getvalue() and f.stat().st_mtime_ns == before


@pytest.mark.parametrize("bs", [4, 1])
def test_loader_draws_and_batches_equal_the_reference(ref, tree, bs):
    seed = int(ref["meta"][5])
    np.random.seed(seed)
    random.seed(seed)
    li, limit = _listinfo(ref)
    draws = {"randint": [], "sample": []}
    ri, rs = np.random.randint, random.sample
    with contextlib.redirect_stdout(io.StringIO()):
        ds = data_sdf_h5_queue.Pt_sdf_img(_flags(bs, int(ref["meta"][3])), listinfo=li, cats_limit=limit,
                                          info={"rendered_dir": str(tree / "views"), "sdf_dir": str(tree / "sdf")})
        try:
            np.random.randint = lambda *a, **k: draws["randint"].append(ri(*a, **k)) or draws["randint"][-1]
            random.sample = lambda pop, k: draws["sample"].append(rs(pop, k)) or draws["sample"][-1]
            ds.order = ds.refill_data_order()
            batches = [ds.get_batch(i * bs) for i in range(ds.num_batches)]
        finally:
            np.random.randint, random.sample = ri, rs
    pre = "bs%d_" % bs
    assert np.array_equal(ds.order, ref[pre + "order"])
    assert np.array_equal(np.concatenate([np.ravel(d) for d in draws["randint"]]), ref[pre + "draws_randint"])
    assert np.array_equal(np.concatenate([np.asarray(d) for d in draws["sample"]]), ref[pre + "draws_sample"])
    for k in ("pc", "sdf_pt", "sdf_val", "sdf_params", "norm_params"):
        a = np.stack([b[k] for b in batches])
        assert a.dtype == np.float32 and a.shape == tuple(ref[pre + k + "_shape"]), k
        assert hashlib.sha256(a.tobytes()).hexdigest() == str(ref[pre + k + "_sha"]), k
    np.testing.assert_array_max_ulp(np.stack([b["trans_mat"] for b in batches]), ref[pre + "trans_mat"], maxulp=1)
    assert [hashlib.sha256(b["img"].tobytes()).hexdigest() for b in batches] == list(ref[pre + "img_sha"])
    ids = [["%s/%s/%d" % t for t in zip(b["cat_id"], b["obj_nm"], b["view_id"])] for b in batches]
    assert np.array_equal(np.array(ids), ref[pre + "ids"])


@pytest.mark.parametrize("bs", [4, 1])
def test_driver_prints_the_reference_lines(ref, tree, bs, tmp_path, capsys):
    weights = {str(k)[len("weight/"):]: ref[k] for k in ref.files if k.startswith("weight/")}
    seed = int(ref["meta"][5])
    np.random.seed(seed)
    random.seed(seed)
    log_dir = tmp_path / "log"
    test_sdf_acc.main(["--view_dir", str(tree / "views"), "--sdf_dir", str(tree / "sdf"), "--test_lst_dir",
                       str(tree / "lst"), "--log_dir", str(log_dir), "--batch_size", str(bs), "--num_sample_points",
                       str(int(ref["meta"][3])), "--img_feat_twostream", "--backcolorwhite"],
                      weights=weights, engine=TwinEngine())
    lines = score_lines(capsys.readouterr().out)
    assert_same_lines(lines, [str(x) for x in ref["bs%d_lines" % bs]])
    log = (log_dir / "log_test.txt").read_text().splitlines()
    assert log[-len(lines):] == lines


@pytest.mark.parametrize("flag", ["alpha", "rot", "binary", "threedcnn", "multi_view"])
def test_refused_flags_raise(flag, tmp_path):
    with pytest.raises(NotImplementedError, match=flag):
        data_sdf_h5_queue.Pt_sdf_img(SimpleNamespace(**{flag: True}), listinfo=[], info={}, cats_limit={})
    with pytest.raises(NotImplementedError, match=flag):
        test_sdf_acc.main(["--view_dir", "v", "--sdf_dir", "s", "--log_dir", str(tmp_path), "--img_feat_twostream",
                           "--" + flag], weights={})


def test_regularization_is_half_the_weight_decay_of_every_conv_kernel():
    w = {"vgg_16/fc8/weights": np.full((1, 1, 2, 2), 2.0, np.float32), "vgg_16/fc8/biases": np.ones(2, np.float32),
         "sdfprediction/fold1/conv1/weights": np.ones((1, 1, 3, 4), np.float32), "other/weights": np.ones(5, np.float32)}
    assert test_sdf_acc.regularization(w) == np.float32(1e-5 * (16 + 12) / 2)
