"""The evaluation drivers (disn_b200/eval_cd_emd.py, eval_f_score.py, eval_iou.py) against the reference's own scripts:
tests/golden/eval_ref.npz holds what test/test_cd_emd.py, test/test_f_score.py and test/test_iou.py drew and printed on
a small fixture dataset (tests/golden/make_golden_eval.py).  Here the drivers run on the same files with the CPU twin
engine (oracle/eval_oracle.py) and must reproduce every draw and every printed result line exactly."""
import contextlib
import io
import os
import random
import re

import numpy as np
import pytest

from disn_b200 import eval_cd_emd, eval_common, eval_f_score, eval_iou
from oracle.eval_oracle import EvalTwin

THRESHOLDS = [[0.5], [1], [2], [5], [10], [20]]


# ------------------------------------------------------------------------------------------------------------ helpers
class Fixture:
    def __init__(self, g, root):
        self.g = g
        self.root = str(root)
        for i, rel in enumerate(g["files"]):
            p = os.path.join(self.root, str(rel))
            os.makedirs(os.path.dirname(p), exist_ok=True)
            with open(p, "wb") as fh:
                fh.write(g["file_%d" % i].tobytes())
        self.gt, self.pred, self.lst = (os.path.join(self.root, d) for d in ("gt", "pred", "lst"))
        self.cats = {str(k): str(v) for k, v in g["cats"]}
        self.view_num, self.npts, self.dim, self.seed_cd, self.seed_pnt, self.seed_iou = (int(x) for x in g["meta"])
        self.truethreshold = float(g["truethreshold"])
        self.pattern = str(g["line_pattern"])

    def lines(self, text):
        text = text.replace(self.root, "<root>")
        return [ln for ln in text.splitlines() if re.match(self.pattern, ln)]

    def run(self, fn, seed):
        """fn() under np.random.seed / random.seed(seed) -> (result, draws, printed result lines)."""
        np.random.seed(seed)
        random.seed(seed)
        draws = {"randint": [], "sample": []}
        ri, rs = np.random.randint, random.sample

        def randint(*a, **k):
            r = ri(*a, **k)
            draws["randint"].append(np.asarray(r, np.int64).reshape(-1))
            return r

        def sample(population, k):
            r = rs(population, k)
            draws["sample"].append(np.array([population.index(x) for x in r], np.int64))
            return r

        buf = io.StringIO()
        np.random.randint, random.sample = randint, sample
        try:
            with contextlib.redirect_stdout(buf):
                res = fn()
        finally:
            np.random.randint, random.sample = ri, rs
        return res, draws, self.lines(buf.getvalue())

    def assert_draws(self, draws, prefix):
        g = self.g
        for kind in ("randint", "sample"):
            got = draws[kind]
            assert [len(x) for x in got] == list(g[prefix + "_%s_len" % kind]), (prefix, kind)
            cat = np.concatenate(got) if got else np.zeros(0, np.int64)
            np.testing.assert_array_equal(cat, g[prefix + "_" + kind], err_msg=prefix + " " + kind)

    def cd_emd(self, batch_size):
        return self.run(lambda: eval_cd_emd.cd_emd_all(self.cats, self.pred, self.gt, self.lst, view_num=self.view_num,
                                                       num_sample_points=self.npts, batch_size=batch_size), self.seed_cd)

    def save_pnt(self):
        def save():
            eval_cd_emd.save_all_cat_gt_pnt(self.cats, self.gt, self.lst, num_sample_points=self.npts)
            eval_cd_emd.save_all_cat_pred_pnt(self.cats, self.pred, self.lst, view_num=self.view_num,
                                              num_sample_points=self.npts)
        return self.run(save, self.seed_pnt)

    def f_score(self, batch_size=None):
        bs = self.view_num if batch_size is None else batch_size
        return self.run(lambda: eval_f_score.cal_f_score_all_cat(self.cats, self.pred, self.gt, self.lst, THRESHOLDS,
                                                                 self.truethreshold, view_num=self.view_num,
                                                                 num_sample_points=self.npts, batch_size=bs), 0)

    def iou(self):
        return self.run(lambda: eval_iou.iou_all(self.cats, self.pred, self.gt, self.lst, dim=self.dim,
                                                 view_num=self.view_num), self.seed_iou)


def cd_numbers(rows_by_cat):
    objs, cats = [], []
    for rows, avg_cf, avg_emd in rows_by_cat.values():
        objs += [[float(x) for x in r[1:]] for r in rows]
        cats.append([float(avg_cf), float(avg_emd)])
    return np.array(objs), np.array(cats)


@pytest.fixture
def fx(golden, tmp_path):
    return Fixture(golden["eval_ref"], tmp_path / "fx")


@pytest.fixture
def twin(monkeypatch):
    t = EvalTwin()
    for mod in (eval_cd_emd, eval_f_score, eval_iou):
        monkeypatch.setattr(mod, "_engine", lambda: t)
    return t


# -------------------------------------------------------------------------------------------------------------- golden
@pytest.mark.parametrize("batch_size", ["view_num", 1])
def test_cd_emd_reproduces_the_reference_script(fx, twin, batch_size):
    bs = fx.view_num if batch_size == "view_num" else 1
    res, draws, lines = fx.cd_emd(bs)
    prefix = "cd_emd_bs%d" % bs
    fx.assert_draws(draws, prefix)
    assert lines == list(fx.g[prefix + "_lines"])
    objs, cats = cd_numbers(res)
    # the printed values are str() of float32 / float64 (shortest round trip), so equal lines mean equal bits
    np.testing.assert_array_equal(np.float32(objs), np.float32(fx.g[prefix + "_obj"]))
    np.testing.assert_array_equal(cats, fx.g[prefix + "_cat"])


def test_save_pnt_and_f_score_reproduce_the_reference_scripts(fx, twin):
    _, draws, lines = fx.save_pnt()
    fx.assert_draws(draws, "save_pnt")
    assert lines == list(fx.g["save_pnt_lines"])
    for rel, want in zip(fx.g["pnt_files"], fx.g["pnt_values"]):
        path = os.path.join(fx.root, str(rel))
        got = np.loadtxt(path, dtype=float, delimiter=",")
        assert got.shape == (fx.npts, 3)
        np.testing.assert_array_equal(got.astype(np.float32), want, err_msg=str(rel))
        with open(path) as fh:
            assert len(fh.readline().split(",")) == 3                  # np.savetxt(..., delimiter=',')
    # first run computes and writes the per-object caches, the second reads them back
    for path in ("computed", "cached"):
        (per_cat, pre, rec, f), _, lines = fx.f_score()
        assert lines == list(fx.g["f_score_%s_lines" % path]), path
        assert set(per_cat) == set(fx.cats) and all(c[2] == 3 for c in per_cat.values())
        np.testing.assert_array_equal(f, 2 * (pre * rec) / (pre + rec))
    for cat_id in fx.cats.values():
        d = os.path.join(fx.pred, "pnt_%d_%s" % (fx.npts, cat_id))
        assert sorted(f for f in os.listdir(d) if f.startswith("for_dist_")) == \
            sorted("for_dist_%s.txt" % o for o in eval_common.read_lst(os.path.join(fx.lst, cat_id + "_test.lst")))


def test_iou_reproduces_the_reference_script(fx, twin):
    res, draws, lines = fx.iou()
    fx.assert_draws(draws, "iou")
    assert lines == list(fx.g["iou_lines"])
    assert set(res) == set(fx.cats)


# ------------------------------------------------------------------------------------------------------------- behaviour
def test_f_score_refuses_to_compute_without_batch_size_view_num(fx, twin):
    fx.save_pnt()
    with pytest.raises(NotImplementedError):
        fx.f_score(batch_size=1)


def test_cd_emd_refuses_other_batch_sizes(fx, twin):
    with pytest.raises(ValueError, match="batch_size"):
        fx.cd_emd(2)


def test_missing_object_raises_key_error(fx, twin):
    fx.save_pnt()
    cat_id = fx.cats["display"]
    with open(os.path.join(fx.lst, cat_id + "_test.lst"), "a") as fh:
        fh.write("zz99\n")
    cats = {"display": cat_id}
    with pytest.raises(KeyError, match="zz99"):
        eval_cd_emd.cd_emd_all(cats, fx.pred, fx.gt, fx.lst, view_num=fx.view_num, num_sample_points=16,
                               batch_size=fx.view_num)
    with pytest.raises(KeyError, match="zz99"):
        eval_iou.iou_all(cats, fx.pred, fx.gt, fx.lst, dim=16, view_num=fx.view_num)
    os.makedirs(os.path.join(fx.gt, cat_id, "zz99"))
    np.savetxt(os.path.join(fx.gt, cat_id, "zz99", "pnt_%d.txt" % fx.npts), np.zeros((fx.npts, 3)), delimiter=",")
    with pytest.raises(KeyError, match="zz99"):
        eval_f_score.cal_f_score_all_cat(cats, fx.pred, fx.gt, fx.lst, THRESHOLDS, 2.5, view_num=fx.view_num,
                                         num_sample_points=fx.npts, batch_size=fx.view_num)


def test_faceless_mesh_raises_value_error_naming_the_file(fx, twin):
    cat_id = fx.cats["rifle"]
    bad = os.path.join(fx.pred, cat_id, "%s_d13_01.obj" % cat_id)
    with open(bad, "w") as fh:
        fh.write("".join("v %.6f 0.1 0.2\n" % (i / 40) for i in range(40)))       # > 200 bytes, vertices only
    with pytest.raises(ValueError, match=re.escape(bad)):
        eval_iou.iou_pymesh(bad, bad, dim=16)
    np.random.seed(0)
    random.seed(0)
    with pytest.raises(ValueError, match="no faces"):
        eval_iou.iou_views(os.path.join(fx.gt, cat_id, "d13", "isosurf.obj"), [bad], dim=16)


def test_category_dicts():
    assert len(eval_common.select_cats("all")) == 13
    assert eval_common.select_cats("chair") == {"chair": "03001627"}
    clean = eval_common.select_cats("clean")
    assert sorted(clean) == ["cabinet", "display", "rifle", "speaker", "watercraft"]
    assert sorted(eval_common.select_cats("clean", eval_common.CATS_CLEAN_IOU)) == sorted(list(clean) + ["lamp"])
    with pytest.raises(KeyError):
        eval_common.select_cats("teapot")


def test_cli_single_category_and_save_pnt(fx, twin, capsys):
    cat_id = fx.cats["rifle"]
    np.random.seed(1)
    random.seed(1)
    out = eval_cd_emd.main(["--cal_dir", fx.pred, "--gt_dir", fx.gt, "--test_lst_dir", fx.lst, "--category", "rifle",
                            "--view_num", str(fx.view_num), "--num_sample_points", "32", "--batch_size",
                            str(fx.view_num), "--save_pnt", "--gpu", "0"])
    assert list(out) == ["rifle"] and len(out["rifle"][0]) == 3
    objs = eval_common.read_lst(os.path.join(fx.lst, cat_id + "_test.lst"))
    for o in objs:
        assert os.path.isfile(os.path.join(fx.gt, cat_id, o, "pnt_32.txt"))
        for v in range(fx.view_num):
            p = os.path.join(fx.pred, "pnt_32_" + cat_id, "pnt_%s_%02d.txt" % (o, v))
            assert np.loadtxt(p, delimiter=",").shape == (32, 3), p
    assert not os.path.exists(os.path.join(fx.pred, "pnt_32_" + fx.cats["display"]))
    per_cat, pre, rec, f = eval_f_score.main(["--cal_dir", fx.pred, "--gt_dir", fx.gt, "--test_lst_dir", fx.lst,
                                              "--category", "rifle", "--view_num", str(fx.view_num),
                                              "--num_sample_points", "32", "--truethreshold", "2.5",
                                              "--batch_size", str(fx.view_num)])
    assert list(per_cat) == ["rifle"] and pre.shape == (6,) and np.all(np.diff(pre) >= 0)
    res = eval_iou.main(["--cal_dir", fx.pred, "--gt_dir", fx.gt, "--test_lst_dir", fx.lst, "--category", "rifle",
                         "--view_num", str(fx.view_num), "--dim", "24"])
    assert list(res) == ["rifle"] and 0 < res["rifle"][0] < 1
    assert "cat_nm: rifle" in capsys.readouterr().out


def test_drivers_have_no_import_time_side_effects():
    import subprocess
    import sys
    code = ("from disn_b200 import eval_cd_emd as a, eval_f_score as b, eval_iou as c; "
            "assert a._ENGINE is None and b._ENGINE is None and c._ENGINE is None")
    r = subprocess.run([sys.executable, "-c", code, "--bogus"], capture_output=True, text=True,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0 and r.stdout == "", r.stderr
