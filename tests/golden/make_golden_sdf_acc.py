"""Generate tests/golden/sdf_acc_ref.npz by running the REFERENCE's own view-file writer (preprocessing/create_img_h5.py
gen_obj_img_h5), loader (data/data_sdf_h5_queue.py Pt_sdf_img: refill_data_order, get_batch) and checkpoint score
(test/test_sdf_acc.py test_one_epoch with models/model_normalization.py get_loss) on a small seeded fixture.

Run in the build container only (the GPU machine has no reference tree):
    python tests/golden/make_golden_sdf_acc.py
Stubs, as in make_golden_eval.py:
  * h5py: File backed by .npz content (a missing ori_sample.h5 is read from the fixture's ori_sample.npz);
  * tensorflow: the lazy numpy graph of make_golden_eval.py, extended with constant / greater / equal / less_equal /
    to_float / cast / abs / add_n, so that the reference's own get_loss (taken from its source) runs;
  * the model: pred_sdf = twin_pred(sample_pc, imgs), a closed-form function of the fed points and image;
  * slim / tf.get_collection('regularizer'): the float32 l2 terms of the fixture's weights;
  * trimesh, joblib, create_file_lst: unused or sequential.
The fixture: 2 categories x 2 objects x 24 views, RGBA PNGs written with cv2, renderings.txt and
rendering_metadata.txt, and ori_sample.npz files in create_point_sdf_grid's layout (write_sample_file) holding analytic
signed distances of spheres.  Recorded: every view file's datasets, the epoch order, every draw, the batches, and the
printed lines; bitwise-compared images and batch arrays as SHA-256 digests.  Only the data is committed.
"""
import ast
import contextlib
import hashlib
import importlib.util
import io
import os
import random
import sys
import tempfile
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
from make_golden import _stub  # noqa: E402
import make_golden_eval as mge  # noqa: E402

CATS = {"display": "03211117", "rifle": "04090263"}
NOBJ, NVIEW, NSAMPLE, NPTS, BATCH, SEED = 2, 24, 600, 64, 4, 31


# ---------------------------------------------------------------------------------------------------------------- fixture
def twin_pred(pts, imgs):
    """The stub model's pred_sdf [B,N,1] float32: 10 (|p - c_b| - r_b) with c_b, r_b from image b's mean colour."""
    pts = np.asarray(pts, np.float32)
    m = np.asarray(imgs, np.float32).reshape(len(pts), -1, 3).mean(axis=1, dtype=np.float64).astype(np.float32)
    c = (m - np.float32(0.5)) * np.float32(0.2)
    r = np.float32(0.35) + np.float32(0.1) * m.mean(axis=1, dtype=np.float32)
    d = np.sqrt(((pts - c[:, None, :]) ** 2).sum(axis=2, dtype=np.float32))
    return (np.float32(10) * (d - r[:, None]))[..., None].astype(np.float32)


def fixture_weights():
    rng = np.random.default_rng(5)
    w = {}
    for name, shp in (("vgg_16/conv1/conv1_1/weights", (3, 3, 3, 8)), ("vgg_16/fc8/weights", (1, 1, 16, 8)),
                      ("sdfprediction/fold1/conv1/weights", (1, 1, 3, 16)),
                      ("sdfprediction_imgfeat/fold2/conv5/weights", (1, 1, 16, 1))):
        w[name] = rng.standard_normal(shp).astype(np.float32)
        w[name[:-len("weights")] + "biases"] = rng.standard_normal(shp[-1]).astype(np.float32)
    return w


def objects():
    return [(cat_id, "%s%02d" % ("ab"[ci], k)) for ci, cat_id in enumerate(CATS.values()) for k in range(NOBJ)]


def fixture_files():
    """relative path -> bytes: lst/, render/<cat>/<obj>/rendering/, sdf/<cat>/<obj>/ori_sample.npz."""
    import cv2
    from disn_b200.create_point_sdf_grid import write_sample_file
    from disn_b200.test_sdf_acc import CATS as ALL
    rng = np.random.default_rng(2025)
    files = {}
    for cat_id in ALL.values():
        objs = [o for c, o in objects() if c == cat_id]
        files["lst/%s_test.lst" % cat_id] = "".join(o + "\n" for o in objs).encode()
        files["lst/%s_train.lst" % cat_id] = b""
    with tempfile.TemporaryDirectory() as td:
        for cat_id, obj in objects():
            base = "render/%s/%s/rendering/" % (cat_id, obj)
            files[base + "renderings.txt"] = "".join("%02d.png\n" % v for v in range(NVIEW)).encode()
            meta = [(rng.uniform(0, 360), rng.uniform(25, 30), 0, rng.uniform(0.65, 0.95), 25) for _ in range(NVIEW)]
            files[base + "rendering_metadata.txt"] = "".join("%r %r %r %r %r\n" % m for m in meta).encode()
            for v in range(NVIEW):
                yy, xx = np.mgrid[:137, :137]
                img = np.zeros((137, 137, 4), np.uint8)          # colour bands: small PNGs
                img[..., :3] = rng.integers(0, 256, size=(1, 4, 3))[:, (xx // 35) % 4][0]
                img[..., 3] = np.where((yy - 68) ** 2 + (xx - 68) ** 2 < rng.integers(900, 2500), 255, 0)
                files[base + "%02d.png" % v] = cv2.imencode(".png", img)[1].tobytes()
            centre = rng.uniform(-0.1, 0.1, 3)
            radius = rng.uniform(0.3, 0.5)
            pts = rng.integers(-38, 39, size=(NSAMPLE, 3)) / 64.0        # on a 1/64 lattice: a small file
            sdf = np.linalg.norm(pts - centre, axis=1) - radius
            out = os.path.join(td, "s.npz")
            write_sample_file(out, os.path.join(td, "flag.txt"), np.c_[pts, sdf], False, rng.uniform(-0.05, 0.05, 3),
                              rng.uniform(0.4, 0.6), [-1, -1, -1, 1, 1, 1])
            files["sdf/%s/%s/ori_sample.npz" % (cat_id, obj)] = open(out, "rb").read()
    return files


# ------------------------------------------------------------------------------------------------------------- stubs
class _Dataset:
    def __init__(self, a):
        self.a = a

    def __getitem__(self, key):
        return self.a[key]


class _H5File:
    def __init__(self, path, mode="r"):
        self.path, self.mode, self.data = path, mode, {}
        if mode == "r":
            src = path if os.path.exists(path) else path[:-3] + ".npz"
            with open(src, "rb") as fh:
                z = np.load(fh)
                self.data = {k: z[k] for k in z.files}

    def keys(self):
        return self.data.keys()

    def __getitem__(self, k):
        return _Dataset(self.data[k])

    def create_dataset(self, name, data=None, dtype=None, **kw):
        self.data[name] = np.asarray(data, dtype=dtype)

    def close(self):
        if self.mode == "w":
            with open(self.path, "wb") as fh:
                np.savez(fh, **self.data)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()
        return False


def install_stubs(weights):
    mge.install_stubs()
    _stub("h5py", File=_H5File)
    _stub("trimesh")
    tf = sys.modules["tensorflow"]
    N = mge.Node
    N.__sub__ = lambda a, b: N(lambda x, y: x - y, a, b)
    N.__truediv__ = lambda a, b: N(lambda x, y: x / y, a, b)
    f32 = lambda x: np.asarray(x, np.float32)
    tf.int32 = np.int32
    tf.constant = lambda v, dtype=np.float32: f32(v)
    tf.greater = lambda a, b: N(np.greater, a, b)
    tf.less_equal = lambda a, b: N(np.less_equal, a, b)
    tf.equal = lambda a, b: N(np.equal, a, b)
    tf.to_float = lambda a: N(f32, a)
    tf.cast = lambda a, dtype: N(lambda x: np.asarray(x, dtype), a)
    tf.abs = lambda a: N(np.abs, a)
    tf.reduce_mean = lambda x, axis=None: N(lambda a: np.float32(np.mean(a, axis=axis)), x)
    l2 = lambda w: np.float32(1e-5) * (np.sum(w * w, dtype=np.float32) / np.float32(2))
    vgg = [l2(w) for k, w in weights.items() if k.startswith("vgg_16/") and k.endswith("/weights")]
    dec = [l2(w) for k, w in weights.items() if k.startswith("sdfprediction") and k.endswith("/weights")]
    tf.add_n = lambda xs: N(lambda *v: np.float32(np.sum(np.asarray(v, np.float32), dtype=np.float32)), *xs)
    tf.get_collection = lambda name: dec
    slim = SimpleNamespace(losses=SimpleNamespace(get_regularization_losses=lambda: vgg))
    return tf, slim


class _Queue:
    def __init__(self, n, fetch):
        self.n, self.fetch = n, fetch

    def __len__(self):
        return self.n


def reference_function(path, name, namespace):
    """Compile one top-level function of a reference file into `namespace` (the rest of the file needs TF)."""
    src = open(path).read()
    node = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == name)
    exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), namespace)
    return namespace[name]


def import_ref(rel, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    mod = importlib.util.module_from_spec(spec)
    sys.path.insert(0, os.path.dirname(os.path.join(REF, rel)))
    with contextlib.redirect_stdout(io.StringIO()):
        spec.loader.exec_module(mod)
    return mod


def loader_flags(batch_size):
    return SimpleNamespace(num_points=1, num_sample_points=NPTS, batch_size=batch_size, img_h=137, img_w=137,
                           cat_limit=168000, alpha=False, rot=False, threedcnn=False, img_feat_onestream=False,
                           img_feat_twostream=True, augcolorfore=False, augcolorback=False, backcolorwhite=True,
                           max_epoch=1, binary=False, multi_view=False, mask_weight=4.0)


def listinfo():
    from disn_b200.test_sdf_acc import CATS as ALL
    info, limit = [], {c: 0 for c in ALL.values()}
    for cat_id in ALL.values():
        for c, obj in objects():
            if c == cat_id:
                for render in range(24):
                    limit[cat_id] += 1
                    info.append((cat_id, obj, render))
    return info, limit


def main():
    weights = fixture_weights()
    tf, slim = install_stubs(weights)
    _stub("create_file_lst", get_all_info=lambda: (None, None, None, None))
    img_h5 = import_ref("preprocessing/create_img_h5.py", "ref_create_img_h5")
    queue_mod = import_ref("data/data_sdf_h5_queue.py", "ref_data_sdf_h5_queue")
    files = fixture_files()
    out = {"files": np.array(sorted(files)), "meta": np.array([NOBJ, NVIEW, NSAMPLE, NPTS, BATCH, SEED], np.int64),
           "cats": np.array([[k, v] for k, v in CATS.items()])}
    # the fixture's files, concatenated: file i is file_blob[file_offsets[i]:file_offsets[i + 1]]
    out["file_blob"] = np.frombuffer(b"".join(files[rel] for rel in sorted(files)), np.uint8)
    out["file_offsets"] = np.cumsum([0] + [len(files[rel]) for rel in sorted(files)]).astype(np.int64)
    for k, w in weights.items():
        out["weight/" + k] = w
    with tempfile.TemporaryDirectory() as td:
        mge.write_tree(td, files)
        view_dir = os.path.join(td, "views")
        views = {}
        for cat_id, obj in objects():
            with contextlib.redirect_stdout(io.StringIO()):
                img_h5.gen_obj_img_h5(os.path.join(td, "render"), os.path.join(view_dir, cat_id), os.path.join(td, "sdf"),
                                      cat_id, obj)
            for v in range(NVIEW):
                with np.load(os.path.join(view_dir, cat_id, obj, "%02d.h5" % v)) as z:
                    views["%s/%s/%02d" % (cat_id, obj, v)] = {k: z[k] for k in z.files}
        # one array per dataset over all views, in the order of view_ids; the decoded PNGs as digests
        out["view_ids"] = np.array(list(views))
        out["view_datasets"] = np.array(sorted(next(iter(views.values()))))
        assert all(sorted(d) == list(out["view_datasets"]) for d in views.values())
        for k in out["view_datasets"]:
            if k == "img_arr":
                out["view_img_arr_sha"] = np.array([hashlib.sha256(d[k].tobytes()).hexdigest() for d in views.values()])
                out["view_img_arr_shape"] = np.array([d[k].shape for d in views.values()])
            else:
                out["view_" + k] = np.stack([d[k] for d in views.values()])
        info = {"rendered_dir": view_dir, "sdf_dir": os.path.join(td, "sdf")}
        for bs in (BATCH, 1):
            np.random.seed(SEED)
            random.seed(SEED)
            li, limit = listinfo()
            rec = mge.Recorder()
            with contextlib.redirect_stdout(io.StringIO()):
                ds = queue_mod.Pt_sdf_img(loader_flags(bs), listinfo=li, info=info, cats_limit=limit)
                with rec.active():
                    ds.order = ds.refill_data_order()
                    batches = [ds.get_batch(i * bs) for i in range(ds.num_batches)]
            pre = "bs%d_" % bs
            out[pre + "order"] = np.array(ds.order, np.int64)
            for k, a in rec.arrays(pre + "draws").items():
                assert a.max(initial=0) < 2 ** 15
                out[k] = a.astype(np.int16)
            out[pre + "trans_mat"] = np.stack([b["trans_mat"] for b in batches])
            for k in ("pc", "sdf_pt", "sdf_val", "sdf_params", "norm_params"):      # bitwise: kept as digests
                a = np.stack([b[k] for b in batches])
                out[pre + k + "_sha"] = np.array(hashlib.sha256(a.tobytes()).hexdigest())
                out[pre + k + "_shape"] = np.array(a.shape)
            out[pre + "img_sha"] = np.array([hashlib.sha256(b["img"].tobytes()).hexdigest() for b in batches])
            out[pre + "ids"] = np.array([["%s/%s/%d" % t for t in zip(b["cat_id"], b["obj_nm"], b["view_id"])]
                                         for b in batches])
            # test_one_epoch on those batches, with the reference's get_loss over the stub model
            ns = {"tf": tf, "slim": slim, "np": np}
            get_loss = reference_function(os.path.join(REF, "models/model_normalization.py"), "get_loss", ns)
            pls = {k: mge.Node(None) for k in ("sample_pc", "sample_pc_rot", "sdf", "imgs", "trans_mat")}
            end_points = {"ref_sdf": pls["sdf"], "ref_img": pls["imgs"],
                          "pred_sdf": mge.Node(twin_pred, pls["sample_pc"], pls["imgs"]),
                          "sample_img_points": mge.Node(lambda p: p[..., :2], pls["sample_pc"])}
            flags = loader_flags(bs)
            with contextlib.redirect_stdout(io.StringIO()):
                loss, end_points = get_loss(end_points, sdf_weight=10., mask_weight=flags.mask_weight,
                                            num_sample_points=NPTS, FLAGS=flags)
            it = iter(batches)
            lines = []
            ns.update(TEST_DATASET=_Queue(len(li), lambda: next(it)), FLAGS=flags, log_string=lines.append,
                      datetime=SimpleNamespace(now=lambda: "<now>"))
            test_one_epoch = reference_function(os.path.join(REF, "test/test_sdf_acc.py"), "test_one_epoch", ns)
            ops = {"is_training_pl": mge.Node(None), "input_pls": pls, "end_points": end_points}
            with contextlib.redirect_stdout(io.StringIO()):
                test_one_epoch(mge._Session(), ops)
            out[pre + "lines"] = np.array(lines[1:])
            print("batch_size", bs, *lines[1:3], lines[-1], sep="\n  ")
    np.savez_compressed(os.path.join(HERE, "sdf_acc_ref.npz"), **out)


if __name__ == "__main__":
    main()
