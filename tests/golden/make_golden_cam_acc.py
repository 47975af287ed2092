"""Generate tests/golden/cam_acc_ref.npz by running the REFERENCE's own view-file writer (preprocessing/create_img_h5.py
gen_obj_img_h5), camera loader (data/data_sdf_h5_queue_mask_imgh5_cammat.py Pt_sdf_img: refill_data_order, get_batch),
camera losses (cam_est/model_cam.py get_img_points, get_loss) and test driver (cam_est/train_sdf_cam.py eval_one_epoch
and create_img_h5) on the fixture of make_golden_sdf_acc.py (2 categories x 2 objects x 24 views, read back from
sdf_acc_ref.npz), at batch sizes 4 and 1, with --test and --create.

Run in the build container only (the GPU machine has no reference tree):
    python tests/golden/make_golden_cam_acc.py
Stubs, on top of make_golden_sdf_acc.py's (h5py backed by .npz, the lazy numpy `tf`):
  * tf.matmul sums its products in k order, one float32 rounding per op; concat, ones, divide, minimum, maximum, sqrt,
    square and reduce_sum (float32, in index order) are numpy's float32 ops;
  * tf.reduce_mean and tf.nn.l2_loss sum exactly (float64) and round once to float32, so that every printed value has
    one float32 answer (TF's own float32 sums can differ in the last bit);
  * the camera model: pred_RT = twin_pose(imgs), a scaled rotation about y and a translation set by the fed image's
    mean colour (rational arithmetic only); pred_trans_mat = pred_RT . K^T as in get_model (model_cam.py:102-103);
  * slim's regularisation losses: 2e-3 * sum(w^2) / 2 over the fixture's vgg_16 kernels, exact, added by add_n.
Recorded: the epoch order, every draw, the batches (digests of the bitwise-compared arrays), the loss lines and the
summary lines, every .xyz file and err_log.txt, and every view file create_img_h5 wrote.  Only the data is committed.
"""
import ast
import contextlib
import glob
import hashlib
import io
import math
import os
import random
import sys
import tempfile
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_eval as mge  # noqa: E402
import make_golden_sdf_acc as mgs  # noqa: E402
from make_golden import _stub  # noqa: E402

REF = mgs.REF
NPTS, SEED, WD = 64, 41, 2e-3
RUNS = ((4, "3DM", 2), (1, "mix", 5))      # (batch size, --loss_mode, --verbose_freq)
K = np.array([[149.84375, 0., 68.5], [0., 149.84375, 68.5], [0., 0., 1.]], dtype=np.float32)    # model_cam.py:28


def kmatmul(a, b):
    """tf.matmul with the products summed in k order, one float32 rounding per op: a [..., M, K], b [..., K, P]."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    r = a[..., :, 0:1] * b[..., 0:1, :]
    for k in range(1, a.shape[-1]):
        r = r + a[..., :, k:k + 1] * b[..., k:k + 1, :]
    return r


def twin_pose(imgs):
    """The stub camera net's pred_RT [B,4,3]: s * R_y(t) with t, s and a translation from image b's mean colour."""
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


def fixture_weights():
    rng = np.random.default_rng(6)
    w = {}
    for name, shp in (("vgg_16/conv1/conv1_1/weights", (3, 3, 3, 8)), ("vgg_16/fc8/weights", (1, 1, 16, 8)),
                      ("cameraprediction/scale/fc1/weights", (8, 4)), ("cameraprediction/ortho6d/fc3/weights", (4, 6))):
        w[name] = rng.standard_normal(shp).astype(np.float32)
        w[name[:-len("weights")] + "biases"] = rng.standard_normal(shp[-1]).astype(np.float32)
    return w


def install_stubs(weights):
    tf, _ = mgs.install_stubs(weights)
    N = mge.Node
    N.__radd__ = lambda a, b: N(lambda x, y: y + x, a, b)
    f32 = np.float32

    def reduce_sum(x, axis=None):
        def fn(a):
            a = np.moveaxis(np.asarray(a, f32), axis, 0)
            r = a[0]
            for v in a[1:]:
                r = r + v
            return r
        return N(fn, x)

    tf.matmul = lambda a, b: N(kmatmul, a, b)
    tf.concat = lambda xs, axis: N(lambda *v: np.concatenate([np.asarray(e, f32) for e in v], axis=axis), *xs)
    tf.ones = lambda shape, dtype=f32: np.ones(shape, dtype)
    tf.divide = lambda a, b: N(np.divide, a, b)
    tf.minimum = lambda a, b: N(np.minimum, a, b)
    tf.maximum = lambda a, b: N(np.maximum, a, b)
    tf.sqrt = lambda a: N(np.sqrt, a)
    tf.square = lambda a: N(np.square, a)
    tf.reduce_sum = reduce_sum
    tf.reduce_mean = lambda x, axis=None: N(lambda a: f32(np.mean(np.asarray(a, np.float64), axis=axis)), x)
    tf.nn = SimpleNamespace(l2_loss=lambda x: N(lambda a: f32(np.sum(np.square(np.asarray(a, f32)), dtype=np.float64) / 2), x))
    vgg = [WD * float(np.sum(np.asarray(w, np.float64) ** 2)) / 2 for k, w in weights.items()
           if k.startswith("vgg_16/") and k.endswith("/weights")]
    tf.add_n = lambda xs: N(lambda *v: f32(math.fsum(v)), *xs)
    slim = SimpleNamespace(losses=SimpleNamespace(get_regularization_losses=lambda: vgg))
    return tf, slim


def cat_list():
    """cam_est/train_sdf_cam.py:122 CAT_LIST, read from its source."""
    src = open(os.path.join(REF, "cam_est/train_sdf_cam.py")).read()
    node = next(n for n in ast.parse(src).body if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", "") == "CAT_LIST")
    return ast.literal_eval(node.value)


def listinfo(lst_dir):
    """cam_est/train_sdf_cam.py:144-151 (TEST_LISTINFO, cats_limit_test)."""
    info, limit = [], {}
    for cat in cat_list():
        limit[cat] = 0
    for cat in cat_list():
        with open(os.path.join(lst_dir, "%s_test.lst" % cat)) as f:
            for line in f.read().splitlines():
                for render in range(24):
                    limit[cat] += 1
                    info.append((cat, line.strip(), render))
    return info, limit


def flags(bs, loss_mode, verbose_freq, img_h5_dir):
    return SimpleNamespace(num_points=1, num_sample_points=NPTS, batch_size=bs, img_h=137, img_w=137, cat_limit=168000,
                           max_epoch=1, img_feat=True, shift=False, rotation=False, loss_mode=loss_mode,
                           verbose_freq=verbose_freq, test=True, create=True, img_h5_dir=img_h5_dir)


def pack_files(paths, root):
    """relative names, concatenated bytes and offsets of the given files."""
    data = [open(p, "rb").read() for p in paths]
    return (np.array([os.path.relpath(p, root) for p in paths]), np.frombuffer(b"".join(data), np.uint8),
            np.cumsum([0] + [len(d) for d in data]).astype(np.int64))


def main():
    sdf_ref = np.load(os.path.join(HERE, "sdf_acc_ref.npz"))
    weights = fixture_weights()
    tf, slim = install_stubs(weights)
    _stub("create_file_lst", get_all_info=lambda: (None, None, None, None))
    img_h5 = mgs.import_ref("preprocessing/create_img_h5.py", "ref_create_img_h5")
    queue_mod = mgs.import_ref("data/data_sdf_h5_queue_mask_imgh5_cammat.py", "ref_data_cammat")
    files = {str(rel): sdf_ref["file_blob"][sdf_ref["file_offsets"][i]:sdf_ref["file_offsets"][i + 1]].tobytes()
             for i, rel in enumerate(sdf_ref["files"])}
    out = {"meta": np.array([NPTS, SEED], np.int64), "runs": np.array([[str(x) for x in r] for r in RUNS])}
    for k, w in weights.items():
        out["weight/" + k] = w
    with tempfile.TemporaryDirectory() as td:
        mge.write_tree(td, files)
        view_dir = os.path.join(td, "views")
        for cat_id, obj in mgs.objects():
            with contextlib.redirect_stdout(io.StringIO()):
                img_h5.gen_obj_img_h5(os.path.join(td, "render"), os.path.join(view_dir, cat_id), os.path.join(td, "sdf"),
                                      cat_id, obj)
        info = {"rendered_dir": view_dir, "rendered_dir_v2": os.path.join(td, "render"), "sdf_dir": os.path.join(td, "sdf"), "iso_value": 0.003}
        for bs, loss_mode, verbose_freq in RUNS:
            pre = "bs%d_" % bs
            est_dir = os.path.join(td, "est%d" % bs)
            result_path = os.path.join(td, "results%d" % bs)
            os.makedirs(result_path)
            FLAGS = flags(bs, loss_mode, verbose_freq, est_dir)
            np.random.seed(SEED)
            random.seed(SEED)
            li, limit = listinfo(os.path.join(td, "lst"))
            rec = mge.Recorder()
            with contextlib.redirect_stdout(io.StringIO()):
                ds = queue_mod.Pt_sdf_img(FLAGS, listinfo=li, info=info, cats_limit=limit)
                with rec.active():
                    ds.order = ds.refill_data_order()
                    batches = [ds.get_batch(i * bs) for i in range(ds.num_batches)]
            out[pre + "order"] = np.array(ds.order, np.int64)
            for k, a in rec.arrays(pre + "draws").items():
                assert a.max(initial=0) < 2 ** 15
                out[k] = a.astype(np.int16)
            for k in ("pc", "sdf_pt", "sdf_val", "sdf_params", "norm_params", "img", "trans_mat", "RT", "shifts"):
                a = np.stack([b[k] for b in batches])
                out[pre + k + "_sha"] = np.array(hashlib.sha256(a.tobytes()).hexdigest())
                out[pre + k + "_shape"] = np.array(a.shape)
            out[pre + "ids"] = np.array([["%s/%s/%d" % t for t in zip(b["cat_id"], b["obj_nm"], b["view_id"])]
                                         for b in batches])
            # get_model's tail (model_cam.py:97-109) around the stub camera net, then the reference's get_loss
            ns = {"tf": tf, "slim": slim, "np": np}
            get_img_points = mgs.reference_function(os.path.join(REF, "cam_est/model_cam.py"), "get_img_points", ns)
            get_loss = mgs.reference_function(os.path.join(REF, "cam_est/model_cam.py"), "get_loss", ns)
            pls = {k: mge.Node(None, shape=s) for k, s in (("sample_pc", (bs, NPTS, 3)), ("sample_pc_rot", (bs, NPTS, 3)),
                                                           ("imgs", (bs, 137, 137, 3)), ("trans_mat", (bs, 4, 3)),
                                                           ("RT", (bs, 4, 3)), ("shifts", (bs, 2)))}
            pred_RT = mge.Node(twin_pose, pls["imgs"])
            with contextlib.redirect_stdout(io.StringIO()):
                sample_img_points, gt_xy = get_img_points(pls["sample_pc"], pls["trans_mat"], pls["shifts"], FLAGS)
                pred_trans_mat = tf.matmul(pred_RT, np.tile(K.T[None], (bs, 1, 1)))
                pred_sample_img_points, pred_xy = get_img_points(pls["sample_pc"], pred_trans_mat, None, FLAGS)
                end_points = {"RT": pls["RT"], "gt_xyshift": pls["shifts"], "trans_mat": pls["trans_mat"],
                              "sample_pc": pls["sample_pc"], "ref_img": pls["imgs"], "pred_RT": pred_RT,
                              "pred_xyshift": None, "sample_img_points": sample_img_points, "gt_xy": gt_xy,
                              "pred_sample_img_points": pred_sample_img_points, "pred_trans_mat": pred_trans_mat,
                              "pred_xy": pred_xy}
                loss, end_points = get_loss(end_points, sdf_weight=10., FLAGS=FLAGS)
            it = iter(batches)
            lines = []
            ns.update(VALID_DATASET=mgs._Queue(len(li), lambda: next(it)), FLAGS=FLAGS, BATCH_SIZE=bs,
                      TEST_RESULT_PATH=result_path, log_string=lines.append, time=__import__("time"), os=os, info=info,
                      cv2=__import__("cv2"), h5py=sys.modules["h5py"])
            ns["create_img_h5"] = mgs.reference_function(os.path.join(REF, "cam_est/train_sdf_cam.py"), "create_img_h5", ns)
            eval_one_epoch = mgs.reference_function(os.path.join(REF, "cam_est/train_sdf_cam.py"), "eval_one_epoch", ns)
            ops = {"is_training_pl": mge.Node(None), "input_pls": pls, "loss": loss, "end_points": end_points}
            with contextlib.redirect_stdout(io.StringIO()) as printed:
                eval_one_epoch(mge._Session(), ops)
            out[pre + "lines"] = np.array(lines)
            out[pre + "summary"] = np.array([ln for ln in printed.getvalue().splitlines() if ln.startswith("avg ")])
            res = sorted(glob.glob(os.path.join(result_path, "*.xyz")))
            out[pre + "xyz_names"], out[pre + "xyz_blob"], out[pre + "xyz_offsets"] = pack_files(res, result_path)
            out[pre + "err_log"] = np.array(open(os.path.join(result_path, "err_log.txt")).read())
            # the est view files: ids, then one array per dataset (img_arr as digests, bitwise-compared)
            est = sorted(glob.glob(os.path.join(est_dir, "*", "*", "*.h5")))
            out[pre + "est_ids"] = np.array([os.path.relpath(p, est_dir)[:-3] for p in est])
            zs = [dict(np.load(p)) for p in est]
            out[pre + "est_datasets"] = np.array(sorted(zs[0]))
            for k in zs[0]:
                if k == "img_arr":
                    out[pre + "est_img_arr_sha"] = np.array([hashlib.sha256(z[k].tobytes()).hexdigest() for z in zs])
                else:
                    out[pre + "est_" + k] = np.stack([z[k] for z in zs])
            print("batch_size", bs, lines[0], lines[-1], *out[pre + "summary"], "%d est files" % len(est), sep="\n  ")
    np.savez_compressed(os.path.join(HERE, "cam_acc_ref.npz"), **out)


if __name__ == "__main__":
    main()
