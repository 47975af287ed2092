"""Camera checkpoint score and estimated-camera view files, the reference's ``cam_est/train_sdf_cam.py --test`` and
``--create`` (train :235-347 with the --test/--create branch :324-327, eval_one_epoch :459-565, create_img_h5 :568-612).

Every (object, view) of the test lists is fed through the camera network (Engine.cam_metrics: the VGG-16 embedding,
the pose heads and one reduction kernel).  Every ``--verbose_freq``-th batch prints the loss line (rotpc_loss,
rot2d_loss, rot3d_dist, rot2d_dist, rotmatrix_loss, regularization, overall_loss, time) and writes, for each of its
images, ``<cat>_<obj>_<view>_gt.xyz`` / ``_pred.xyz`` (the samples through RT and pred_RT), a line of ``err_log.txt`` and
the ``_comp.png`` overlay into ``<log_dir>/test_results_<time>``.  The run ends with the ``avg/max/min 2d dist`` and
``3d dist`` lines; everything logged also goes to ``<log_dir>/log_train_<datetime>.txt``.  With ``--create`` each view
file is copied to ``<img_h5_dir>/<cat>/<obj>/%02d.npz`` with ``trans_mat`` replaced by the predicted one, so that
``create_sdf --cam_est --view_dir <img_h5_dir>`` and ``test_sdf_acc --view_dir <img_h5_dir>`` read it as they read
the source.  As in the reference, only whole batches are scored: the last len % batch_size views are not.

``regularization`` is a constant of the checkpoint: 2e-3 * sum(w^2) / 2 over the VGG-16 kernels (get_model passes
wd=2e-3 to slim's conv regulariser; the pose heads carry no weight decay).  The engine encodes at most 8 images at a
time, so a larger batch is scored in groups of 8 whose per-image sums are concatenated.  Training (no --test and no
--create), --shift and --rotation are refused.

    python -m disn_b200.train_sdf_cam --test --create --restore_model checkpoint/cam_DISN --log_dir checkpoint/cam_DISN \\
        --view_dir V --sdf_dir S --test_lst_dir L --img_h5_dir V_est --batch_size 32 --loss_mode 3DM --verbose_freq 1
"""
from __future__ import annotations

import argparse
import os
import time
from datetime import datetime

import numpy as np

from . import data_sdf_h5_queue_mask_imgh5_cammat as data
from .engine import CAM_LOSS_KEYS, cam_losses
from .test_sdf_acc import CATS, build_listinfo, checkpoint_prefix

WD = 2e-3
ENGINE_BATCH = 8        # images per encode of the engine
# cam_est/train_sdf_cam.py:122-123 CAT_LIST: the test lists are read in the order of the category ids
CAM_CATS = dict(sorted(CATS.items(), key=lambda kv: kv[1]))
VIEW_DATASETS = ("img_arr", "trans_mat", "K", "RT", "obj_rot_mat", "regress_mat")    # create_img_h5 :599-611


def parser():
    """cam_est/train_sdf_cam.py:30-59, plus --view_dir / --sdf_dir / --test_lst_dir and --precision."""
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpu', type=str, default='2')
    ap.add_argument('--category', default="all")
    ap.add_argument('--log_dir', default='checkpoint/sdf_2d_twostream_cam_pcrot_all')
    ap.add_argument('--num_points', type=int, default=1)
    ap.add_argument('--num_sample_points', type=int, default=2048)
    ap.add_argument('--max_epoch', type=int, default=200)
    ap.add_argument('--batch_size', type=int, default=32)
    ap.add_argument('--img_h', type=int, default=137)
    ap.add_argument('--img_w', type=int, default=137)
    ap.add_argument('--verbose_freq', type=int, default=100)
    ap.add_argument('--learning_rate', type=float, default=1e-4)
    ap.add_argument('--momentum', type=float, default=0.9)
    ap.add_argument('--optimizer', default='adam')
    ap.add_argument('--restore_model', default='')
    ap.add_argument('--restore_modelpn', default='')
    ap.add_argument('--restore_modelcnn', default='')
    ap.add_argument('--rotation', action='store_true')
    ap.add_argument('--sample', action='store_false')
    ap.add_argument('--img_feat', action='store_false')
    ap.add_argument('--splitvalid', action='store_true')
    ap.add_argument('--decay_step', type=int, default=200000)
    ap.add_argument('--decay_rate', type=float, default=0.9)
    ap.add_argument('--loss_mode', type=str, default="3D")
    ap.add_argument('--test', action="store_true")
    ap.add_argument('--create', action="store_true")
    ap.add_argument('--cat_limit', type=int, default=168000)
    ap.add_argument('--img_h5_dir', type=str, default=None,
                    help="estimated-camera view files: <img_h5_dir>/<cat>/<obj>/%%02d.npz (required with --create)")
    ap.add_argument('--shift', action="store_true")
    ap.add_argument('--shift_weight', type=float, default=0.5)
    ap.add_argument('--view_dir', required=True, help="view files of create_img_h5: <view_dir>/<cat>/<obj>/%%02d.npz")
    ap.add_argument('--sdf_dir', required=True, help="<sdf_dir>/<cat>/<obj>/ori_sample.npz")
    ap.add_argument('--test_lst_dir', default='')
    ap.add_argument('--precision', default="f16f8", choices=("fp32", "bf16x3", "f16f8"))
    return ap


def regularization(weights) -> np.float32:
    """The camera checkpoint's weight decay: 2e-3 * sum(w^2) / 2 over the VGG-16 kernels (vgg_16/*/weights; slim's conv
    regulariser, cam_est/model_cam.py:75-77), in float64 -> float32.  The pose heads carry no decay
    (tf_util.fully_connected with weight_decay=None) and biases none."""
    total = 0.0
    for name, w in weights.items():
        if name.startswith("vgg_16/") and name.endswith("/weights"):
            a = np.asarray(w, np.float64).reshape(-1)
            total += WD * float(np.dot(a, a)) / 2
    return np.float32(total)


def check_flags(FLAGS):
    if not (FLAGS.test or FLAGS.create):
        raise NotImplementedError("training the camera network is not supported: run with --test and/or --create")
    if FLAGS.shift:
        raise NotImplementedError("--shift is not supported: it adds a shift head and random image shifts")
    if FLAGS.rotation:
        raise NotImplementedError("--rotation is not supported: it reads rendered_dir_v2 for rotated samples the camera "
                                  "network never uses")
    if FLAGS.create and not FLAGS.img_h5_dir:
        raise ValueError("--create needs --img_h5_dir")


def homo_points(pts, M):
    """tf.matmul([pts, 1], M) in float32, k order: pts [B,N,3], M [B,4,3] -> [B,N,3]."""
    p = np.asarray(pts, np.float32)
    M = np.asarray(M, np.float32)[:, None]
    return ((p[..., 0:1] * M[..., 0, :] + p[..., 1:2] * M[..., 1, :]) + p[..., 2:3] * M[..., 2, :]) + M[..., 3, :]


def img_points(pts, trans_mat):
    """model_cam.get_img_points (:111-123): the projections clamped to the reference's [0, 136]."""
    xyz = homo_points(pts, trans_mat)
    return np.minimum(np.float32(136), np.maximum(np.float32(0), xyz[..., :2] / xyz[..., 2:3]))


def batch_metrics(engine, batch_data):
    """(pred_trans_mat, pred_RT, sums [B,5]) of one batch: Engine.cam_metrics over groups of at most 8 images."""
    B = len(batch_data["sdf_pt"])
    outs = []
    for b0 in range(0, B, ENGINE_BATCH):
        sl = slice(b0, min(B, b0 + ENGINE_BATCH))
        outs.append(engine.cam_metrics(batch_data["img"][sl, :, :, :3], batch_data["sdf_pt"][sl],
                                       batch_data["trans_mat"][sl], batch_data["RT"][sl]))
    return tuple(np.concatenate([o[i] for o in outs]) for i in range(3))


def save_overlay(path, img, gt_xy, pred_xy, rng):
    """:530-546: the image with 10 ground-truth (green) and predicted (red) projections.  The 10 points come from rng, a
    generator of this run: in the reference they are np.random.randint draws that race with the loader thread's draws
    on the global generator, so they have no single reference value."""
    import cv2
    saveimg = (img * 255).astype(np.uint8)
    choice = rng.integers(gt_xy.shape[0], size=10)
    for xy, colour in ((gt_xy[choice], (0, 255, 0, 255)), (pred_xy[choice], (0, 0, 255, 255))):
        for j in range(xy.shape[0]):
            cv2.circle(saveimg, (int(xy[j, 0]), int(xy[j, 1])), 3, colour, -1)
    cv2.imwrite(path, saveimg)


def create_img_h5(batch_data, transmat, FLAGS):
    """:568-612: each view file of the batch, copied with trans_mat replaced by the predicted float32 trans_mat."""
    for i in range(len(batch_data["cat_id"])):
        name = '{0:02d}'.format(batch_data['view_id'][i]) + ".npz"
        src = os.path.join(FLAGS.view_dir, batch_data["cat_id"][i], batch_data["obj_nm"][i], name)
        print("src:", src)
        tar_dir = os.path.join(FLAGS.img_h5_dir, batch_data["cat_id"][i], batch_data["obj_nm"][i])
        os.makedirs(tar_dir, exist_ok=True)
        tar = os.path.join(tar_dir, name)
        print("tar:", tar)
        with np.load(src) as f:
            d = {k: f[k] for k in VIEW_DATASETS}
        d["trans_mat"] = np.asarray(transmat[i], np.float32)
        np.savez(tar, **d)
        print("write:", tar)


def eval_one_epoch(engine, dataset, FLAGS, reg, log_string, result_path):
    """:459-565."""
    bs = FLAGS.batch_size
    num_batches = int(len(dataset) / bs)
    print('num_batches', num_batches)
    print('len(VALID_DATASET)', len(dataset))
    pc3d_dist_lst, pc2d_dist_lst = [], []
    losses = {k: 0. for k in CAM_LOSS_KEYS}
    rng = np.random.default_rng(0)
    tic = time.time()
    for batch_idx in range(num_batches):
        batch_data = dataset.fetch()
        pred_tm, pred_rt, sums = batch_metrics(engine, batch_data)
        vals, rot3d_all, rot2d_all = cam_losses(sums, batch_data["sdf_pt"].shape[1], reg, FLAGS.loss_mode)
        for lossname in losses.keys():
            if lossname == "rot2d_dist":
                pc2d_dist_lst.append(vals[lossname])
            elif lossname == "rot3d_dist":
                pc3d_dist_lst.append(vals[lossname])
            losses[lossname] += vals[lossname]
        if batch_idx % FLAGS.verbose_freq == 0:
            log_f_name = os.path.join(result_path, "err_log.txt")
            pts = batch_data["sdf_pt"]
            rot_homopc, pred_rot_homopc = homo_points(pts, batch_data["RT"]), homo_points(pts, pred_rt)
            gt_xy, pred_xy = img_points(pts, batch_data["trans_mat"]), img_points(pts, pred_tm)
            for bid in range(bs):
                stem = '%s_%s_%s' % (batch_data['cat_id'][bid], batch_data['obj_nm'][bid], batch_data['view_id'][bid])
                np.savetxt(os.path.join(result_path, stem + '_gt.xyz'), rot_homopc[bid])
                np.savetxt(os.path.join(result_path, stem + '_pred.xyz'), pred_rot_homopc[bid])
                with open(log_f_name, "a") as logf:
                    logf.write("rot3d_dist: {}, rot2d_dist: {}, filename: {}_comp.png \n"
                               .format(rot3d_all[bid], rot2d_all[bid], stem))
                save_overlay(os.path.join(result_path, stem + '_comp.png'), batch_data['img'][bid], gt_xy[bid],
                             pred_xy[bid], rng)
            outstr = ' -- %03d / %03d -- ' % (batch_idx + 1, num_batches)
            for lossname in losses.keys():
                outstr += '%s: %f, ' % (lossname, losses[lossname] / FLAGS.verbose_freq)
                losses[lossname] = 0
            outstr += 'time: %.02f, ' % (time.time() - tic)
            tic = time.time()
            log_string(outstr)
        if FLAGS.create:
            create_img_h5(batch_data, pred_tm, FLAGS)
    pc2d_dist_lst = np.asarray(pc2d_dist_lst)
    pc3d_dist_lst = np.asarray(pc3d_dist_lst)
    print("avg 2d dist {}, max 2d dist {}, min 2d dist {}".
          format(np.mean(pc2d_dist_lst), np.max(pc2d_dist_lst), np.min(pc2d_dist_lst)))
    print("avg 3d dist {}, max 3d dist {}, min 3d dist {}".
          format(np.mean(pc3d_dist_lst), np.max(pc3d_dist_lst), np.min(pc3d_dist_lst)))
    return pc2d_dist_lst, pc3d_dist_lst


def main(argv=None, weights=None, engine=None):
    """The script.  weights (TF variable name -> array) replaces the checkpoint of --restore_model; engine replaces the
    Engine the script creates (anything with cam_metrics)."""
    FLAGS = parser().parse_args(argv)
    check_flags(FLAGS)
    os.makedirs(FLAGS.log_dir, exist_ok=True)
    result_path = os.path.join(FLAGS.log_dir, 'test_results_' + str(time.time()))
    os.makedirs(result_path, exist_ok=True)
    log_fout = open(os.path.join(FLAGS.log_dir, 'log_train_%s.txt' % str(datetime.now())), 'w')
    log_fout.write(str(FLAGS) + '\n')

    def log_string(out_str):
        log_fout.write(out_str + '\n')
        log_fout.flush()
        print(out_str)

    try:
        log_string('pid: %s' % str(os.getpid()))
        log_string(FLAGS.log_dir)
        listinfo, cats_limit = build_listinfo(FLAGS, CAM_CATS)
        dataset = data.Pt_sdf_img(FLAGS, listinfo=listinfo, cats_limit=cats_limit,
                                  info={"rendered_dir": FLAGS.view_dir, "sdf_dir": FLAGS.sdf_dir})
        if weights is None:
            from .tf_checkpoint import load_checkpoint
            prefix = checkpoint_prefix(FLAGS.restore_model)
            if prefix is None:
                raise SystemExit("no checkpoint in %s" % FLAGS.restore_model)
            weights = load_checkpoint(prefix, prefixes=("vgg_16/", "cameraprediction"))
            print("Model loaded in file: %s" % prefix)
        own = engine is None
        if own:
            from .engine import Engine
            engine = Engine(device=0, precision=FLAGS.precision, max_batch=min(FLAGS.batch_size, ENGINE_BATCH),
                            img_h=FLAGS.img_h, img_w=FLAGS.img_w)
            engine.load_weights_raw(weights)
        try:
            dataset.start()
            try:
                return eval_one_epoch(engine, dataset, FLAGS, regularization(weights), log_string,
                                      result_path)
            finally:
                dataset.shutdown()
        finally:
            if own:
                engine.close()
    finally:
        log_fout.close()


if __name__ == "__main__":
    main()
