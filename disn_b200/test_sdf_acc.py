"""Checkpoint score on the test set, the reference's ``test/test_sdf_acc.py``: sign accuracy and weighted L1 of the
predicted field at the ground-truth samples of every (object, view) of the test lists, one line per batch and a
``Summary:`` line, also written to ``<log_dir>/log_test.txt``.

The metrics come from Engine.sdf_metrics (disn_sdf_metrics): the point kernel and one reduction kernel per batch.  The
engine encodes at most 8 images at a time, so a larger batch is scored in groups of 8 whose per-image sums are added.
``regularization`` is a constant of the checkpoint: 1e-5 * sum(w^2) / 2 over the conv kernels of VGG-16 (fc6-8
included; slim.l2_regularizer, models/model_normalization.py:75) and of both sdfprediction heads
(tf_util._variable_with_weight_decay), biases excluded, in float64.  ``--view_dir`` / ``--sdf_dir`` replace the
reference's hard-coded dataset paths.

    python -m disn_b200.test_sdf_acc --view_dir V --sdf_dir S --test_lst_dir L --log_dir checkpoint/SDF_DISN
"""
from __future__ import annotations

import argparse
import os
from datetime import datetime

import numpy as np

from . import data_sdf_h5_queue
from .engine import batch_losses

SDF_WEIGHT = 10.
WD = 1e-5
ENGINE_BATCH = 8        # images per encode of the engine
# preprocessing/info.json "cats", in its order (the order the test lists are read in)
CATS = {"watercraft": "04530566", "rifle": "04090263", "display": "03211117", "lamp": "03636649",
        "speaker": "03691459", "cabinet": "02933112", "chair": "03001627", "bench": "02828884", "car": "02958343",
        "airplane": "02691156", "sofa": "04256520", "table": "04379243", "phone": "04401088"}
LOSS_KEYS = ("accuracy", "sdf_loss_realvalue", "sdf_loss", "regularization", "overall_loss")


def parser():
    """test/test_sdf_acc.py:17-49, plus --view_dir / --sdf_dir and --precision."""
    ap = argparse.ArgumentParser()
    ap.add_argument('--max_epoch', type=int, default=1)
    ap.add_argument('--img_h', type=int, default=137)
    ap.add_argument('--img_w', type=int, default=137)
    ap.add_argument('--learning_rate', type=float, default=1e-4)
    ap.add_argument('--decay_step', type=int, default=200000)
    ap.add_argument('--decay_rate', type=float, default=0.9)
    ap.add_argument('--num_classes', type=int, default=1024)
    ap.add_argument('--num_points', type=int, default=1)
    ap.add_argument('--mask_weight', type=float, default=4.0)
    ap.add_argument('--alpha', action='store_true')
    ap.add_argument('--rot', action='store_true')
    ap.add_argument('--tanh', action='store_true')
    ap.add_argument('--cat_limit', type=int, default=168000)
    ap.add_argument('--gpu', type=str, default='0')
    ap.add_argument('--batch_size', type=int, default=1)
    ap.add_argument('--sdf_res', type=int, default=64)
    ap.add_argument('--log_dir', default='checkpoint/exp_200')
    ap.add_argument('--test_lst_dir', default='')
    ap.add_argument('--num_sample_points', type=int, default=2048)
    ap.add_argument('--threedcnn', action='store_true')
    ap.add_argument('--img_feat', action='store_true')
    ap.add_argument('--img_feat_far', action='store_true')
    ap.add_argument('--img_feat_twostream', action='store_true')
    ap.add_argument('--category', default="all")
    ap.add_argument('--binary', action='store_true')
    ap.add_argument('--create_obj', action='store_true')
    ap.add_argument('--store', action='store_true')
    ap.add_argument('--multi_view', action='store_true')
    ap.add_argument('--cam_est', action='store_true')
    ap.add_argument('--backcolorwhite', action='store_true')
    ap.add_argument('--view_dir', required=True, help="view files of create_img_h5: <view_dir>/<cat>/<obj>/%%02d.npz")
    ap.add_argument('--sdf_dir', required=True, help="<sdf_dir>/<cat>/<obj>/ori_sample.npz")
    ap.add_argument('--precision', default="f16f8", choices=("fp32", "bf16x3", "f16f8"))
    return ap


def build_listinfo(FLAGS, cats=CATS, view_lists=None):
    """test/test_sdf_acc.py:76-99 (view_lists None: every object's 24 views) or test/create_sdf.py:106-149 (view_lists =
    a function returning the views of one object) -> (listinfo [(cat_id, obj, view)], cats_limit)."""
    cat_ids = list(cats.values()) if FLAGS.category == "all" else [cats[FLAGS.category]]
    cats_limit = {c: 0 for c in cat_ids}
    listinfo = []
    for cat_id in cat_ids:
        with open(os.path.join(FLAGS.test_lst_dir, cat_id + "_test.lst"), 'r') as f:
            for line in f.read().splitlines():
                for render in (range(24) if view_lists is None else view_lists()):
                    cats_limit[cat_id] += 1
                    listinfo.append((cat_id, line.strip(), render))
    return listinfo, cats_limit


def regularization(weights) -> np.float32:
    """1e-5 * sum(w^2) / 2 over every conv kernel (vgg_16/* and sdfprediction*/ weights), float64 -> float32."""
    total = 0.0
    for name, w in weights.items():
        if name.endswith("/weights") and (name.startswith("vgg_16/") or name.startswith("sdfprediction")):
            a = np.asarray(w, np.float64)
            total += WD * float(np.dot(a.reshape(-1), a.reshape(-1))) / 2
    return np.float32(total)


def batch_metrics(engine, batch_data, mask_weight):
    """(accuracy, sdf_loss_realvalue, sdf_loss) of one batch: Engine.sdf_metrics over groups of at most 8 images."""
    B, N = batch_data["sdf_pt"].shape[:2]
    sums = []
    for b0 in range(0, B, ENGINE_BATCH):
        sl = slice(b0, min(B, b0 + ENGINE_BATCH))
        engine.encode(batch_data["img"][sl])
        sums.append(engine.sdf_metrics(batch_data["sdf_pt"][sl], batch_data["trans_mat"][sl], batch_data["sdf_val"][sl],
                                       iso_offset=0.003, sdf_weight=SDF_WEIGHT, mask_weight=mask_weight))
    count, wsum, rsum = (np.concatenate([s[i] for s in sums]) for i in range(3))
    return batch_losses(count, wsum, rsum, B * N)


def test_one_epoch(engine, dataset, FLAGS, reg, log_string):
    """test/test_sdf_acc.py:180-217: per-batch and summary lines, in the reference's key order and format."""
    num_batches = int(len(dataset)) // FLAGS.batch_size
    print()
    print('num_batches', num_batches)
    log_string(str(datetime.now()))
    losses = {k: 0 for k in LOSS_KEYS}
    for batch_idx in range(num_batches):
        batch_data = dataset.fetch()
        acc, real, sdf_loss = batch_metrics(engine, batch_data, FLAGS.mask_weight)
        vals = {"accuracy": acc, "sdf_loss_realvalue": real, "sdf_loss": sdf_loss, "regularization": reg,
                "overall_loss": np.float32(sdf_loss + reg)}
        outstr = ' -- %03d / %03d -- ' % (batch_idx + 1, num_batches)
        for lossname in losses.keys():
            losses[lossname] += vals[lossname]
            outstr += '%s: %f, ' % (lossname, vals[lossname])
        log_string(outstr)
    outstr = "Summary: "
    for lossname in losses.keys():
        outstr += '%s: %f, ' % (lossname, losses[lossname] / num_batches)
    log_string(outstr)
    return {k: v / num_batches for k, v in losses.items()}


def checkpoint_prefix(log_dir):
    """tf.train.get_checkpoint_state(log_dir): the model_checkpoint_path of <log_dir>/checkpoint, or None."""
    state = os.path.join(log_dir, "checkpoint")
    if not os.path.exists(state):
        return None
    with open(state) as f:
        for line in f:
            if line.startswith("model_checkpoint_path:"):
                return os.path.join(log_dir, os.path.basename(line.split(":", 1)[1].strip().strip('"')))
    return None


def main(argv=None, weights=None, engine=None):
    """The script.  weights (TF variable name -> array) replaces the checkpoint of --log_dir; engine replaces the
    Engine the script creates (anything with encode and sdf_metrics)."""
    FLAGS = parser().parse_args(argv)
    print('pid: %s' % str(os.getpid()))
    print(FLAGS)
    data_sdf_h5_queue.check_flags(FLAGS)
    if not FLAGS.img_feat_twostream:
        raise NotImplementedError("only the --img_feat_twostream model (DISN) is implemented")
    os.makedirs(FLAGS.log_dir, exist_ok=True)
    os.makedirs(os.path.join(FLAGS.log_dir, 'test_results_allpts'), exist_ok=True)
    log_fout = open(os.path.join(FLAGS.log_dir, 'log_test.txt'), 'w')
    log_fout.write(str(FLAGS) + '\n')

    def log_string(out_str):
        log_fout.write(out_str + '\n')
        log_fout.flush()
        print(out_str)

    listinfo, cats_limit = build_listinfo(FLAGS)
    info = {'rendered_dir': FLAGS.view_dir, 'sdf_dir': FLAGS.sdf_dir}
    dataset = data_sdf_h5_queue.Pt_sdf_img(FLAGS, listinfo=listinfo, info=info, cats_limit=cats_limit)
    print(info)
    log_string(FLAGS.log_dir)
    if weights is None:
        from .tf_checkpoint import load_checkpoint
        prefix = checkpoint_prefix(FLAGS.log_dir)
        if prefix is None:
            raise SystemExit("no checkpoint in %s" % FLAGS.log_dir)
        weights = load_checkpoint(prefix, prefixes=("vgg_16/", "sdfprediction"))
        print("Model loaded in file: %s" % prefix)
    own = engine is None
    if own:
        from .engine import Engine
        engine = Engine(device=0, precision=FLAGS.precision, max_batch=min(FLAGS.batch_size, ENGINE_BATCH),
                        tanh=FLAGS.tanh, img_h=FLAGS.img_h, img_w=FLAGS.img_w, num_classes=FLAGS.num_classes)
        engine.load_weights(weights)
    try:
        dataset.start()
        try:
            return test_one_epoch(engine, dataset, FLAGS, regularization(weights), log_string)
        finally:
            dataset.shutdown()
    finally:
        log_fout.close()
        if own:
            engine.close()


if __name__ == "__main__":
    main()
