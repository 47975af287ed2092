"""Decoder training, the reference's ``train/train_sdf.py`` with the encoder frozen: the epoch loop over the training
views (``<cat>_train.lst``, 24 views per object, ``--cat_limit`` per category) from the loader of test_sdf_acc, one
Engine.train_step per batch (forward of both point streams, get_loss, backward and TF's Adam on the GPU), the
`` -- %03d / %03d -- `` lines every 20 batches and ``avg accuracy`` per epoch, ``log_train.txt``, and ``model.ckpt`` on a
new best average accuracy or ``model_epoch_%03d.ckpt`` every 10 epochs with the ``checkpoint`` state file, so that
create_sdf, test_sdf_acc and ``--restore_model`` find them.

Saved and restored variables follow the reference's Saver (every global variable except ``lr`` and ``batch``): the
encoder and decoder variables, the decoder's Adam slots and the beta powers; the step counter restarts at 0.  The frozen
VGG-16 variables have no Adam slots here.  ``--restore_modelcnn`` loads ``vgg_16/*`` by name and shape; variables no
checkpoint supplies get TF's initialisers (Glorot-uniform kernels, zero biases) from a seeded numpy generator.

Only ``--train_decoder_only`` is implemented: without it the reference trains VGG-16 too, whose backward pass is not
implemented, so the script refuses rather than silently train something else.

    python -m disn_b200.train_sdf --train_decoder_only --img_feat_twostream --view_dir V --sdf_dir S \
        --train_lst_dir L --log_dir checkpoint/SDF_DISN --restore_model checkpoint/SDF_DISN
"""
from __future__ import annotations

import argparse
import os
import time
from datetime import datetime

import numpy as np

from . import data_sdf_h5_queue
from .engine import TRAIN_LOSS_KEYS, train_var_names
from .test_sdf_acc import CATS, checkpoint_prefix

SDF_WEIGHT = 10.
VERBOSE_FREQ = 20
# flags of the reference's parser that select what this script does not implement
REFUSED = ("binary", "img_feat_onestream", "threedcnn", "alpha", "rot", "multi_view", "augcolorfore", "augcolorback")


def parser():
    """train/train_sdf.py:25-66, plus --train_decoder_only, --view_dir / --sdf_dir, --precision and --seed."""
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpu', type=str, default='1')
    ap.add_argument('--category', type=str, default="all")
    ap.add_argument('--log_dir', default='checkpoint')
    ap.add_argument('--num_points', type=int, default=1)
    ap.add_argument("--beta1", type=float, dest="beta1", default=0.5)
    ap.add_argument('--num_sample_points', type=int, default=256)
    ap.add_argument('--max_epoch', type=int, default=200)
    ap.add_argument('--batch_size', type=int, default=32)
    ap.add_argument('--img_h', type=int, default=137)
    ap.add_argument('--img_w', type=int, default=137)
    ap.add_argument('--sdf_res', type=int, default=256)
    ap.add_argument('--num_classes', type=int, default=1024)
    ap.add_argument('--learning_rate', type=float, default=1e-4)
    ap.add_argument('--momentum', type=float, default=0.9)
    ap.add_argument('--optimizer', default='adam')
    ap.add_argument('--restore_model', default='')
    ap.add_argument('--restore_modelpn', default='')
    ap.add_argument('--restore_modelcnn', default='')
    ap.add_argument('--train_lst_dir', default='')
    ap.add_argument('--valid_lst_dir', default='')
    ap.add_argument('--decay_step', type=int, default=200000)
    ap.add_argument('--decay_rate', type=float, default=0.9)
    ap.add_argument('--mask_weight', type=float, default=4.0)
    ap.add_argument('--threedcnn', action='store_true')
    ap.add_argument('--volimp', action='store_true')
    ap.add_argument('--img_feat_onestream', action='store_true')
    ap.add_argument('--img_feat_twostream', action='store_true')
    ap.add_argument('--binary', action='store_true')
    ap.add_argument('--alpha', action='store_true')
    ap.add_argument('--augcolorfore', action='store_true')
    ap.add_argument('--augcolorback', action='store_true')
    ap.add_argument('--backcolorwhite', action='store_true')
    ap.add_argument('--rot', action='store_true')
    ap.add_argument('--tanh', action='store_true')
    ap.add_argument('--cam_est', action='store_true')
    ap.add_argument('--cat_limit', type=int, default=168000)
    ap.add_argument('--multi_view', action='store_true')
    ap.add_argument('--train_decoder_only', action='store_true',
                    help="train the decoder with VGG-16 frozen (the only mode implemented)")
    ap.add_argument('--view_dir', default='', help="view files of create_img_h5: <view_dir>/<cat>/<obj>/%%02d.npz")
    ap.add_argument('--sdf_dir', default='', help="<sdf_dir>/<cat>/<obj>/ori_sample.npz")
    ap.add_argument('--precision', default="fp32", choices=("fp32", "bf16x3", "f16f8"),
                    help="arithmetic of the frozen encoder")
    ap.add_argument('--seed', type=int, default=0, help="numpy seed of the initialisers")
    return ap


def check_flags(FLAGS):
    """Refuse what the script does not implement, before any work."""
    if not FLAGS.train_decoder_only:
        raise NotImplementedError("training VGG-16 needs its backward pass, which is not implemented: pass "
                                  "--train_decoder_only to train the decoder with the encoder frozen")
    if FLAGS.optimizer != 'adam':
        raise NotImplementedError("--optimizer %s is not implemented (only adam)" % FLAGS.optimizer)
    for flag in REFUSED:
        if getattr(FLAGS, flag, False):
            raise NotImplementedError("--%s selects an ablation branch of the reference that is not implemented" % flag)
    if FLAGS.tanh:
        raise NotImplementedError("--tanh is not implemented for training")
    if not FLAGS.img_feat_twostream:
        raise NotImplementedError("only the --img_feat_twostream model (DISN) is implemented")


def get_learning_rate(step, FLAGS):
    """get_learning_rate (train_sdf.py:153-161): exponential_decay(base, step * batch_size, decay_step, decay_rate,
    staircase=True) in float32, clipped below at 1e-6."""
    p = np.floor(np.float32(step * FLAGS.batch_size) / np.float32(FLAGS.decay_step))
    lr = np.float32(FLAGS.learning_rate) * np.power(np.float32(FLAGS.decay_rate), np.float32(p), dtype=np.float32)
    return float(max(np.float32(lr), np.float32(1e-6)))


def initial_weights(num_classes=1024, seed=0):
    """TF's initialisers of every model variable: Glorot-uniform kernels (xavier_initializer for the decoder, slim's
    default for VGG-16) and zero biases, from np.random.default_rng(seed)."""
    from .synth import weight_shapes
    rng = np.random.default_rng(seed)
    out = {}
    for name, shape in weight_shapes(num_classes).items():
        if name.endswith("/biases"):
            out[name] = np.zeros(shape, np.float32)
            continue
        rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
        fan_in, fan_out = shape[-2] * rf, shape[-1] * rf
        lim = np.sqrt(6.0 / (fan_in + fan_out))
        out[name] = rng.uniform(-lim, lim, size=shape).astype(np.float32)
    return out


def build_listinfo(FLAGS, cats=CATS):
    """train_sdf.py:113-129: every object of <cat>_train.lst with its 24 views."""
    cat_ids = list(cats.values()) if FLAGS.category == "all" else [cats[FLAGS.category]]
    cats_limit = {c: 0 for c in cat_ids}
    listinfo = []
    for cat_id in cat_ids:
        with open(os.path.join(FLAGS.train_lst_dir, cat_id + "_train.lst"), 'r') as f:
            for line in f.read().splitlines():
                for render in range(24):
                    cats_limit[cat_id] += 1
                    listinfo.append((cat_id, line.strip(), render))
    return listinfo, cats_limit


def saved_variables(engine, weights):
    """What the reference's Saver writes: the model variables (the encoder's as loaded, the decoder's as trained), the
    decoder's Adam slots and the beta powers."""
    out = {k: np.asarray(v, np.float32) for k, v in weights.items()}
    out.update(engine.train_state())
    return out


def save(log_dir, name, tensors):
    from .tf_checkpoint import save_checkpoint
    prefix = os.path.join(log_dir, name)
    save_checkpoint(prefix, tensors)
    with open(os.path.join(log_dir, "checkpoint"), "w") as f:
        f.write('model_checkpoint_path: "%s"\nall_model_checkpoint_paths: "%s"\n' % (name, name))
    return prefix


def train_one_epoch(engine, dataset, FLAGS, step, log_string):
    """train_sdf.py:349-440 -> (average accuracy, the next step)."""
    num_batches = int(len(dataset) / FLAGS.batch_size)
    print('num_batches', num_batches)
    log_string(str(datetime.now()))
    losses = {k: 0 for k in TRAIN_LOSS_KEYS}
    tic = time.time()
    fetch_time = 0
    accuracy_epoch = 0
    for batch_idx in range(num_batches):
        t0 = time.time()
        batch_data = dataset.fetch()
        fetch_time += time.time() - t0
        lr_val = get_learning_rate(step, FLAGS)
        vals = engine.train_step(batch_data['img'], batch_data['sdf_pt'], batch_data['sdf_pt_rot'], batch_data['trans_mat'],
                                 batch_data['sdf_val'] - 0.003, lr_val)
        step += 1
        for k, v in zip(TRAIN_LOSS_KEYS, vals):
            losses[k] += np.float32(v)
        accuracy_epoch += np.float32(vals[0])
        if (batch_idx + 1) % VERBOSE_FREQ == 0:
            outstr = ' -- %03d / %03d -- ' % (batch_idx + 1, num_batches)
            for lossname in losses.keys():
                outstr += '%s: %f, ' % (lossname, losses[lossname] / float(VERBOSE_FREQ))
                losses[lossname] = 0
            outstr += "lr: %f" % lr_val
            outstr += ' time: %.02f, ' % (time.time() - tic)
            outstr += ', fetch time per b: %.02f, ' % (fetch_time / float(VERBOSE_FREQ))
            tic = time.time()
            fetch_time = 0
            log_string(outstr)
    print("avg accuracy:", accuracy_epoch / num_batches)
    return accuracy_epoch / num_batches, step


def main(argv=None, engine=None, weights=None):
    """The script.  engine replaces the Engine it creates (anything with load_weights, train_begin, train_step,
    train_state and load_train_state); weights (TF variable name -> array) replaces the initialisers, before
    --restore_modelcnn / --restore_model apply."""
    FLAGS = parser().parse_args(argv)
    check_flags(FLAGS)
    from .tf_checkpoint import load_checkpoint
    os.makedirs(FLAGS.log_dir, exist_ok=True)
    log_fout = open(os.path.join(FLAGS.log_dir, 'log_train.txt'), 'w')
    log_fout.write(str(FLAGS) + '\n')

    def log_string(out_str):
        log_fout.write(out_str + '\n')
        log_fout.flush()
        print(out_str)

    log_string('pid: %s' % str(os.getpid()))
    log_string(FLAGS.log_dir)
    weights = initial_weights(FLAGS.num_classes, FLAGS.seed) if weights is None else \
        {k: np.asarray(v, np.float32) for k, v in weights.items()}
    state = {}
    if FLAGS.restore_modelcnn:
        for k, v in load_checkpoint(FLAGS.restore_modelcnn, prefixes=("vgg_16/",)).items():
            if k in weights and np.shape(v) == weights[k].shape:
                weights[k] = np.asarray(v, np.float32)
    prefix = checkpoint_prefix(FLAGS.restore_model) if FLAGS.restore_model else None
    if prefix is not None:
        ckpt = load_checkpoint(prefix, model_variables_only=False)
        for k, v in ckpt.items():
            if k in weights:
                weights[k] = np.asarray(v, np.float32)
            elif k.endswith(("/Adam", "/Adam_1")) or k in ("beta1_power", "beta2_power"):
                state[k] = v
        print("Model loaded in file: %s" % prefix)
    listinfo, cats_limit = build_listinfo(FLAGS)
    info = {'rendered_dir': FLAGS.view_dir, 'sdf_dir': FLAGS.sdf_dir}
    dataset = data_sdf_h5_queue.Pt_sdf_img(FLAGS, listinfo=listinfo, info=info, cats_limit=cats_limit)
    own = engine is None
    if own:
        from .engine import Engine
        engine = Engine(device=0, precision=FLAGS.precision, max_batch=min(FLAGS.batch_size, 8), img_h=FLAGS.img_h,
                        img_w=FLAGS.img_w, num_classes=FLAGS.num_classes)
    try:
        engine.load_weights(weights)
        engine.train_begin(beta1=FLAGS.beta1, mask_weight=FLAGS.mask_weight, sdf_weight=SDF_WEIGHT)
        names = set(train_var_names())
        engine.load_train_state({k: v for k, v in state.items()
                                 if k in ("beta1_power", "beta2_power") or k.rsplit("/", 1)[0] in names})
        dataset.start()
        best_acc, step = 0, 0
        try:
            for epoch in range(FLAGS.max_epoch):
                log_string('**** EPOCH %03d ****' % epoch)
                avg_accuracy, step = train_one_epoch(engine, dataset, FLAGS, step, log_string)
                if avg_accuracy > best_acc:
                    best_acc = avg_accuracy
                    path = save(FLAGS.log_dir, "model.ckpt", saved_variables(engine, weights))
                    log_string("best Model saved in file: %s" % path)
                elif epoch % 10 == 0:
                    path = save(FLAGS.log_dir, "model_epoch_%03d.ckpt" % epoch, saved_variables(engine, weights))
                    log_string("Model saved in file: %s" % path)
        finally:
            dataset.shutdown()
    finally:
        log_fout.close()
        if own:
            engine.close()
    return best_acc


if __name__ == "__main__":
    main()
