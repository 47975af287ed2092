"""TEST INFRASTRUCTURE ONLY -- float64 CPU restatement of one decoder training step of the reference
(train/train_sdf.py with --img_feat_twostream, bn=False; models/model_normalization.py:169-206,254-299,
models/sdfnet.py:69-92,171-190, utils/tf_util.py:23-47): both point streams given the encoder's outputs, get_loss, the
gradient of overall_loss by hand with TF's conventions (d|x|/dx = sign(x), ReLU passes where its output is > 0, the mean
divides by B*N), and tf.train.AdamOptimizer's update.

`masks` / `signs` let a test take the branch decisions (ReLU masks, |.| signs, the 0.01 weight mask) from the device's
forward, so that what is compared is arithmetic, not tie-breaking; `absolute=True` runs the same passes on |.| of every
operand, the magnitude sums an error bound scales with.
"""
from __future__ import annotations

import numpy as np

SCOPES = ("sdfprediction", "sdfprediction_imgfeat")
LAYERS = ("fold1/conv1", "fold1/conv2", "fold1/conv3", "fold2/conv1", "fold2/conv2", "fold2/conv5")
COUT = (64, 256, 512, 512, 256, 1)
WD = 1e-5
SDF_WEIGHT = 10.0
MASK_WEIGHT = 4.0


def var_names():
    """The 24 decoder variables, in the library's order (stream, layer, weights before biases)."""
    return ["%s/%s/%s" % (s, l, k) for s in SCOPES for l in LAYERS for k in ("weights", "biases")]


def _w(W, s, l):
    return np.asarray(W["%s/%s/weights" % (s, l)], np.float64).reshape(-1, COUT[LAYERS.index(l)])


def _b(W, s, l):
    return np.asarray(W["%s/%s/biases" % (s, l)], np.float64).reshape(-1)


def forward(W, emb, feat, pts_rot, masks=None, absolute=False):
    """pred [B*N] and the cache backward needs.  emb [B,nc], feat [B,N,1472] (point_img_feat), pts_rot [B,N,3].
    masks: None (ReLU decides) or masks[stream][layer] boolean [B*N, width] for layers 0..4."""
    f = np.abs if absolute else (lambda a: a)
    B, N = np.asarray(pts_rot).shape[:2]
    x = f(np.asarray(pts_rot, np.float64).reshape(B * N, 3))
    e = f(np.asarray(emb, np.float64).reshape(B, -1))
    ft = f(np.asarray(feat, np.float64).reshape(B * N, -1))
    cache = {"B": B, "N": N, "xin": [[None] * 6 for _ in SCOPES], "mask": [[None] * 5 for _ in SCOPES]}
    pred = 0.0
    for si, s in enumerate(SCOPES):
        h = x
        for li, l in enumerate(LAYERS):
            if li == 3:
                extra = np.repeat(e, N, axis=0) if si == 0 else ft
                h = np.concatenate([h, extra], axis=1)
            cache["xin"][si][li] = h
            z = h @ f(_w(W, s, l)) + f(_b(W, s, l))
            if li == 5:
                pred = pred + z[:, 0]
                break
            m = (z > 0) if masks is None else np.asarray(masks[si][li], bool)
            cache["mask"][si][li] = m
            h = z * m
    return pred, cache


def loss_terms(pred, gt, signs=None, weights=None, sdf_weight=SDF_WEIGHT, mask_weight=MASK_WEIGHT):
    """get_loss's sdf terms in float64: (sdf_loss, sdf_loss_realvalue, accuracy, dpred).  gt = the fed ground truth."""
    p = np.asarray(pred, np.float64).reshape(-1)
    g = np.asarray(gt, np.float64).reshape(-1)
    d = g * sdf_weight - p
    w = np.where(g <= 0.01, mask_weight, 1.0) if weights is None else np.asarray(weights, np.float64).reshape(-1)
    sg = np.sign(d) if signs is None else np.asarray(signs, np.float64).reshape(-1)
    P = p.size
    sdf_loss = 1000.0 * np.sum(np.abs(d) * w) / P
    real = np.sum(np.abs(g - p / sdf_weight)) / P
    acc = np.mean((g > 0) == (p > 0))
    dpred = -1000.0 / P * w * sg
    return sdf_loss, real, acc, dpred


def backward(W, cache, dpred, wd=WD, absolute=False):
    """Gradients of overall_loss (the sdf loss through dpred, plus wd * W for every kernel) -> {name: array of the
    variable's stored shape}."""
    f = np.abs if absolute else (lambda a: a)
    grads = {}
    for si, s in enumerate(SCOPES):
        dz = f(np.asarray(dpred, np.float64)).reshape(-1, 1)
        for li in range(5, -1, -1):
            l = LAYERS[li]
            Wl = f(_w(W, s, l))
            xin = cache["xin"][si][li]
            dW = xin.T @ dz + wd * Wl
            name = "%s/%s/" % (s, l)
            grads[name + "weights"] = dW.reshape(np.shape(W[name + "weights"]))
            grads[name + "biases"] = dz.sum(axis=0).reshape(np.shape(W[name + "biases"]))
            if li == 0:
                break
            width = COUT[li - 1]
            dz = (dz @ Wl[:width].T) * cache["mask"][si][li - 1]
    return grads


def step_grads(W, emb, feat, pts, pts_rot, gt, masks=None, signs=None, weights=None, absolute=False, wd=WD):
    """One step's (pred, grads) in float64; absolute=True gives the magnitude sums of the same passes."""
    pred, cache = forward(W, emb, feat, pts_rot, masks=masks, absolute=absolute)
    if absolute:
        g = np.asarray(gt, np.float64).reshape(-1)
        w = np.where(g <= 0.01, MASK_WEIGHT, 1.0) if weights is None else np.asarray(weights, np.float64).reshape(-1)
        dpred = 1000.0 / g.size * w
    else:
        dpred = loss_terms(pred, gt, signs, weights)[3]
    return pred, backward(W, cache, dpred, wd=wd, absolute=absolute)


def regularization(weights, wd=WD):
    """wd * l2_loss over every kernel (vgg_16/* through slim.l2_regularizer, sdfprediction*/ through the 'regularizer'
    collection), biases excluded, float64."""
    total = 0.0
    for name, w in weights.items():
        if name.endswith("/weights") and (name.startswith("vgg_16/") or name.startswith("sdfprediction")):
            a = np.asarray(w, np.float64).reshape(-1)
            total += wd * float(a @ a) / 2
    return total


def reported_losses(pred, gt, weights, wd=WD):
    """The five values train_sdf.py reports for a step, rounded to float32 as TF reports them: accuracy,
    sdf_loss_realvalue, sdf_loss, regularization, overall_loss."""
    sdf_loss, real, acc, _ = loss_terms(pred, gt)
    reg = regularization(weights, wd)
    loss32 = np.float32(sdf_loss)
    return np.array([np.float32(acc), np.float32(real), loss32, np.float32(reg), np.float32(loss32 + np.float32(reg))],
                    np.float64)


def adam(w, g, m, v, lr, beta1_power, beta2_power, beta1=0.5, beta2=0.999, eps=1e-8, dtype=np.float64):
    """tf.train.AdamOptimizer's ApplyAdam: lr_t = lr sqrt(1 - beta2^t) / (1 - beta1^t); m += (g - m)(1 - beta1);
    v += (g^2 - v)(1 - beta2); w -= (m lr_t) / (sqrt(v) + eps); then beta powers *= betas.  dtype=np.float32 rounds every
    operation to float32 in that order.  -> (w, m, v, beta1_power, beta2_power)."""
    t = dtype
    w, g, m, v = (np.asarray(a, t) for a in (w, g, m, v))
    lr, b1p, b2p, b1, b2, e = (t(x) for x in (lr, beta1_power, beta2_power, beta1, beta2, eps))
    one = t(1)
    alpha = lr * np.sqrt(one - b2p) / (one - b1p)
    m = m + (g - m) * (one - b1)
    v = v + (g * g - v) * (one - b2)
    w = w - (m * alpha) / (np.sqrt(v) + e)
    return w, m, v, b1p * b1, b2p * b2


def learning_rate(step, base_lr, batch_size, decay_step, decay_rate):
    """get_learning_rate: tf.train.exponential_decay(base, step * batch_size, decay_step, decay_rate, staircase=True),
    clipped below at 1e-6."""
    return max(base_lr * decay_rate ** ((step * batch_size) // decay_step), 1e-6)
