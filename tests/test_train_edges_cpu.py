"""CPU tests of the float64 training oracle (oracle/train_oracle.py) at non-default loss weights and weight decay, at the
loss's tie points and through a dead ReLU layer, against an autograd twin.

The twin restates the decoder forward and get_loss in torch.float64 and takes the gradient of
sdf_loss + wd * sum l2_loss(kernels) with autograd; it shares no code with the oracle's hand-written backward.  Central
differences cannot see ties (|.| at 0, a ReLU at 0, the weight mask at 0.01); autograd follows TF's conventions there:
d|x|/dx = 0 at 0, and a ReLU passes the gradient where its output is > 0.
"""
import numpy as np
import pytest
import torch

from disn_b200 import synth
from oracle import train_oracle as orc

REL = 1e-12
NC = 16


def _problem(seed=0, B=2, N=8, exact=False):
    """Decoder weights, encoder outputs, points and float32-valued ground truth.  exact=True rounds every weight and
    input to a multiple of 2^-6: each layer's products and sums are then exact in float64 (the forward's values are
    multiples of 2^-42 far below 2^11), so any two restatements give the same pred, bit for bit, and a tie written
    from one pred is a tie in the other."""
    rng = np.random.default_rng(seed)
    W = {k: v for k, v in synth.make_weights(seed=seed, num_classes=NC).items() if k.startswith("sdfprediction")}
    emb = rng.normal(0, 1, (B, NC))
    feat = rng.normal(0, 1, (B, N, 1472))
    pts = rng.uniform(-0.5, 0.5, (B, N, 3))
    gt = rng.uniform(-0.1, 0.1, (B, N)).astype(np.float32).astype(np.float64)
    if exact:
        q = lambda a: np.round(np.asarray(a, np.float64) * 64) / 64
        W = {k: q(v) for k, v in W.items()}
        emb, feat, pts = q(emb), q(feat), q(pts)
    return W, emb, feat, pts, gt


def _twin(W, emb, feat, pts, gt, sdf_weight, mask_weight, wd):
    """-> (grads {name: float64 array of the variable's shape}, losses dict) from torch.float64 autograd."""
    B, N = pts.shape[:2]
    T = {n: torch.tensor(np.asarray(W[n], np.float64), requires_grad=True) for n in orc.var_names()}
    x = torch.tensor(pts.reshape(B * N, 3))
    extra = (torch.tensor(np.repeat(emb, N, axis=0)), torch.tensor(feat.reshape(B * N, -1)))
    pred = 0
    for si, scope in enumerate(orc.SCOPES):
        h = x
        for li, layer in enumerate(orc.LAYERS):
            w = T["%s/%s/weights" % (scope, layer)]
            b = T["%s/%s/biases" % (scope, layer)]
            if li == 3:
                h = torch.cat([h, extra[si]], dim=1)
            z = h @ w.reshape(-1, w.shape[-1]) + b
            h = z[:, 0] if li == 5 else torch.relu(z)
        pred = pred + h
    g = torch.tensor(gt.reshape(-1))
    g32 = torch.tensor(np.asarray(gt, np.float32).reshape(-1))
    thr = torch.tensor(0.01, dtype=torch.float32)
    mask = (g32 <= thr).double() * mask_weight + (g32 > thr).double()
    sdf_loss = 1000.0 * torch.mean(torch.abs(g * sdf_weight - pred) * mask)
    reg = sum(wd * torch.sum(T[n] ** 2) / 2 for n in orc.var_names() if n.endswith("/weights"))
    (sdf_loss + reg).backward()
    losses = dict(pred=pred.detach().numpy(), sdf_loss=float(sdf_loss.detach()), reg=float(reg.detach()),
                  real=float(torch.mean(torch.abs(g - pred.detach() / sdf_weight))),
                  acc=float(torch.mean(((g > 0) == (pred.detach() > 0)).double())))
    return {n: T[n].grad.numpy() for n in orc.var_names()}, losses


def _compare(W, emb, feat, pts, gt, sdf_weight=orc.SDF_WEIGHT, mask_weight=orc.MASK_WEIGHT, wd=orc.WD):
    want, tw = _twin(W, emb, feat, pts, gt, sdf_weight, mask_weight, wd)
    pred, got = orc.step_grads(W, emb, feat, pts, pts, gt, wd=wd, sdf_weight=sdf_weight, mask_weight=mask_weight)
    assert np.allclose(pred, tw["pred"], rtol=REL, atol=0)
    for n in orc.var_names():
        a, b = np.asarray(got[n]).reshape(-1), want[n].reshape(-1)
        scale = np.abs(b).max()
        assert np.abs(a - b).max() <= REL * scale, (n, np.abs(a - b).max(), scale)
    # the five reported values, rounded to float32 as TF reports them
    rep = orc.reported_losses(pred, gt, W, wd, sdf_weight, mask_weight)
    twin = [tw["acc"], tw["real"], tw["sdf_loss"], tw["reg"], np.float32(tw["sdf_loss"]) + np.float32(tw["reg"])]
    assert rep[0] == np.float32(twin[0])
    for k in range(1, 5):
        assert abs(rep[k] - np.float32(twin[k])) <= np.spacing(np.float32(twin[k])), (k, rep[k], twin[k])
    return pred, got


@pytest.mark.parametrize("sdf_weight,mask_weight,wd", [(25.0, 0.25, 1e-3), (8.0, 1.0, 0.0), (10.0, 4.0, 1e-5)])
def test_oracle_flags_match_autograd(sdf_weight, mask_weight, wd):
    W, emb, feat, pts, gt = _problem(seed=1)
    _compare(W, emb, feat, pts, gt, sdf_weight, mask_weight, wd)


def _ties(pred, gt, sw):
    """gt with exact ties: g = pred/sw at points 0, 1 and 8 (d = 0 exactly, sw a power of two), g = 0 and g = -0.0 at
    2 and 3, and g = float32(0.01) and its float32 neighbours below and above at 4, 5 and 6."""
    g = gt.reshape(-1).copy()
    p = np.asarray(pred, np.float64).reshape(-1)
    t = np.float32(0.01)
    for i in (0, 1, 8):
        g[i] = p[i] / sw
        assert g[i] * sw - p[i] == 0.0
    g[2], g[3] = 0.0, -0.0
    g[4], g[5], g[6] = t, np.nextafter(t, np.float32(0)), np.nextafter(t, np.float32(1))
    assert np.signbit(g[3])
    return g.reshape(gt.shape)


@pytest.mark.parametrize("sw", [8.0, 16.0])
def test_oracle_ties_match_autograd(sw):
    W, emb, feat, pts, gt = _problem(seed=2, exact=True)
    pred, _ = orc.forward(W, emb, feat, pts)
    gt = _ties(pred, gt, sw)
    assert np.array_equal(pred, _twin(W, emb, feat, pts, gt, sw, 0.25, 1e-4)[1]["pred"])
    _compare(W, emb, feat, pts, gt, sdf_weight=sw, mask_weight=0.25, wd=1e-4)
    # the tie points contribute nothing: dpred is 0 where d = 0
    dpred = orc.loss_terms(pred, gt, sdf_weight=sw, mask_weight=0.25)[3]
    assert dpred[0] == 0 and dpred[1] == 0 and dpred[8] == 0
    w = orc.weight_mask(gt, 0.25)
    assert list(w[2:7]) == [0.25, 0.25, 0.25, 0.25, 1.0]      # 0, -0, 0.01f, below: masked; above: not


@pytest.mark.parametrize("scope", orc.SCOPES)
@pytest.mark.parametrize("layer", ["fold2/conv2", "fold1/conv1"])
def test_oracle_dead_relu_layer_matches_autograd(scope, layer):
    W, emb, feat, pts, gt = _problem(seed=3)
    W = dict(W)
    W["%s/%s/biases" % (scope, layer)] = np.full_like(W["%s/%s/biases" % (scope, layer)], -1e3)
    wd = 1e-3
    _, grads = _compare(W, emb, feat, pts, gt, sdf_weight=10.0, mask_weight=4.0, wd=wd)
    # up to the dead layer nothing but the decay reaches a weight and no bias gradient survives; the layer after it
    # reads only zeros, so its weight gradient is the decay alone too
    li = orc.LAYERS.index(layer)
    for l in orc.LAYERS[:li + 2]:
        n = "%s/%s/" % (scope, l)
        assert np.array_equal(grads[n + "weights"], wd * np.asarray(W[n + "weights"], np.float64)), n
        if l != orc.LAYERS[li + 1]:
            assert not np.any(grads[n + "biases"]), n


def test_weight_mask_threshold_is_float32():
    t = np.float32(0.01)
    g = np.array([t, np.nextafter(t, np.float32(1)), np.nextafter(t, np.float32(0)), 0.0, -0.0], np.float32)
    assert list(orc.weight_mask(g, 4.0)) == [4.0, 1.0, 4.0, 4.0, 4.0]
    # for float32 inputs the float32 comparison is the float64 one
    assert np.array_equal(g <= np.float32(0.01), g.astype(np.float64) <= 0.01)
