"""GPU tests of decoder training at the edges test_gpu_train.py does not reach: unaligned shapes (padded point axis,
uneven and empty column-sum chunks, a last encode group of one image), non-default loss weights, weight decay and Adam
betas, exact ties at the loss's three comparisons, dead ReLU layers checked bit for bit, a context reused across
shapes, a six-step Adam chain checked bit for bit, and the refusals.

Every gradient is held to the bound of test_gpu_train.py: |g_dev - g_64| <= C_GRAD * 2^-24 * g_abs, with g_64 the float64
oracle's gradient under the device's ReLU masks and |.| signs and g_abs the same passes on |.| of every operand.  Each
check prints its worst fraction of the bound.
"""
import ctypes as C
import re

import numpy as np
import pytest

from disn_b200 import _lib, synth
from disn_b200._lib import DisnError
from disn_b200.engine import Engine, train_var_names
from oracle import train_oracle as orc

pytestmark = pytest.mark.gpu

C_GRAD = 4096.0
U = 2.0 ** -24
LR = 1e-4
WIDTHS = (64, 256, 512, 512, 256)


def _problem(B, N, seed=0, outside=False):
    """imgs, pts, pts_rot, tm and the fed ground truth (a sphere's field - 0.003).  Odd seeds rotate the decoder's
    points apart from the projected ones.  outside=True puts every other point in [-1.5, 1.5]^3 beyond the unit box:
    their projections are clamped at the map's edge."""
    rng = np.random.default_rng(seed)
    imgs = synth.synthetic_images(B, seed=100 + seed)
    tm = synth.synthetic_trans_mats(B, seed=200 + seed).astype(np.float32)
    pts = rng.uniform(-0.5, 0.5, size=(B, N, 3)).astype(np.float32)
    if outside:
        far = rng.uniform(0.6, 1.5, size=(B, N, 3)) * rng.choice([-1.0, 1.0], size=(B, N, 3))
        pts[:, ::2] = far[:, ::2].astype(np.float32)
    pts_rot = pts if seed % 2 == 0 else rng.uniform(-0.5, 0.5, size=(B, N, 3)).astype(np.float32)
    r = np.linalg.norm(pts_rot.astype(np.float64), axis=2)
    gt = ((r - 0.3) - 0.003).astype(np.float32)
    return imgs, pts, pts_rot, tm, gt


def _engine(W, max_batch=8, **train):
    eng = Engine(device=0, precision="fp32", max_batch=max_batch)
    eng.load_weights(W)
    eng.train_begin(**train)
    return eng


def _device_inputs(eng, imgs, pts, tm):
    """The frozen encoder's embedding and point features, encoded in groups of 8 as a step does."""
    embs, feats = [], []
    for b0 in range(0, len(imgs), 8):
        sl = slice(b0, b0 + 8)
        eng.encode(imgs[sl])
        embs.append(eng.get_encoded(0))
        feats.append(eng.point_img_feat(pts[sl], tm[sl])[0][:, :, 0, :])
    return np.concatenate(embs), np.concatenate(feats)


def _debug_grads(eng, imgs, pts, pts_rot, tm, gt):
    """One step's gradients without the update (the diagnostic library) -> (grads by name, pred, the ReLU masks of
    both streams' layers 1-5, the five reported values)."""
    lib = _lib.load_test()
    B, N, _ = pts.shape
    names = train_var_names()
    sizes = [eng._numel(n) for n in names]
    grads = np.empty(sum(sizes), np.float32)
    pred = np.empty(B * N, np.float32)
    acts = np.empty(2 * B * N * sum(WIDTHS), np.float32)
    losses = np.empty(5, np.float64)
    a = [np.ascontiguousarray(x, np.float32) for x in (imgs, pts, pts_rot, tm, gt)]
    ptr = lambda x: x.ctypes.data_as(C.c_void_p)
    _lib.check(lib.disn_debug_train_grads(eng._h, ptr(a[0]), imgs.shape[1], imgs.shape[2], 3, ptr(a[1]), ptr(a[2]),
                                          ptr(a[3]), ptr(a[4]), B, N, ptr(grads), ptr(pred), ptr(acts), ptr(losses)))
    out, o = {}, 0
    for n, s in zip(names, sizes):
        out[n] = grads[o:o + s]
        o += s
    masks, o = [[], []], 0
    for si in range(2):
        for w in WIDTHS:
            masks[si].append(acts[o:o + B * N * w].reshape(B * N, w) > 0)
            o += B * N * w
    return out, pred, masks, losses


def _check(label, W, emb, feat, pts_rot, gt, g_dev, pred, masks, losses, sdf_weight=10.0, mask_weight=4.0, wd=1e-5):
    """Every gradient within the bound of the oracle under the device's branch decisions, and the five reported values
    within 2 float32 ulp.  The |.| signs are those of the float32 d = gt * sw - pred the device forms: 0 at a tie."""
    d = gt.reshape(-1) * np.float32(sdf_weight) - pred
    signs = np.sign(d.astype(np.float64))
    kw = dict(masks=masks, wd=wd, sdf_weight=sdf_weight, mask_weight=mask_weight)
    _, g64 = orc.step_grads(W, emb, feat, None, pts_rot, gt, signs=signs, **kw)
    _, gabs = orc.step_grads(W, emb, feat, None, pts_rot, gt, absolute=True, **kw)
    worst = 0.0
    for name in orc.var_names():
        err = np.abs(g_dev[name].astype(np.float64) - g64[name].reshape(-1))
        bound = C_GRAD * U * gabs[name].reshape(-1) + 1e-30
        frac = float(np.max(err / bound))
        worst = max(worst, frac)
        assert frac <= 1.0, (label, name, frac)
    print("%s: worst gradient error = %.3g of the bound (C = %g)" % (label, worst, C_GRAD))
    want = orc.reported_losses(pred, gt, W, wd, sdf_weight, mask_weight)
    for k in range(5):
        assert abs(losses[k] - want[k]) <= 2 * np.spacing(np.float32(want[k])), (label, k, losses[k], want[k])


def _bits(state):
    return {k: np.asarray(v, np.float32).view(np.uint32).copy() for k, v in state.items()}


def _same_bits(a, b, label):
    assert set(a) == set(b), label
    for k in a:
        assert np.array_equal(a[k], b[k]), (label, k)


# ---------------------------------------------------------------------------------------------------------------------
# a. shapes: B*N not a multiple of 128 (padding rows), N not a multiple of 16 or below 16 (uneven and empty column-sum
# chunks), a last encode group of one image (B = 9, 17), the driver's default batch and the reference shape minus one
@pytest.mark.parametrize("B,N,outside", [(1, 1, False), (1, 7, False), (3, 77, False), (9, 333, False),
                                         (17, 129, False), (32, 256, False), (20, 2047, False), (5, 100, True)])
def test_gradients_at_unaligned_shapes(B, N, outside):
    seed = B + N
    W = synth.make_weights(seed=seed % 5)
    imgs, pts, pts_rot, tm, gt = _problem(B, N, seed, outside)
    eng = _engine(W)
    try:
        emb, feat = _device_inputs(eng, imgs, pts, tm)
        g_dev, pred, masks, losses = _debug_grads(eng, imgs, pts, pts_rot, tm, gt)
    finally:
        eng.close()
    _check("B=%d N=%d%s" % (B, N, " outside" if outside else ""), W, emb, feat, pts_rot, gt, g_dev, pred, masks, losses)


# ---------------------------------------------------------------------------------------------------------------------
# b. flags: the loss weights and the weight decay reach the kernels, and Adam takes the configured betas and epsilon
@pytest.mark.parametrize("sdf_weight,mask_weight,wd", [(8.0, 1.0, 0.0), (25.0, 0.25, 1e-3)])
def test_gradients_with_non_default_flags(sdf_weight, mask_weight, wd):
    B, N = 3, 77
    W = synth.make_weights(seed=3)
    imgs, pts, pts_rot, tm, gt = _problem(B, N, seed=1)
    eng = _engine(W, sdf_weight=sdf_weight, mask_weight=mask_weight, wd=wd)
    try:
        emb, feat = _device_inputs(eng, imgs, pts, tm)
        g_dev, pred, masks, losses = _debug_grads(eng, imgs, pts, pts_rot, tm, gt)
    finally:
        eng.close()
    _check("sw=%g mw=%g wd=%g" % (sdf_weight, mask_weight, wd), W, emb, feat, pts_rot, gt, g_dev, pred, masks, losses,
           sdf_weight, mask_weight, wd)


def test_adam_step_with_non_default_betas():
    B, N = 3, 77
    beta1, beta2, eps = 0.9, 0.99, 1e-4
    W = synth.make_weights(seed=7)
    imgs, pts, pts_rot, tm, gt = _problem(B, N, seed=2)
    rng = np.random.default_rng(11)
    names = train_var_names()
    probe = _engine(W, beta1=beta1, beta2=beta2, epsilon=eps)
    try:
        g, _, _, _ = _debug_grads(probe, imgs, pts, pts_rot, tm, gt)
        m0 = {n: rng.normal(0, 1e-3, probe._numel(n)).astype(np.float32) for n in names}
        v0 = {n: rng.uniform(0, 1e-5, probe._numel(n)).astype(np.float32) for n in names}
    finally:
        probe.close()
    b1p, b2p = np.float32(0.9 ** 3), np.float32(0.99 ** 3)
    state = {n + "/Adam": m0[n] for n in names}
    state.update({n + "/Adam_1": v0[n] for n in names})
    state.update(beta1_power=b1p, beta2_power=b2p)
    eng = _engine(W, beta1=beta1, beta2=beta2, epsilon=eps)
    try:
        eng.load_train_state(state)
        eng.train_step(imgs, pts, pts_rot, tm, gt, LR)
        after = eng.train_state()
    finally:
        eng.close()
    for n in names:
        w0 = np.asarray(W[n], np.float32).reshape(-1)
        w32, m32, v32, p1, p2 = orc.adam(w0, g[n], m0[n], v0[n], LR, b1p, b2p, beta1, beta2, eps, dtype=np.float32)
        assert np.array_equal(after[n].reshape(-1), w32), n
        assert np.array_equal(after[n + "/Adam"].reshape(-1), m32), n
        assert np.array_equal(after[n + "/Adam_1"].reshape(-1), v32), n
    assert after["beta1_power"] == p1 and after["beta2_power"] == p2


# ---------------------------------------------------------------------------------------------------------------------
# c. the loss's branch points: exact ties of d = gt * sw - pred, gt = +-0 (the accuracy's sign test) and gt at 0.01f and
# its float32 neighbours (the weight mask).  At B * N = 64 one point's share of g_abs is ~1/64, far above the bound
# (~2.4e-4 of g_abs), so a wrong branch at a single point fails.
def test_loss_branch_points_at_exact_ties():
    B, N, sw = 1, 64, 8.0
    W = synth.make_weights(seed=5)
    imgs, pts, pts_rot, tm, gt = _problem(B, N, seed=4)
    eng = _engine(W, sdf_weight=sw)
    try:
        emb, feat = _device_inputs(eng, imgs, pts, tm)
        _, pred, _, _ = _debug_grads(eng, imgs, pts, pts_rot, tm, gt)
        g = gt.reshape(-1).copy()
        ties = np.arange(0, 40, 4)                 # ten points with d = 0 exactly in float32
        g[ties] = pred[ties] / np.float32(sw)
        assert np.array_equal(g[ties] * np.float32(sw), pred[ties])
        t = np.float32(0.01)
        g[41], g[43] = np.float32(0.0), np.float32(-0.0)
        g[45], g[47], g[49] = t, np.nextafter(t, np.float32(0)), np.nextafter(t, np.float32(1))
        gt = g.reshape(B, N)
        g_dev, pred2, masks, losses = _debug_grads(eng, imgs, pts, pts_rot, tm, gt)
    finally:
        eng.close()
    assert np.array_equal(pred2, pred)             # the diagnostic does not update the weights
    d = gt.reshape(-1) * np.float32(sw) - pred
    assert not np.any(d[ties]) and np.signbit(gt.reshape(-1)[43])
    assert list(orc.weight_mask(gt, 4.0)[[45, 47, 49]]) == [4.0, 4.0, 1.0]
    _check("ties B=%d N=%d sw=%g" % (B, N, sw), W, emb, feat, pts_rot, gt, g_dev, pred, masks, losses, sdf_weight=sw)


# ---------------------------------------------------------------------------------------------------------------------
# d. a dead ReLU layer: no gradient reaches below it, so what is left of the gradients there is exact
@pytest.mark.parametrize("stream,layer,wd", [(0, "fold2/conv2", 1e-5), (1, "fold2/conv2", 0.0), (0, "fold1/conv1", 0.0),
                                             (1, "fold1/conv1", 1e-5)])
def test_dead_relu_layer_gradients_are_exact(stream, layer, wd):
    B, N = 2, 100
    scope = orc.SCOPES[stream]
    li = orc.LAYERS.index(layer)
    W = dict(synth.make_weights(seed=6))
    bname = "%s/%s/biases" % (scope, layer)
    W[bname] = np.full_like(W[bname], np.float32(-1e3))
    imgs, pts, pts_rot, tm, gt = _problem(B, N, seed=3)
    eng = _engine(W, wd=wd)
    try:
        emb, feat = _device_inputs(eng, imgs, pts, tm)
        g_dev, pred, masks, losses = _debug_grads(eng, imgs, pts, pts_rot, tm, gt)
    finally:
        eng.close()
    assert not masks[stream][li].any()             # the layer is dead for every point
    wd32 = np.float32(wd)
    # layers up to the dead one: the decay alone in every weight gradient, nothing in a bias gradient; the layer after
    # it (the head, or layer 2) reads only zeros, so its weight gradient is the decay alone too
    for l in orc.LAYERS[:li + 2]:
        n = "%s/%s/" % (scope, l)
        w = np.asarray(W[n + "weights"], np.float32).reshape(-1)
        assert np.array_equal(g_dev[n + "weights"], wd32 * w), n
        if wd == 0.0:
            assert not g_dev[n + "weights"].any(), n
        if l != orc.LAYERS[li + 1]:
            assert not g_dev[n + "biases"].any(), n
    _check("dead %s/%s wd=%g" % (scope, layer, wd), W, emb, feat, pts_rot, gt, g_dev, pred, masks, losses, wd=wd)


# ---------------------------------------------------------------------------------------------------------------------
# e. a context reused across shapes gives the bits of a fresh context loaded with the same state
def _step_on_fresh(W, state, data, max_batch=8):
    eng = _engine(W, max_batch=max_batch)
    try:
        eng.load_train_state(state)
        losses = eng.train_step(*data, LR)
        return losses, _bits(eng.train_state())
    finally:
        eng.close()


def test_reused_context_matches_fresh_contexts():
    W = synth.make_weights(seed=7)
    eng = _engine(W)
    try:
        for i, (B, N) in enumerate([(20, 2048), (3, 77), (1, 1), (9, 333)]):
            data = _problem(B, N, seed=i)
            state = eng.train_state()
            want_l, want_s = _step_on_fresh(W, state, data)
            got_l = eng.train_step(*data, LR)
            assert np.array_equal(got_l, want_l), (B, N, got_l, want_l)
            _same_bits(_bits(eng.train_state()), want_s, (B, N))
    finally:
        eng.close()


def test_small_max_batch_and_default_pts_rot_change_no_bit():
    W = synth.make_weights(seed=7)
    imgs, pts, _, tm, gt = _problem(3, 77, seed=0)
    state = {}
    want_l, want_s = _step_on_fresh(W, state, (imgs, pts, pts, tm, gt))
    got_l, got_s = _step_on_fresh(W, state, (imgs, pts, pts, tm, gt), max_batch=1)   # the encoder grows to 3 images
    assert np.array_equal(got_l, want_l)
    _same_bits(got_s, want_s, "max_batch=1")
    got_l, got_s = _step_on_fresh(W, state, (imgs, pts, None, tm, gt))
    assert np.array_equal(got_l, want_l)
    _same_bits(got_s, want_s, "pts_rot=None")


# ---------------------------------------------------------------------------------------------------------------------
# f. six steps at B = 17 (encodes of 8, 8 and 1 images: the embedding-only graph is captured, replayed and replaced),
# each update bit for bit TF's float32 Adam applied to a probe context's gradients of the same pre-step state
def test_six_step_adam_chain_is_exact():
    B, N, beta1 = 17, 129, 0.9
    W = synth.make_weights(seed=7)
    names = train_var_names()
    eng = _engine(W, beta1=beta1)
    probe = _engine(W, beta1=beta1)
    try:
        for step in range(6):
            data = _problem(B, N, seed=step)
            pre = eng.train_state()
            probe.load_train_state(pre)
            g, _, _, want_losses = _debug_grads(probe, *data)
            losses = eng.train_step(*data, LR)
            post = eng.train_state()
            assert np.array_equal(losses, want_losses), (step, losses, want_losses)
            for n in names:
                w, m, v, p1, p2 = orc.adam(pre[n].reshape(-1), g[n], pre[n + "/Adam"].reshape(-1),
                                           pre[n + "/Adam_1"].reshape(-1), LR, pre["beta1_power"], pre["beta2_power"],
                                           beta1=beta1, dtype=np.float32)
                assert np.array_equal(post[n].reshape(-1), w), (step, n)
                assert np.array_equal(post[n + "/Adam"].reshape(-1), m), (step, n)
                assert np.array_equal(post[n + "/Adam_1"].reshape(-1), v), (step, n)
            assert post["beta1_power"] == p1 and post["beta2_power"] == p2, step
    finally:
        probe.close()
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# g. refusals raise with their message and leave the training state as it was
def test_refusals_leave_the_state_untouched():
    W = synth.make_weights(seed=7)
    imgs, pts, pts_rot, tm, gt = _problem(2, 16, seed=0)
    eng = _engine(W)
    try:
        eng.train_step(imgs, pts, pts_rot, tm, gt, LR)
        before = _bits(eng.train_state())

        def refused(msg, call, *args, **kw):
            with pytest.raises(DisnError, match=re.escape(msg)):
                call(*args, **kw)
            _same_bits(_bits(eng.train_state()), before, msg)

        shape_msg = "train_step: B >= 1, N >= 1, 3-channel images"
        refused(shape_msg, eng.train_step, imgs[:0], pts[:0], pts_rot[:0], tm[:0], gt[:0], LR)
        refused(shape_msg, eng.train_step, imgs, pts[:, :0], pts_rot[:, :0], tm, gt[:, :0], LR)
        big = 4096                              # tiny 8 x 8 images: nothing is read before the refusal
        z = lambda *s: np.zeros(s, np.float32)
        refused("train_step: B <= 4095 images per step", eng.train_step, z(big, 8, 8, 3), z(big, 1, 3), None,
                z(big, 4, 3), z(big, 1), LR)
        n = (1 << 23) + 1                        # B * N = 2^24 + 2
        refused("train_step: B * N <= 2^24 points", eng.train_step, z(2, 8, 8, 3), z(2, n, 3), None, z(2, 4, 3),
                z(2, n), LR)
        for lr in (float("nan"), float("inf")):
            refused("train_step: losses and a finite lr", eng.train_step, imgs, pts, pts_rot, tm, gt, lr)
        begin_msg = "train_begin: beta1, beta2 in [0,1), epsilon > 0"
        refused(begin_msg, eng.train_begin, beta1=1.0)
        refused(begin_msg, eng.train_begin, epsilon=0.0)
    finally:
        eng.close()
    fresh = Engine(device=0, precision="fp32", max_batch=8)
    try:
        fresh.load_weights(W)
        with pytest.raises(DisnError, match="disn_train_begin has not been called"):
            fresh.train_step(imgs, pts, pts_rot, tm, gt, LR)
    finally:
        fresh.close()
    tanh = Engine(device=0, precision="fp32", max_batch=8, tanh=True)
    try:
        tanh.load_weights(W)
        with pytest.raises(DisnError, match=re.escape("train_begin: training with --tanh is not implemented")):
            tanh.train_begin()
    finally:
        tanh.close()
