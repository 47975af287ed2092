"""GPU tests of decoder training (disn_train_*, Engine.train_*): one step's gradients, losses and Adam update against the
float64 oracle (oracle/train_oracle.py), ten steps, determinism, the handoff to inference and the frozen encoder.

Gradient bound: every device gradient g_dev of the 24 variables satisfies |g_dev - g_64| <= C_GRAD * 2^-24 * g_abs, where
g_64 is the oracle's gradient with the device's ReLU masks and |.| signs, and g_abs is the same passes run on |.| of every
operand.  C_GRAD covers the bf16 hi/lo split products (about 2^-15 relative each, 2^9 units of 2^-24), fp32 accumulation
and the depth of the forward and backward chains; the tests print the measured fraction of the bound.
"""
import ctypes as C

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


def _problem(B, N, seed=0):
    rng = np.random.default_rng(seed)
    imgs = synth.synthetic_images(B, seed=100 + seed)
    tm = synth.synthetic_trans_mats(B, seed=200 + seed).astype(np.float32)
    pts = rng.uniform(-0.5, 0.5, size=(B, N, 3)).astype(np.float32)
    pts_rot = pts if seed % 2 == 0 else rng.uniform(-0.5, 0.5, size=(B, N, 3)).astype(np.float32)
    r = np.linalg.norm(pts_rot.astype(np.float64), axis=2)
    gt = ((r - 0.3) - 0.003).astype(np.float32)          # a sphere's field, fed as sdf_val - 0.003
    return imgs, pts, pts_rot, tm, gt


def _engine(W, precision="fp32"):
    eng = Engine(device=0, precision=precision, max_batch=8)
    eng.load_weights(W)
    eng.train_begin()
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
    lib = _lib.load_test()
    B, N, _ = pts.shape
    names = train_var_names()
    sizes = [eng._numel(n) for n in names]
    grads = np.empty(sum(sizes), np.float32)
    pred = np.empty(B * N, np.float32)
    acts = np.empty(2 * B * N * (64 + 256 + 512 + 512 + 256), np.float32)
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
        for w in (64, 256, 512, 512, 256):
            masks[si].append(acts[o:o + B * N * w].reshape(B * N, w) > 0)
            o += B * N * w
    return out, pred, masks, losses


@pytest.mark.parametrize("B,N", [(2, 256), (20, 2048)])
@pytest.mark.parametrize("seed", [7, 3])
def test_gradients_match_oracle(B, N, seed):
    W = synth.make_weights(seed=seed)
    imgs, pts, pts_rot, tm, gt = _problem(B, N, seed)
    eng = _engine(W)
    try:
        emb, feat = _device_inputs(eng, imgs, pts, tm)
        g_dev, pred, masks, losses = _debug_grads(eng, imgs, pts, pts_rot, tm, gt)
    finally:
        eng.close()
    d = gt.reshape(-1) * np.float32(10) - pred
    signs = np.sign(d.astype(np.float64))
    _, g64 = orc.step_grads(W, emb, feat, pts, pts_rot, gt, masks=masks, signs=signs)
    _, gabs = orc.step_grads(W, emb, feat, pts, pts_rot, gt, masks=masks, absolute=True)
    worst = 0.0
    for name in orc.var_names():
        err = np.abs(g_dev[name].astype(np.float64) - g64[name].reshape(-1))
        bound = C_GRAD * U * gabs[name].reshape(-1) + 1e-30
        frac = float(np.max(err / bound))
        worst = max(worst, frac)
        assert frac <= 1.0, (name, frac)
    print("B=%d N=%d seed=%d: worst gradient error = %.3g of the bound (C = %g)" % (B, N, seed, worst, C_GRAD))
    # the five reported values: within 2 float32 ulp of get_loss on the device's pred
    want = orc.reported_losses(pred, gt, W)
    for k in range(5):
        assert abs(losses[k] - want[k]) <= 2 * np.spacing(np.float32(want[k])), (k, losses[k], want[k])


def test_adam_step_matches_restatement():
    B, N = 2, 256
    W = synth.make_weights(seed=7)
    imgs, pts, pts_rot, tm, gt = _problem(B, N)
    rng = np.random.default_rng(5)
    names = train_var_names()
    probe = _engine(W)      # the diagnostic library's gradients, on a context of its own (the libraries share no state)
    try:
        g, _, _, _ = _debug_grads(probe, imgs, pts, pts_rot, tm, gt)
        m0 = {n: rng.normal(0, 1e-3, probe._numel(n)).astype(np.float32) for n in names}
        v0 = {n: rng.uniform(0, 1e-5, probe._numel(n)).astype(np.float32) for n in names}
    finally:
        probe.close()
    state = {n + "/Adam": m0[n] for n in names}
    state.update({n + "/Adam_1": v0[n] for n in names})
    state.update(beta1_power=np.float32(0.125), beta2_power=np.float32(0.997))
    eng = _engine(W)
    try:
        eng.load_train_state(state)
        eng.train_step(imgs, pts, pts_rot, tm, gt, LR)
        after = eng.train_state()
    finally:
        eng.close()
    for n in names:
        w0 = np.asarray(W[n], np.float32).reshape(-1)
        w32, m32, v32, b1, b2 = orc.adam(w0, g[n], m0[n], v0[n], LR, 0.125, 0.997, dtype=np.float32)
        assert np.array_equal(after[n].reshape(-1), w32), n                    # TF's float32 operations, bit for bit
        assert np.array_equal(after[n + "/Adam"].reshape(-1), m32), n
        assert np.array_equal(after[n + "/Adam_1"].reshape(-1), v32), n
        # the float32 twin against float64: three roundings of 2^-24 relative each, on the magnitudes of the operands
        _, m64, v64, _, _ = orc.adam(w0, g[n], m0[n], v0[n], LR, 0.125, 0.997)
        gd, md, vd = (np.asarray(a, np.float64) for a in (g[n], m0[n], v0[n]))
        assert np.all(np.abs(m32 - m64) <= 2.0 ** -22 * (np.abs(md) + np.abs(gd))), n
        assert np.all(np.abs(v32 - v64) <= 2.0 ** -22 * (vd + gd * gd)), n
    assert after["beta1_power"] == np.float32(0.125) * np.float32(0.5)
    assert after["beta2_power"] == np.float32(0.997) * np.float32(0.999)


def _run(W, data, steps, precision="fp32"):
    eng = _engine(W, precision)
    try:
        losses = [eng.train_step(*data, LR) for _ in range(steps)]
        return eng.train_state(), np.array(losses)
    finally:
        eng.close()


def test_ten_steps_match_oracle_and_are_deterministic():
    B, N = 2, 256
    W = synth.make_weights(seed=7)
    imgs, pts, pts_rot, tm, gt = _problem(B, N)
    data = (imgs, pts, pts_rot, tm, gt)
    s1, l1 = _run(W, data, 10)
    s2, l2 = _run(W, data, 10)
    assert np.array_equal(l1, l2)
    for k in s1:
        assert np.array_equal(s1[k], s2[k]), k
    eng = _engine(W)
    try:
        emb, feat = _device_inputs(eng, imgs, pts, tm)
    finally:
        eng.close()
    w = {n: np.asarray(W[n], np.float64) for n in orc.var_names()}
    m = {n: np.zeros(w[n].size) for n in w}
    v = {n: np.zeros(w[n].size) for n in w}
    b1p, b2p = 0.5, 0.999
    full = dict(W)
    for step in range(10):
        full.update(w)
        pred, g = orc.step_grads(full, emb, feat, pts, pts_rot, gt)
        want = orc.reported_losses(pred, gt, full)
        assert abs(l1[step][2] - want[2]) <= 1e-2 * abs(want[2]), (step, l1[step], want)
        for n in w:
            nw, m[n], v[n], _, _ = orc.adam(w[n].reshape(-1), g[n].reshape(-1), m[n], v[n], LR, b1p, b2p)
            w[n] = nw.reshape(w[n].shape)
        b1p, b2p = b1p * 0.5, b2p * 0.999
    # Adam moves a weight by about lr per step whatever the gradient's size, so a gradient that is ~0 in exact arithmetic
    # may move its weight either way on the device: the median element must agree to a tenth of one step, and at most
    # 1 % of all elements may differ by more than one step (lr)
    far, total = 0, 0
    for n in w:
        diff = np.abs(s1[n].reshape(-1).astype(np.float64) - w[n].reshape(-1))
        print("%s: max %.3g lr, median %.3g lr, %d of %d beyond one step" % (n, diff.max() / LR, np.median(diff) / LR,
                                                                         int((diff > LR).sum()), diff.size))
        assert np.median(diff) <= 0.1 * LR, (n, np.median(diff))
        far += int((diff > LR).sum())
        total += diff.size
    # only weights whose gradient is ~0 in exact arithmetic may drift by more than one step: at most 1 % of them
    assert far <= 0.01 * total, (far, total)


def test_inference_after_training():
    B, N = 2, 256
    W = synth.make_weights(seed=7)
    imgs, pts, pts_rot, tm, gt = _problem(B, N)
    eng = Engine(device=0, precision="fp32", max_batch=8)
    try:
        eng.load_weights(W)
        eng.encode(imgs)
        emb0 = eng.get_encoded(0)
        taps0 = [eng.get_encoded(t) for t in range(1, 6)]
        eng.train_begin()
        for _ in range(3):
            eng.train_step(imgs, pts, pts_rot, tm, gt, LR)
        with pytest.raises(DisnError, match="stale"):
            eng.eval_points(pts, tm)
        with pytest.raises(DisnError, match="stale"):
            eng.sdf_metrics(pts, tm, gt)
        state = eng.train_state()
        for name, a in W.items():         # the frozen encoder's variables, bit for bit as loaded
            if name.startswith("vgg_16/"):
                assert np.array_equal(eng.train_get(name, a.size), np.asarray(a, np.float32).reshape(-1)), name
        W2 = dict(W)
        W2.update({n: state[n] for n in train_var_names()})
        for prec in ("fp32", "bf16x3", "f16f8"):
            eng.set_precision(prec)
            eng.encode(imgs)
            if prec == "fp32":      # the frozen encoder: bit for bit its output before training
                assert np.array_equal(eng.get_encoded(0), emb0)
                for t in range(1, 6):
                    assert np.array_equal(eng.get_encoded(t), taps0[t - 1])
            got = eng.eval_points(pts, tm, pts_rot=pts_rot)
            got_m = eng.sdf_metrics(pts, tm, gt + np.float32(0.003), want_pred=True)
            fresh = Engine(device=0, precision=prec, max_batch=8)
            try:
                fresh.load_weights(W2)
                fresh.encode(imgs)
                assert np.array_equal(got, fresh.eval_points(pts, tm, pts_rot=pts_rot)), prec
                want_m = fresh.sdf_metrics(pts, tm, gt + np.float32(0.003), want_pred=True)
                for a, b in zip(got_m, want_m):
                    assert np.array_equal(a, b), prec
            finally:
                fresh.close()
        assert not np.array_equal(state["sdfprediction_imgfeat/fold2/conv1/weights"],
                                  np.asarray(W["sdfprediction_imgfeat/fold2/conv1/weights"], np.float32))
    finally:
        eng.close()


def test_overfits_one_batch():
    """300 steps on one batch at lr 1e-4 bring sdf_loss to at most half its first value (a loose check of learning)."""
    B, N = 2, 256
    W = synth.make_weights(seed=7)
    data = _problem(B, N)
    _, losses = _run(W, data, 300)
    print("sdf_loss: first %.4f, last %.4f" % (losses[0][2], losses[-1][2]))
    assert losses[-1][2] <= 0.5 * losses[0][2], (losses[0], losses[-1])


def test_phase_times_cover_the_step():
    W = synth.make_weights(seed=7)
    data = _problem(20, 2048)
    eng = _engine(W)
    try:
        for _ in range(2):
            eng.train_step(*data, LR)
        ph = eng.train_phase_ms()
    finally:
        eng.close()
    print("phases (ms):", {k: round(v, 3) for k, v in ph.items()})
    assert set(ph) == {"encode", "gather", "forward", "loss", "backward", "adam"}
    assert all(v > 0 for v in ph.values()), ph


def test_driver_end_to_end_feeds_create_sdf_and_test_sdf_acc(he_weights, golden, tmp_path, capsys):
    """train_sdf on the SDF fixture with the GPU engine; its checkpoint drives create_sdf and test_sdf_acc."""
    import glob
    import random
    from disn_b200 import create_sdf, test_sdf_acc, train_sdf
    from disn_b200.tf_checkpoint import load_checkpoint
    from tests.test_train_cpu import LOG_LINE, driver_args, train_fixture
    root = train_fixture(golden, tmp_path)
    log_dir = tmp_path / "log"
    np.random.seed(0)
    random.seed(0)
    train_sdf.main(driver_args(root, log_dir), weights=he_weights)
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith(" -- ")]
    assert len(lines) == 1 and LOG_LINE.match(lines[0]), lines
    ckpt = load_checkpoint(str(log_dir / "model.ckpt"), model_variables_only=False)
    assert "beta1_power" in ckpt and "sdfprediction/fold2/conv1/weights/Adam_1" in ckpt
    assert not np.array_equal(ckpt["sdfprediction_imgfeat/fold2/conv1/weights"],
                              he_weights["sdfprediction_imgfeat/fold2/conv1/weights"])
    assert np.array_equal(ckpt["vgg_16/conv1/conv1_1/weights"], he_weights["vgg_16/conv1/conv1_1/weights"])
    random.seed(3)
    written = create_sdf.main(["--view_dir", str(root / "views"), "--sdf_dir", str(root / "sdf"), "--test_lst_dir",
                               str(root / "lst"), "--log_dir", str(log_dir), "--sdf_res", "16", "--view_num", "2"])
    objs = sorted(glob.glob(str(log_dir / "test_objs" / "17_0.0" / "*" / "*.obj")))
    assert len(objs) == 4 * 2 and sorted(written) == objs
    test_sdf_acc.main(["--view_dir", str(root / "views"), "--sdf_dir", str(root / "sdf"), "--test_lst_dir",
                       str(root / "lst"), "--log_dir", str(log_dir), "--batch_size", "8", "--img_feat_twostream",
                       "--precision", "bf16x3"])
    out = capsys.readouterr().out
    assert "Model loaded in file: %s" % (log_dir / "model.ckpt") in out
    summary = [ln for ln in out.splitlines() if ln.startswith("Summary: ")]
    assert len(summary) == 1 and "accuracy: " in summary[0]
