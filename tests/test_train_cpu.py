"""CPU tests of decoder training: the float64 oracle's gradients against central differences, its Adam step against the
formula, the learning-rate schedule of get_learning_rate, and the driver's refusals."""
import random
import re

import numpy as np
import pytest

from disn_b200 import synth
from disn_b200 import train_sdf
from oracle import train_oracle as orc


def _small(seed=0, B=2, N=5, nc=16):
    rng = np.random.default_rng(seed)
    W = {k: v for k, v in synth.make_weights(seed=seed, num_classes=nc).items() if k.startswith("sdfprediction")}
    emb = rng.normal(0, 1, (B, nc))
    feat = rng.normal(0, 1, (B, N, 1472))
    pts = rng.uniform(-0.5, 0.5, (B, N, 3))
    gt = rng.uniform(-0.1, 0.1, (B, N))
    return W, emb, feat, pts, gt


def _overall(W, emb, feat, pts, gt):
    pred, _ = orc.forward(W, emb, feat, pts)
    return orc.loss_terms(pred, gt)[0] + orc.regularization(W)


def test_oracle_gradients_match_central_differences():
    W, emb, feat, pts, gt = _small()
    _, grads = orc.step_grads(W, emb, feat, pts, pts, gt)
    rng = np.random.default_rng(1)
    h = 1e-6
    for name in orc.var_names():
        w = np.asarray(W[name], np.float64)
        for _ in range(3):
            i = int(rng.integers(w.size))
            plus, minus = dict(W), dict(W)
            wp, wm = w.copy().reshape(-1), w.copy().reshape(-1)
            wp[i] += h
            wm[i] -= h
            plus[name], minus[name] = wp.reshape(w.shape), wm.reshape(w.shape)
            fd = (_overall(plus, emb, feat, pts, gt) - _overall(minus, emb, feat, pts, gt)) / (2 * h)
            g = grads[name].reshape(-1)[i]
            assert abs(fd - g) <= 1e-5 * max(1.0, abs(g)), (name, i, fd, g)


def test_oracle_abs_pass_bounds_the_gradient():
    W, emb, feat, pts, gt = _small(seed=2)
    _, g = orc.step_grads(W, emb, feat, pts, pts, gt)
    pred, cache = orc.forward(W, emb, feat, pts)
    masks = cache["mask"]
    _, gabs = orc.step_grads(W, emb, feat, pts, pts, gt, masks=masks, absolute=True)
    for name in orc.var_names():
        assert np.all(np.abs(g[name]) <= gabs[name] * (1 + 1e-12) + 1e-300), name


def test_adam_matches_formula_over_several_steps():
    beta1, beta2, eps, lr = 0.5, 0.999, 1e-8, 1e-3
    w = np.array([1.0, -2.0, 0.5])
    m = np.zeros(3)
    v = np.zeros(3)
    b1p, b2p = beta1, beta2
    grads = [np.array([0.1, -0.2, 0.0]), np.array([0.3, 0.1, -1.0]), np.array([-0.2, 0.0, 2.0])]
    for t, g in enumerate(grads, start=1):
        w_new, m, v, b1p, b2p = orc.adam(w, g, m, v, lr, b1p, b2p, beta1, beta2, eps)
        # TF's powers enter with the current step's value: beta^t
        lr_t = lr * np.sqrt(1 - beta2 ** t) / (1 - beta1 ** t)
        assert np.isclose(b1p, beta1 ** (t + 1)) and np.isclose(b2p, beta2 ** (t + 1))
        assert np.allclose(w_new, w - lr_t * m / (np.sqrt(v) + eps), rtol=0, atol=1e-15)
        w = w_new
    # the first step with m = v = 0 moves every weight with a non-zero gradient by about lr
    w1, _, _, _, _ = orc.adam(np.zeros(2), np.array([5.0, -1e-3]), np.zeros(2), np.zeros(2), lr, beta1, beta2)
    assert np.allclose(np.abs(w1), lr, rtol=1e-3)


@pytest.mark.parametrize("step", [0, 1, 6249, 6250, 6251, 12500, 10 ** 6, 10 ** 8])
def test_learning_rate_schedule(step):
    F = train_sdf.parser().parse_args(["--batch_size", "32"])
    want = orc.learning_rate(step, 1e-4, 32, 200000, 0.9)
    got = train_sdf.get_learning_rate(step, F)
    assert abs(got - want) <= 1e-6 * want, (step, got, want)
    if step == 10 ** 8:
        assert got == np.float32(1e-6)          # clipped
    if step == 6249:
        assert got == np.float32(1e-4)          # 6249 * 32 < 200000: still the base rate
    if step == 6250:
        assert abs(got - 0.9e-4) <= 1e-10       # the first staircase boundary


def test_driver_requires_train_decoder_only():
    with pytest.raises(NotImplementedError, match="VGG-16"):
        train_sdf.main(["--img_feat_twostream", "--log_dir", "/nonexistent"])


@pytest.mark.parametrize("flags", [["--optimizer", "momentum"], ["--binary"], ["--img_feat_onestream"], ["--threedcnn"],
                                   ["--alpha"], ["--rot"], ["--multi_view"], ["--augcolorfore"], ["--augcolorback"]])
def test_driver_refuses_unimplemented_flags(flags):
    with pytest.raises(NotImplementedError):
        train_sdf.main(["--train_decoder_only", "--img_feat_twostream", "--log_dir", "/nonexistent"] + flags)


def test_initial_weights_follow_tf_initialisers():
    W = train_sdf.initial_weights(num_classes=1024, seed=3)
    w = W["sdfprediction/fold2/conv1/weights"]
    assert w.shape == (1, 1, 1536, 512)
    lim = np.sqrt(6.0 / (1536 + 512))
    assert np.abs(w).max() <= lim and np.abs(w).max() > 0.99 * lim
    assert not W["sdfprediction/fold2/conv1/biases"].any()
    assert np.array_equal(W["vgg_16/fc8/weights"], train_sdf.initial_weights(seed=3)["vgg_16/fc8/weights"])


# ---------------------------------------------------------------------------------------------------------------------
# the driver on the SDF fixture with a CPU twin engine
LOG_LINE = re.compile(r"^ -- \d{3} / \d{3} -- accuracy: -?[0-9.]+, sdf_loss_realvalue: -?[0-9.]+, sdf_loss: -?[0-9.]+, "
                      r"regularization: -?[0-9.]+, overall_loss: -?[0-9.]+, lr: [0-9.]+ time: [0-9.]+, , "
                      r"fetch time per b: [0-9.]+, $")


class TwinTrainer:
    """Engine's training surface on the host: the oracle's decoder forward, gradients and TF's float32 Adam.  The frozen
    encoder is replaced by a stand-in (the embedding and point features are per-image channel means of the image)."""

    def load_weights(self, weights):
        self.W = {k: np.asarray(v, np.float32) for k, v in weights.items()}

    def train_begin(self, beta1=0.5, beta2=0.999, epsilon=1e-8, wd=1e-5, mask_weight=4.0, sdf_weight=10.0):
        self.beta1, self.beta2, self.eps = beta1, beta2, epsilon
        self.m = {n: np.zeros_like(self.W[n]) for n in orc.var_names()}
        self.v = {n: np.zeros_like(self.W[n]) for n in orc.var_names()}
        self.b1p, self.b2p = np.float32(beta1), np.float32(beta2)
        self.vgg_reg = orc.regularization({k: v for k, v in self.W.items() if k.startswith("vgg_16/")})
        self.loaded_state = {}

    def load_train_state(self, state):
        self.loaded_state = dict(state)
        for k, a in state.items():
            if k == "beta1_power":
                self.b1p = np.float32(a)
            elif k == "beta2_power":
                self.b2p = np.float32(a)
            elif k.endswith("/Adam_1"):
                self.v[k[:-7]] = np.asarray(a, np.float32).reshape(self.W[k[:-7]].shape)
            elif k.endswith("/Adam"):
                self.m[k[:-5]] = np.asarray(a, np.float32).reshape(self.W[k[:-5]].shape)

    def train_step(self, imgs, pts, pts_rot, trans_mat, sdf_gt, lr):
        B, N = np.asarray(pts).shape[:2]
        mean = np.asarray(imgs, np.float64).reshape(B, -1, 3).mean(axis=1)
        nc = self.W["sdfprediction/fold2/conv1/weights"].reshape(-1, 512).shape[0] - 512
        emb = np.tile(mean, (1, -(-nc // 3)))[:, :nc]
        feat = np.broadcast_to(np.tile(mean, (1, 1472 // 3 + 1))[:, None, :1472], (B, N, 1472))
        pred, g = orc.step_grads(self.W, emb, feat, pts, pts_rot, sdf_gt)
        sdf_loss, real, acc, _ = orc.loss_terms(pred, sdf_gt)
        reg = np.float32(self.vgg_reg + orc.regularization({n: self.W[n] for n in orc.var_names()}))
        loss32 = np.float32(sdf_loss)
        for n in orc.var_names():
            w, m, v, _, _ = orc.adam(self.W[n], g[n], self.m[n], self.v[n], lr, self.b1p, self.b2p, self.beta1,
                                     self.beta2, self.eps, dtype=np.float32)
            self.W[n], self.m[n], self.v[n] = w.reshape(self.W[n].shape), m, v
        self.b1p, self.b2p = self.b1p * np.float32(self.beta1), self.b2p * np.float32(self.beta2)
        return np.array([np.float32(acc), np.float32(real), loss32, reg, np.float32(loss32 + reg)], np.float64)

    def train_state(self):
        st = {}
        for n in orc.var_names():
            st[n] = self.W[n]
            st[n + "/Adam"] = self.m[n].reshape(self.W[n].shape)
            st[n + "/Adam_1"] = self.v[n].reshape(self.W[n].shape)
        st["beta1_power"], st["beta2_power"] = self.b1p, self.b2p
        return st


def train_fixture(golden, root):
    """The SDF fixture's views and samples under root, with its test lists copied as the training lists."""
    from tests.test_sdf_acc_cpu import write_fixture
    write_fixture(golden["sdf_acc_ref"], root)
    lst = root / "train_lst"
    lst.mkdir()
    for f in (root / "lst").glob("*_test.lst"):
        (lst / f.name.replace("_test.lst", "_train.lst")).write_text(f.read_text())
    return root


def driver_args(root, log_dir, *extra):
    return ["--train_decoder_only", "--img_feat_twostream", "--view_dir", str(root / "views"), "--sdf_dir",
            str(root / "sdf"), "--train_lst_dir", str(root / "train_lst"), "--log_dir", str(log_dir), "--batch_size", "4",
            "--num_sample_points", "16", "--max_epoch", "1", "--backcolorwhite"] + list(extra)


def test_driver_on_the_fixture_logs_saves_and_restores(golden, tmp_path, capsys):
    from disn_b200 import test_sdf_acc
    from disn_b200.tf_checkpoint import load_checkpoint
    root = train_fixture(golden, tmp_path)
    W = {k: v for k, v in synth.make_weights(seed=7, num_classes=16).items()
         if k.startswith("sdfprediction") or k == "vgg_16/fc8/weights"}
    log_dir = tmp_path / "log"
    np.random.seed(0)
    random.seed(0)
    twin = TwinTrainer()
    train_sdf.main(driver_args(root, log_dir, "--num_classes", "16"), engine=twin, weights=W)
    out = capsys.readouterr().out
    lines = [ln for ln in out.splitlines() if ln.startswith(" -- ")]
    assert len(lines) == 1 and lines[0].startswith(" -- 020 / 024 -- "), lines        # 96 views / 4, a line every 20
    assert LOG_LINE.match(lines[0]), lines[0]
    assert "avg accuracy:" in out and "**** EPOCH 000 ****" in out
    log = (log_dir / "log_train.txt").read_text()
    assert lines[0] in log and "best Model saved in file: " in log
    # the Saver's checkpoint: the model variables, the decoder's slots under TF's names, the beta powers
    prefix = test_sdf_acc.checkpoint_prefix(str(log_dir))
    assert prefix == str(log_dir / "model.ckpt")
    ckpt = load_checkpoint(prefix, model_variables_only=False)
    want = set(W) | {n + s for n in orc.var_names() for s in ("/Adam", "/Adam_1")} | {"beta1_power", "beta2_power"}
    assert set(ckpt) == want
    st = twin.train_state()
    for k, a in st.items():
        assert np.array_equal(np.asarray(ckpt[k], np.float32).reshape(-1), np.asarray(a, np.float32).reshape(-1)), k
    assert ckpt["beta1_power"] == np.float32(0.5) ** 25          # 24 steps after the initial beta1
    assert np.array_equal(ckpt["vgg_16/fc8/weights"], W["vgg_16/fc8/weights"])    # the frozen encoder as loaded
    # --restore_model: variables, slots and beta powers come back; the step counter restarts (lr at the base rate)
    twin2 = TwinTrainer()
    train_sdf.main(driver_args(root, tmp_path / "log2", "--num_classes", "16", "--restore_model", str(log_dir)),
                   engine=twin2, weights={k: np.zeros_like(v) for k, v in W.items()})
    assert set(twin2.loaded_state) == want - set(W)
    assert twin2.loaded_state["beta1_power"] == ckpt["beta1_power"]
    assert "lr: 0.000100" in capsys.readouterr().out
