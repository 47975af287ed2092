"""oracle/tc_emulator.py without a GPU: its exact mode against the float64 oracle, its quantizers at their edges, and the
power of tests/test_gpu_tc_emulated.py -- every single fault of the operand scheme that the 1e-4 oracle bar lets through
must move the result by at least three times the bounds that GPU test holds the kernel to."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from disn_b200 import synth
from oracle import disn_oracle as orc
from oracle import tc_emulator as te
from tests.test_gpu_tc_emulated import BOUND


# --------------------------------------------------------------------------------------------------- exact mode
@pytest.mark.parametrize("tanh", [False, True])
def test_exact_mode_equals_the_float64_oracle(he_weights, tanh):
    """Exact mode fed the maps folded the way the encoder folds them (pmap = sum of maps @ Wl, gbias = embedding @ Wg + b)
    equals orc.decode on the same maps: pins the folds, the gather and its borders, the two streams and the output."""
    rng = np.random.default_rng(3)
    H = 40
    maps = [rng.standard_normal((1, H, H, c)) * 0.5 for c in orc.TAP_CHANNELS]
    emb = rng.standard_normal((1, 1024))
    tm = synth.DEMO_TRANS_MAT.astype(np.float64).copy()
    tm[..., :2] *= (H + 4) / 137.0          # the projection covers the small map and runs past its far edge
    pts = rng.uniform(-1, 1, size=(1, 700, 3)).astype(np.float32)
    Wg = np.asarray(he_weights["sdfprediction/fold2/conv1/weights"], np.float64).reshape(-1, 512)
    Wl = np.asarray(he_weights["sdfprediction_imgfeat/fold2/conv1/weights"], np.float64).reshape(-1, 512)
    gbias = emb @ Wg[512:] + np.asarray(he_weights["sdfprediction/fold2/conv1/biases"], np.float64)
    offs = np.cumsum([512] + list(orc.TAP_CHANNELS[:-1]))
    pmap = sum(m @ Wl[o:o + c] for m, o, c in zip(maps, offs, orc.TAP_CHANNELS))
    ref = orc.decode(SimpleNamespace(img_embedding=emb, maps=maps), pts, pts, tm, he_weights,
                     FLAGS=orc.default_flags(tanh=tanh), dtype=np.float64)
    got = te.emulate(he_weights, pts, tm, pmap, gbias, "exact", tanh=tanh)
    assert np.abs(got["pred"] - ref["pred_sdf"][..., 0]).max() <= 1e-12
    assert np.abs(got["global"] + got["local"] - ref["pred_sdf_value_global"][..., 0]
                  - ref["pred_sdf_value_local"][..., 0]).max() <= 1e-12
    assert np.abs(got["uv"] - ref["sample_img_points"]).max() <= 1e-12
    u = got["uv"][..., 0]
    assert (u >= H - 1).any() and (u < H - 1).mean() > 0.5        # inside, on the last column's far taps and past them


@pytest.mark.parametrize("hw", [(24, 40), (40, 24)])
def test_exact_mode_equals_the_float64_oracle_on_a_non_square_map(he_weights, hw):
    """The same on img_h != img_w maps, resized from the taps the way FLAGS.img_h / img_w select, with the projection
    run past both far edges and the constant clamp at 136 beyond them: pins u to img_w and v to img_h in the emulation's
    gather, so that tests/test_gpu_map_sizes.py can lean on it at non-square map sizes."""
    H, W = hw
    F = orc.default_flags(img_h=H, img_w=W)
    rng = np.random.default_rng(5)
    maps = [orc.tf_resize_bilinear(rng.standard_normal((1, 17, 17, c)) * 0.5, F.img_h, F.img_w, np.float64)
            for c in orc.TAP_CHANNELS]
    emb = rng.standard_normal((1, 1024))
    tm = synth.DEMO_TRANS_MAT.astype(np.float64) * np.array([(W + 6) / 137.0, (H + 6) / 137.0, 1.0])
    pts = rng.uniform(-1.3, 1.3, size=(1, 900, 3)).astype(np.float32)
    pts[0, :100] *= 8.0                     # far outside: projections clamped to 0 and to 136
    Wg = np.asarray(he_weights["sdfprediction/fold2/conv1/weights"], np.float64).reshape(-1, 512)
    Wl = np.asarray(he_weights["sdfprediction_imgfeat/fold2/conv1/weights"], np.float64).reshape(-1, 512)
    gbias = emb @ Wg[512:] + np.asarray(he_weights["sdfprediction/fold2/conv1/biases"], np.float64)
    offs = np.cumsum([512] + list(orc.TAP_CHANNELS[:-1]))
    pmap = sum(m @ Wl[o:o + c] for m, o, c in zip(maps, offs, orc.TAP_CHANNELS))
    assert pmap.shape == (1, H, W, 512)
    ref = orc.decode(SimpleNamespace(img_embedding=emb, maps=maps), pts, pts, tm, he_weights, FLAGS=F, dtype=np.float64)
    got = te.emulate(he_weights, pts, tm, pmap, gbias, "exact")
    assert np.abs(got["pred"] - ref["pred_sdf"][..., 0]).max() <= 1e-12
    assert np.abs(got["local"] - ref["pred_sdf_value_local"][..., 0]).max() <= 1e-12
    assert np.abs(got["uv"] - ref["sample_img_points"]).max() <= 1e-12
    u, v = got["uv"][0, :, 0], got["uv"][0, :, 1]
    for x, n in ((u, W), (v, H)):           # inside, between the last texel and the map's edge, past it, clamped
        assert ((x > 1) & (x < n - 1)).mean() > 0.3 and ((x > n - 1) & (x < n)).any() and ((x >= n) & (x < 136)).any()
        assert (x == 136).any() and (x == 0).any()


def test_exact_mode_streams_equal_the_oracle_streams(he_weights):
    rng = np.random.default_rng(4)
    maps = [rng.standard_normal((1, 20, 20, c)) * 0.5 for c in orc.TAP_CHANNELS]
    emb = rng.standard_normal((1, 1024))
    tm = synth.DEMO_TRANS_MAT.astype(np.float64) * np.array([20 / 137.0, 20 / 137.0, 1.0])
    pts = rng.uniform(-1, 1, size=(1, 300, 3)).astype(np.float32)
    Wg = np.asarray(he_weights["sdfprediction/fold2/conv1/weights"], np.float64).reshape(-1, 512)
    Wl = np.asarray(he_weights["sdfprediction_imgfeat/fold2/conv1/weights"], np.float64).reshape(-1, 512)
    gbias = emb @ Wg[512:] + np.asarray(he_weights["sdfprediction/fold2/conv1/biases"], np.float64)
    offs = np.cumsum([512] + list(orc.TAP_CHANNELS[:-1]))
    pmap = sum(m @ Wl[o:o + c] for m, o, c in zip(maps, offs, orc.TAP_CHANNELS))
    ref = orc.decode(SimpleNamespace(img_embedding=emb, maps=maps), pts, pts, tm, he_weights, dtype=np.float64)
    got = te.emulate(he_weights, pts, tm, pmap, gbias, "exact")
    assert np.abs(got["global"] - ref["pred_sdf_value_global"][..., 0]).max() <= 1e-12
    assert np.abs(got["local"] - ref["pred_sdf_value_local"][..., 0]).max() <= 1e-12


# --------------------------------------------------------------------------------------------------- quantizers
def _e5m2_reference(x):
    """fp32 -> e5m2 by search over every finite e5m2 value: nearest, ties to the even code, |x| > 57344 saturates."""
    codes = np.arange(0x7C, dtype=np.uint8)                        # +0 .. 57344
    vals = torch.from_numpy(codes).view(torch.float8_e5m2).float().numpy().astype(np.float64)
    out = np.empty(len(x))
    for i, v in enumerate(np.asarray(x, np.float64)):
        a = min(abs(v), te.E5M2_MAX)
        j = int(np.searchsorted(vals, a))
        cands = [k for k in (j - 1, j) if 0 <= k < len(vals)]
        best = min(cands, key=lambda k: (abs(vals[k] - a), codes[k] & 1))
        out[i] = np.copysign(vals[best], v)
    return out


def test_e5m2_saturates_and_rounds_to_nearest_even():
    x = np.array([57344.0, 57345.0, 59392.0, 61439.0, 61440.0, 65536.0, 1e9, -61440.0, -1e30,
                  2.0 ** -16, 2.0 ** -17, 2.0 ** -17 * (1 + 2.0 ** -20), 3 * 2.0 ** -17, 5 * 2.0 ** -17, 2.0 ** -18,
                  2.0 ** -14, 2.0 ** -14 * 1.125, 2.0 ** -14 * 1.375, 1.125, 1.375, 1.625, 1.875, -1.125, 0.0, -0.0,
                  7.0 * 2.0 ** -16 / 2, 2.0 ** -15 * 1.5], np.float32)
    got = te.q_e5m2(torch.from_numpy(x)).float().numpy()
    np.testing.assert_array_equal(got, _e5m2_reference(x))
    assert got[4] == 57344.0 and got[5] == 57344.0 and got[7] == -57344.0      # SATFINITE, never inf
    assert got[10] == 0.0 and got[11] == 2.0 ** -16 and got[12] == 2.0 ** -15  # subnormal ties to even, above a tie rounds up
    rng = np.random.default_rng(0)
    r = (rng.standard_normal(4000) * 2.0 ** rng.uniform(-20, 17, 4000)).astype(np.float32)
    np.testing.assert_array_equal(te.q_e5m2(torch.from_numpy(r)).float().numpy(), _e5m2_reference(r))


def test_f16f8_activation_copy_rounds_in_fp16():
    """The e5m2 copy of an activation is e5m2(fp16(h * fp16(sc_hi))): the fp16 multiply goes subnormal for small h and
    rounds there first.  h = (1 + 2^-8) 2^-5 times 2^-12 is 2^-17 (1 + 2^-8): fp16 rounds it to 2^-17 (tie to even at
    the subnormal step 2^-24), which e5m2 rounds to 0 (tie to even between 0 and 2^-16); a single rounding would give
    2^-16."""
    a = torch.tensor([(1 + 2.0 ** -8) * 2.0 ** -5, 1.0, 2.0 ** -3], dtype=torch.float32)
    h, lo, g = te.act_operands_f16f8(a, 2.0 ** 9, 2.0 ** -12)
    assert te.q_e5m2(a[:1] * 2.0 ** -12).float().item() == 2.0 ** -16
    assert g.float().tolist() == [0.0, 2.0 ** -12, 2.0 ** -15]
    assert h.float().tolist() == a.tolist() and lo.float().tolist() == [0.0, 0.0, 0.0]
    # the multiplier itself is an fp16: 2^-25 rounds to 0 there, and the copy vanishes
    assert te.act_operands_f16f8(a, 1.0, 2.0 ** -25)[2].float().tolist() == [0.0, 0.0, 0.0]
    # the residual is taken in fp32 and scaled before its e5m2 rounding
    h, lo, _ = te.act_operands_f16f8(torch.tensor([1.0 + 2.0 ** -12], dtype=torch.float32), 2.0 ** 12, 1.0)
    assert h.float().item() == 1.0 and lo.float().item() == 1.0


def test_scale_rule_rounds_halves_away_from_zero_and_clamps():
    assert [te.lround(x) for x in (2.5, -2.5, 3.5, -3.5, 0.49999999999999994, -0.5, 1.4999999)] == [3, -3, 4, -4, 0, -1, 1]
    assert np.round(-2.5) == -2.0                                   # what np.round would have done
    w = np.full((64, 256), 2.0 ** -4, np.float32)
    assert te.layer_scales(w) == (6, 8)
    assert te.layer_scales(w * np.float32(2.0 ** 0.6)) == (7, 9)   # log2 rms = -3.4
    assert te.layer_scales(w * np.float32(2.0 ** -0.6)) == (5, 7)  # log2 rms = -4.6
    assert te.layer_scales(np.zeros((64, 256), np.float32)) == (6, 8)
    assert te.layer_scales(np.full((64, 256), 2.0 ** -30, np.float32)) == (-8, -8)
    assert te.layer_scales(np.full((64, 256), 2.0 ** 20, np.float32)) == (24, 28)
    w[0, 0] = -w[0, 0]                                              # the rms, not the mean
    assert te.layer_scales(w) == (6, 8)


# --------------------------------------------------------------------------------------------------- negative controls
@pytest.fixture(scope="module")
def study(he_weights):
    """He weights, 4000 points through the demo camera, a random image-feature map and global bias of O(1)."""
    rng = np.random.default_rng(0)
    pts = rng.uniform(-1, 1, (1, 4000, 3)).astype(np.float32)
    pmap = (rng.standard_normal((1, 137, 137, 512)) * 0.7).astype(np.float32)
    gbias = (rng.standard_normal((1, 512)) * 0.7).astype(np.float32)
    run = lambda mode, **kw: te.emulate(he_weights, pts, synth.DEMO_TRANS_MAT, pmap, gbias, mode, **kw)["pred"]
    return SimpleNamespace(run=run, W=he_weights, f16f8=run("f16f8"), bf16x3=run("bf16x3"))


def _distance(a, b):
    d = np.abs(a.astype(np.float64) - b) / orc.SDF_WEIGHT
    return float(d.max()), float(np.sqrt(np.mean(d * d)))


def _assert_detectable(mode, variant, ref):
    mx, rms = _distance(variant, ref)
    b = BOUND[mode]
    assert mx >= 3 * b["max"] and rms >= 3 * b["rms"], (mx, rms, b)


KEPT = [bit for bit in range(8) if (te.CORR_DEFAULT >> bit) & 1]


@pytest.mark.parametrize("bit", KEPT)
def test_dropping_any_kept_correction_is_detectable(study, bit):
    assert len(KEPT) == 7
    _assert_detectable("f16f8", study.run("f16f8", corr_mask=te.CORR_DEFAULT & ~(1 << bit)), study.f16f8)


SCALES = [(l, j) for l in range(4) for j in range(2) if (te.CORR_DEFAULT >> (2 * l + j)) & 1]


def _off_by_one(study, layer, which, shift):
    sc = te.act_scales(study.W)
    sc[:, layer, which] *= np.float32(2.0 ** shift)
    return study.run("f16f8", act_scale=sc)


@pytest.mark.parametrize("layer,which", SCALES)
def test_an_activation_scale_one_bit_too_large_is_detectable(study, layer, which):
    """act_scale[.][layer][which] of both streams doubled against the weights' own scale (a wrong table entry or layer
    index); the entry of the correction the shipped mask drops is not read."""
    assert len(SCALES) == 7
    _assert_detectable("f16f8", _off_by_one(study, layer, which, 1), study.f16f8)


@pytest.mark.parametrize("layer,which", SCALES)
def test_an_activation_scale_one_bit_too_small_is_detectable(study, layer, which):
    """Halved, the correction is off by half its size instead of all of it: measured 1.9e-5 .. 2.9e-5 max and 4.0e-6 ..
    8.0e-6 RMS, which clears three times the RMS bound but only twice the max bound."""
    mx, rms = _distance(_off_by_one(study, layer, which, -1), study.f16f8)
    b = BOUND["f16f8"]
    assert rms >= 3 * b["rms"] and mx >= 2 * b["max"], (mx, rms, b)


def test_the_full_correction_mask_is_detectable(study):
    _assert_detectable("f16f8", study.run("f16f8", corr_mask=0xFF), study.f16f8)


def test_bf16x3_without_hi_lo_is_detectable(study):
    _assert_detectable("bf16x3", study.run("bf16x3", keep_hi_lo=False), study.bf16x3)


def test_the_emulation_of_the_shipped_scheme_is_within_the_oracle_bar(study):
    """The shipped schemes themselves against the exact mode: the emulation is the kernel's arithmetic, not a different
    function (the 1e-4 bar of the oracle tests; the operand-rounding budget of DESIGN.md section 3)."""
    exact = study.run("exact")
    assert _distance(study.f16f8, exact)[0] < 5e-5
    assert _distance(study.bf16x3, exact)[0] < 5e-6
