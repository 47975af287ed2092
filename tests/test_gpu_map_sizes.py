"""The image-feature path at feature-map sizes (img_h, img_w) other than the default 137 x 137, square and not.

On a square map, swapping x and y, or img_h and img_w, changes nothing, so a transposed bound, scale or offset in the
encoder's fold (resize-then-project / project-then-resize, pmap_accumulate_kernel), the point kernels' gathers, the
decoder's point_img_feat or the per-image map offsets would pass every 137 x 137 test.  The sizes below reach each branch:

    (137, 137)  control;
    (64, 64)    conv1_2 and conv2_2 both resized before the projection; most projections fall beyond the map;
    (112, 112)  conv2_2 exactly at the hw > img_h boundary (projected first, identity resize);
    (128, 128)  the band (127, 136] between the map's edge and the reference's constant clamp at 136;
    (137, 173), (173, 137)  non-square: projected first at every level, img_w != img_h;
    (256, 256)  larger than the 224 input: nothing resized first, and the clamp at 136 lies inside the map.

Per size and precision: the folded map against float64, the points against oracle/tc_emulator.py on the device's own map
(B = 2 with different images and cameras, N = 4099 so tiles straddle the per-image map offset), the points against the
float64 oracle built at the same FLAGS.img_h / img_w (this pins the projection clamp to the reference's 136), the decoder's
point_img_feat against a float64 resize + resampler of the device's own taps, the grid path, and a non-square input image.
The float64 VGG runs once per input image; every size's maps are resized from its end points.

The bounds are those measured at 137 x 137 (tests/test_gpu_tc_emulated.py, test_gpu_parity.py, test_gpu_tc.py); the
arithmetic does not change with the map size.  Largest values over all sizes on an H100 SXM (80 GB HBM3, 700 W power
limit), in sdf units (pred / 10) unless noted, max / RMS:
    points vs emulation   bf16x3 2.86e-6 / 4.05e-7 (64 x 64), f16f8 4.92e-6 / 5.85e-7 (256 x 256),
                          fp32 vs "exact" 1.87e-7 / 3.67e-8 (137 x 173);
    grid res 40           bf16x3 1.43e-6 / 3.27e-7, f16f8 3.65e-6 / 4.62e-7, fp32 1.50e-7 / 3.35e-8;
    vs float64 oracle     bf16x3 5.28e-6 / 1.95e-6, f16f8 4.28e-5 / 7.66e-6, fp32 5.28e-7 / 6.56e-8;
    folded map            2.84e-5 (tensor cores), 1.21e-6 (fp32) of max |pmap|;
    point_img_feat        3.6 u max |tap| (u = 2^-24).
Border targets beyond 150 pixels (all clamped to 136) placed points farther out and pushed the global stream, which
reads no image feature, past these bounds at every size, 137 x 137 included; the targets stop at 150, as in
test_gpu_tc_emulated.py."""
from types import SimpleNamespace

import numpy as np
import pytest

from disn_b200 import synth
from oracle import disn_oracle as orc
from oracle import tc_emulator as te
from tests.test_gpu_tc_emulated import BOUND, FP32_BOUND, RMS_MIN_COUNT, _points_on_pixels, _stats

pytestmark = pytest.mark.gpu

SIZES = [(137, 137), (64, 64), (112, 112), (128, 128), (137, 173), (173, 137), (256, 256)]
PRECS = ("fp32", "bf16x3", "f16f8")
PMAP_REL = {"fp32": 3e-5, "bf16x3": 5e-5, "f16f8": 5e-5}        # test_gpu_parity.py / test_gpu_tc.py, of max |pmap|
TAP_REL = {"fp32": 2e-5, "bf16x3": 5e-5, "f16f8": 5e-5}
ORACLE_TOL = {"fp32": 1e-5, "bf16x3": 1e-4, "f16f8": 1e-4}     # on pred / SDF_WEIGHT
FEAT_ULPS = 64          # point_img_feat bound, in units of 2^-24 max |tap|: see test_point_img_feat
CLAMP = 136.0
N = 4099
ids = lambda hw: "%dx%d" % hw


# --------------------------------------------------------------------------------------------------- shared inputs
@pytest.fixture(scope="module")
def inputs(he_weights):
    """Two 137 x 137 images and cameras, and their float64 VGG end points (the one expensive oracle run)."""
    imgs = synth.synthetic_images(2, seed=301)
    tm = np.concatenate([synth.DEMO_TRANS_MAT, synth.synthetic_trans_mats(1, seed=302)], axis=0)
    net, ep = orc.vgg_16(orc.tf_resize_bilinear(imgs, orc.VGG_IN, orc.VGG_IN, np.float64),
                         {k: np.asarray(v, np.float64) for k, v in he_weights.items() if k.startswith("vgg_16")},
                         np.float64)
    return SimpleNamespace(imgs=imgs, tm=tm, emb=net.reshape(2, -1), ep=ep, cache={})


def _cached(inp, key, make):
    if key not in inp.cache:
        inp.cache[key] = make()
    return inp.cache[key]


def _enc(inp, hw):
    """orc.encode at FLAGS.img_h, img_w = hw, from the shared end points."""
    return _cached(inp, ("enc", hw), lambda: SimpleNamespace(
        img_embedding=inp.emb, maps=[orc.tf_resize_bilinear(inp.ep[t], hw[0], hw[1], np.float64) for t in orc.VGG_TAPS]))


def _pmap64(inp, W, hw):
    def make():
        Wl = np.asarray(W["sdfprediction_imgfeat/fold2/conv1/weights"], np.float64).reshape(-1, 512)
        offs = np.cumsum([512] + list(orc.TAP_CHANNELS[:-1]))
        return sum(m @ Wl[o:o + c] for m, o, c in zip(_enc(inp, hw).maps, offs, orc.TAP_CHANNELS))
    return _cached(inp, ("pmap", hw), make)


def _edges(n):
    """Pixel coordinates along an axis of n texels: before the map, its first texels, the last texel, between it and the
    map's edge, the edge, beyond it up to the clamp at 136, the clamp and past it (clamped).  Targets beyond 150 all
    clamp to 136 and are taken at 150: farther ones only place the points farther from the object, and the tensor-core
    error grows with the coordinates, beyond what the bounds (measured on points like these) cover."""
    e = [-7.0, -0.5, 0.0, 0.5, 1.0, n / 2 + 0.25, n - 2.0, n - 1.5, n - 1.0, n - 0.75, n - 0.5, n, n + 0.5,
         (n + CLAMP) / 2, 135.5, CLAMP, 136.5, 150.0]
    return np.unique(np.minimum(np.array(e), 150.0))


def _points(inp, hw):
    """[2, N, 3]: per image a grid of u edges (img_w) x v edges (img_h), integer pixels, and random points."""
    def make():
        rng = np.random.default_rng(303 + hw[0] * 1000 + hw[1])
        H, Wd = hw
        grid = np.stack(np.meshgrid(_edges(Wd), _edges(H), indexing="ij"), axis=-1).reshape(-1, 2)
        out = []
        for b in range(2):
            ints = np.stack([rng.integers(0, min(Wd + 8, 151), 1000), rng.integers(0, min(H + 8, 151), 1000)],
                            axis=1).astype(np.float64)
            p = _points_on_pixels(inp.tm[b], np.concatenate([np.tile(grid, (3, 1)), ints], axis=0), rng)
            p = np.concatenate([p, rng.uniform(-1, 1, size=(N - len(p), 3)).astype(np.float32)], axis=0)
            out.append(p)
        return np.stack(out)
    return _cached(inp, ("pts", hw), make)


def _assert_edges_reached(uv, hw):
    H, Wd = hw
    for x, n, axis in ((uv[..., 0], Wd, "u"), (uv[..., 1], H, "v")):
        assert (x == 0).any() and (x == CLAMP).any(), axis
        if n - 1 < CLAMP:
            assert ((x > n - 1) & (x < n)).any(), axis                # the last texel's far taps fall outside
            assert ((x >= n) & (x < CLAMP)).any(), axis               # beyond the map, below the clamp
        else:
            assert ((x > CLAMP - 1) & (x < CLAMP)).any(), axis        # inside the map, next to the clamp
        assert ((x > 1) & (x < min(n, CLAMP) - 1)).mean() > 0.3, axis
    assert (uv == np.round(uv)).mean() > 0.15                      # integer pixels: both taps of an axis on one texel


@pytest.fixture(scope="module", params=[(hw, p) for hw in SIZES for p in PRECS],
                ids=["%s-%s" % (ids(hw), p) for hw in SIZES for p in PRECS])
def ctx(request, he_weights, inputs):
    """One context per (map size, precision), the two images encoded."""
    from disn_b200.engine import Engine
    hw, prec = request.param
    eng = Engine(device=0, precision=prec, max_batch=2, img_h=hw[0], img_w=hw[1])
    eng.load_weights(he_weights)
    eng.encode(inputs.imgs)
    yield hw, prec, eng
    eng.close()


# --------------------------------------------------------------------------------------------------- 1. folded map
def test_folded_map(ctx, he_weights, inputs):
    """get_encoded(6) = sum over the taps of resize(tap_l, img_h, img_w) @ Wl[off_l] against float64; the taps, embedding
    and global bias are size-independent and checked by test_gpu_parity.py / test_gpu_tc.py."""
    hw, prec, eng = ctx
    got, want = eng.get_encoded(6), _pmap64(inputs, he_weights, hw)
    assert got.shape == (2,) + hw + (512,)
    err, scale = float(np.abs(got - want).max()), float(np.abs(want).max())
    print("map-sizes %-9s %-6s pmap max err / max |pmap| %.2e" % (ids(hw), prec, err / scale))
    assert err <= PMAP_REL[prec] * scale, (hw, prec, err / scale)


# --------------------------------------------------------------------------------------------------- 2. emulation
def test_points_against_the_emulation(ctx, he_weights, inputs):
    """eval_points_ex against oracle/tc_emulator.py on the device's own pmap / gbias and the kernel's own uv (itself
    held to the float32 projection with the clamp at 136): the tensor-core modes at test_gpu_tc_emulated.BOUND, the fp32
    path against the float64 restatement ("exact") at FP32_BOUND."""
    hw, prec, eng = ctx
    pts, tm = _points(inputs, hw), inputs.tm
    pred, uv, g, l = eng.eval_points_ex(pts, tm)
    uv32 = te.project_f32(pts, tm, CLAMP)
    assert (np.abs(uv - uv32) <= 4 * np.spacing(np.maximum(np.abs(uv32), np.float32(1)))).all()
    _assert_edges_reached(uv, hw)
    emu = te.emulate(he_weights, pts, tm, eng.get_encoded(6), eng.get_encoded(7), "exact" if prec == "fp32" else prec,
                     uv=uv)
    bad = []
    for name, got, ref in (("pred", pred, emu["pred"]), ("global", g, emu["global"]), ("local", l, emu["local"])):
        mx, rms, n = _stats(got, ref, orc.SDF_WEIGHT)
        print("map-sizes %-9s %-6s vs emulation %-6s max %.2e rms %.2e (n=%d)" % (ids(hw), prec, name, mx, rms, n))
        if prec == "fp32":
            ok = mx <= FP32_BOUND
        else:
            ok = mx <= BOUND[prec]["max"] and (n < RMS_MIN_COUNT or rms <= BOUND[prec]["rms"])
        if not ok:
            bad.append((name, mx, rms))
    assert not bad, (hw, prec, bad)


# --------------------------------------------------------------------------------------------------- 3. float64 oracle
def _band_report(err, tol, pts, tm, hw):
    """Where the points over the bound project before any clamp: beyond min(img - 1, 136) on an axis a clamp at the map's
    last texel and the reference's constant clamp at 136 give different coordinates; split into the band (img - 1, 136]
    and beyond 136."""
    H, Wd = hw
    bad = err > tol
    q = te.project_f64(pts, tm, np.inf)[bad]
    lim = np.array([min(Wd - 1, CLAMP), min(H - 1, CLAMP)])
    edge = np.array([Wd - 1, H - 1])
    past = (q > lim).any(axis=1)
    band = ((q > edge) & (q <= CLAMP)).any(axis=1)
    worst = np.unravel_index(np.argmax(err), err.shape)
    return ("%d points over %.0e, %d of them projecting beyond min(img_w - 1, 136) on u or min(img_h - 1, 136) on v, "
            "where a clamp at the map's last texel and the reference's clamp at 136 differ (%d in the clamp band "
            "(img - 1, 136], %d beyond 136); worst %.3e at unclamped uv %s" % (
                bad.sum(), tol, past.sum(), band.sum(), (q > CLAMP).any(axis=1).sum(), err.max(),
                np.round(te.project_f64(pts[worst[0]][None, worst[1]][None], tm[worst[0]][None], np.inf)[0, 0], 3).tolist()))


def test_points_against_the_float64_oracle(ctx, he_weights, inputs):
    """eval_points against orc.encode / orc.decode at FLAGS.img_h, img_w = the context's size, in float64: random points
    and the border points above, some projecting between the map's last texel and 136, some beyond 136 on each axis.
    The returned uv equals the float32 projection clamped at the reference's constant 136, whatever the map size."""
    hw, prec, eng = ctx
    pts, tm = _points(inputs, hw), inputs.tm
    F = orc.default_flags(img_h=hw[0], img_w=hw[1])
    ref = _cached(inputs, ("decode", hw), lambda: orc.decode(_enc(inputs, hw), pts, pts, tm, he_weights, FLAGS=F,
                                                             dtype=np.float64))
    pred, uv = eng.eval_points(pts, tm, want_uv=True)
    err = np.abs(pred[..., 0].astype(np.float64) - ref["pred_sdf"][..., 0]) / orc.SDF_WEIGHT
    rms = float(np.sqrt(np.mean(err ** 2)))
    print("map-sizes %-9s %-6s vs float64 oracle max %.2e rms %.2e" % (ids(hw), prec, err.max(), rms))
    uv32 = te.project_f32(pts, tm, CLAMP)
    uv_ok = np.abs(uv - uv32) <= 4 * np.spacing(np.maximum(np.abs(uv32), np.float32(1)))
    assert err.max() <= ORACLE_TOL[prec], (hw, prec, _band_report(err, ORACLE_TOL[prec], pts, tm, hw))
    assert uv_ok.all(), (hw, prec, "uv differs from the projection clamped at 136 at %d points, e.g. %s for %s" % (
        (~uv_ok).sum(), uv[~uv_ok][:3].tolist(), uv32[~uv_ok][:3].tolist()))


# --------------------------------------------------------------------------------------------------- 4. point_img_feat
def test_point_img_feat(ctx, inputs):
    """decoder.cu's point_img_feat against float64 resize(tap_l, img_h, img_w) + tf_resampler of the device's own taps
    (get_encoded(1..5)) at the kernel's own uv.  Each output sums four resized texels, each three float32 lerps of taps
    of magnitude <= M; with the resampler weights' and the sum's roundings the float32 error stays below about 41 u M
    (u = 2^-24), so the bound is 64 u M per level, M = max |tap_l| -- where test_gpu_surface.py allows 1e-4 M at 137."""
    hw, prec, eng = ctx
    pts, tm = _points(inputs, hw), inputs.tm
    feat, uv = eng.point_img_feat(pts, tm)
    np.testing.assert_array_equal(uv.view(np.uint32), eng.eval_points(pts, tm, want_uv=True)[1].view(np.uint32))
    off, worst = 0, 0.0
    for l, c in enumerate(orc.TAP_CHANNELS):
        tap = eng.get_encoded(1 + l).astype(np.float64)
        want = orc.tf_resampler(orc.tf_resize_bilinear(tap, hw[0], hw[1], np.float64), uv.astype(np.float64), np.float64)
        err = float(np.abs(feat[:, :, 0, off:off + c] - want).max())
        M = float(np.abs(tap).max())
        worst = max(worst, err / (M * 2.0 ** -24))
        assert err <= FEAT_ULPS * 2.0 ** -24 * M, (hw, prec, orc.VGG_TAPS[l], err / (M * 2.0 ** -24))
        off += c
    print("map-sizes %-9s %-6s point_img_feat max err %.1f u max|tap|" % (ids(hw), prec, worst))


# --------------------------------------------------------------------------------------------------- 5. grid paths
def test_grid_sampled_points(ctx, he_weights, inputs):
    """eval_grid at sdf_res 40, the whole grid and one z-slab, both images: sampled points against the emulation (fp32:
    the float64 restatement) on the reference's grid coordinates, divided by sdf_weight like the grid path."""
    hw, prec, eng = ctx
    tm = inputs.tm
    sp = np.array([[-1.0, -0.9, -0.8, 1.0, 0.7, 0.9], [-0.9, -1.0, -0.7, 0.8, 1.0, 1.0]])
    R = 41
    pmap, gbias = eng.get_encoded(6), eng.get_encoded(7)
    rng = np.random.default_rng(304)
    mode = "exact" if prec == "fp32" else prec
    for z0, z1, n in ((0, R, 3000), (17, 29, 2000)):
        grid = eng.eval_grid(sp, tm, R - 1, z0=z0, z1=z1).reshape(2, -1)
        idx = rng.choice(grid.shape[1], n, replace=False)
        pts = np.stack([orc.grid_points(sp[b], R)[z0 * R * R + idx] for b in range(2)])
        emu = te.emulate(he_weights, pts, tm, pmap, gbias, mode, uv=te.project_f32(pts, tm, CLAMP), out_div=orc.SDF_WEIGHT)
        mx, rms, cnt = _stats(grid[:, idx], emu["pred"], 1.0)
        print("map-sizes %-9s %-6s grid res 40 z [%d, %d) max %.2e rms %.2e (n=%d)" % (ids(hw), prec, z0, z1, mx, rms, cnt))
        if prec == "fp32":
            assert mx <= FP32_BOUND, (hw, z0, z1, mx)
        else:
            assert mx <= BOUND[prec]["max"] and rms <= BOUND[prec]["rms"], (hw, prec, z0, z1, mx, rms)


@pytest.mark.parametrize("prec", PRECS)
def test_indexed_and_adaptive_grids_equal_the_dense_grid_non_square(he_weights, inputs, prec):
    """At 137 x 173, B = 2, image 1 (the second image's map lies one img_h * img_w * 512 block into pmap): the indexed
    points and the coarse-to-fine grid equal the dense grid bit for bit (band = inf: everywhere; band = 1: the numpy
    refinement of the dense grid)."""
    from disn_b200.engine import Engine
    from oracle import adaptive_oracle as ao
    bits = lambda a: np.ascontiguousarray(a, np.float32).view(np.uint32)
    box = np.array([[-1.0, -1.0, -1.0, 1.0, 1.0, 1.0], [-0.8, -0.9, -1.0, 0.9, 1.0, 0.7]])
    res, R = 64, 65
    eng = Engine(device=0, precision=prec, max_batch=2, img_h=137, img_w=173)
    try:
        eng.load_weights(he_weights)
        eng.encode(inputs.imgs)
        dense = eng.eval_grid(box, inputs.tm, res)[1]
        idx = np.random.default_rng(305).choice(R ** 3, 50_000, replace=False)
        got = eng.eval_grid_indexed(box[1], inputs.tm[1], res, idx, image=1)
        np.testing.assert_array_equal(bits(got), bits(dense.reshape(-1)[idx]))
        ptr, counts = eng.eval_grid_adaptive(box[1], inputs.tm[1], res, band=np.inf, image=1)
        assert sum(counts) == R ** 3
        np.testing.assert_array_equal(bits(eng.fetch(ptr, (R, R, R))), bits(dense))
        iso = float(np.median(dense))
        ptr, counts = eng.eval_grid_adaptive(box[1], inputs.tm[1], res, iso=iso, band=1.0, image=1)
        _, want_counts, want = ao.refine(dense, box[1], iso=iso, band=1.0)
        assert counts == want_counts and sum(counts) < R ** 3
        np.testing.assert_array_equal(bits(eng.fetch(ptr, (R, R, R))), bits(want))
    finally:
        eng.close()


# --------------------------------------------------------------------------------------------------- 6. input image
@pytest.mark.parametrize("prec", PRECS)
def test_non_square_input_image(he_weights, prec):
    """A 150 x 190 input (resize_bilinear_tf_kernel with H != W) at map size 137 x 173: the resized input against
    orc.tf_resize_bilinear, the taps against the float64 VGG, the folded map against float64."""
    from disn_b200.engine import Engine
    img = np.random.default_rng(306).random((1, 150, 190, 3), dtype=np.float32)
    F = orc.default_flags(img_h=137, img_w=173)
    enc = orc.encode(img, he_weights, FLAGS=F, dtype=np.float64)
    eng = Engine(device=0, precision=prec, max_batch=1, img_h=137, img_w=173)
    try:
        eng.load_weights(he_weights)
        eng.encode(img)
        np.testing.assert_allclose(eng.get_encoded(8), orc.tf_resize_bilinear(img, 224, 224), rtol=0, atol=1e-6)
        for i, tap in enumerate(orc.VGG_TAPS):
            got, ref = eng.get_encoded(1 + i), enc.vgg_end_points[tap]
            assert np.abs(got - ref).max() <= TAP_REL[prec] * np.abs(ref).max(), tap
        Wl = np.asarray(he_weights["sdfprediction_imgfeat/fold2/conv1/weights"], np.float64).reshape(-1, 512)
        offs = np.cumsum([512] + list(orc.TAP_CHANNELS[:-1]))
        pmap = sum(m @ Wl[o:o + c] for m, o, c in zip(enc.maps, offs, orc.TAP_CHANNELS))
        got = eng.get_encoded(6)
        assert got.shape == (1, 137, 173, 512)
        assert np.abs(got - pmap).max() <= PMAP_REL[prec] * np.abs(pmap).max()
    finally:
        eng.close()


# --------------------------------------------------------------------------------------------------- 7. Session
@pytest.mark.parametrize("prec", ["fp32", "f16f8"])
def test_session_builds_its_engine_at_the_graphs_map_size(he_weights, inputs, prec):
    """Session + get_model with FLAGS.img_h = img_w = 128 runs on 128 x 128 maps (the Session rebuilds the engine it
    made at the default size, with its weights) and equals orc.decode at the same FLAGS."""
    from disn_b200 import create_sdf as cs
    from disn_b200 import model_normalization as model
    hw = (128, 128)
    F = cs.default_flags(sdf_res=8, img_h=hw[0], img_w=hw[1])
    pts = _points(inputs, hw)
    pls = model.placeholder_inputs(2, 1, (137, 137), num_sample_pc=N, scope="inputs_pl", FLAGS=F)
    ep = model.get_model(pls, 1, None, bn=False, FLAGS=F)
    sess = model.Session(weights=he_weights, precision=prec, max_batch=2)
    try:
        pred, uv = sess.run([ep["pred_sdf"], ep["sample_img_points"]], feed_dict={
            pls["imgs"]: inputs.imgs, pls["sample_pc"]: pts, pls["sample_pc_rot"]: pts, pls["trans_mat"]: inputs.tm})
        assert (sess.engine.cfg.img_h, sess.engine.cfg.img_w) == hw and sess.engine.get_encoded(6).shape[1:3] == hw
    finally:
        sess.close()
    ref = _cached(inputs, ("decode", hw), lambda: orc.decode(_enc(inputs, hw), pts, pts, inputs.tm, he_weights,
                                                             FLAGS=orc.default_flags(img_h=hw[0], img_w=hw[1]),
                                                             dtype=np.float64))
    err = np.abs(pred[..., 0] - ref["pred_sdf"][..., 0]) / orc.SDF_WEIGHT
    assert err.max() <= ORACLE_TOL[prec], _band_report(err, ORACLE_TOL[prec], pts, inputs.tm, hw)
    np.testing.assert_allclose(uv, ref["sample_img_points"], rtol=0, atol=2e-4)
