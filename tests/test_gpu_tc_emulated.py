"""The tensor-core point kernel against oracle/tc_emulator.py, a CPU restatement of its own operand arithmetic.

The 1e-4 bar against the float64 oracle (test_gpu_tc.py, test_gpu_configs.py) is loose enough to pass a DISN_PREC_F16F8
kernel that drops one correction product, uses a wrong e5m2 scale or runs another correction mask.  Here both tensor-core
modes are held to the emulation of exactly the shipped scheme, fed the device's own encoder products (pmap, gbias) and,
for eval_points, the kernel's own projected points, so that what remains is the fp32 accumulation order of the warpgroup
MMAs.  tests/test_tc_emulator_cpu.py checks on every CPU run that each of those faults moves the result by at least three
times the bounds below.

Every case compares pred and each stream (global, local) separately -- the global stream alone has no gather -- and
prints max and RMS of |kernel - emulation| in sdf units (pred / 10).  Each bound is about twice the largest value measured
over all cases and outputs on an H100 SXM (80 GB HBM3, 700 W power limit):
    bf16x3  max 2.60e-6 (gather borders, pred), RMS 3.98e-7;
    f16f8   max 3.67e-6 (grid res 40, pred),    RMS 5.95e-7 (gather borders, pred);
    fp32 path against the float64 restatement: max 1.51e-7.
RMS bounds apply to comparisons of at least RMS_MIN_COUNT values."""
import numpy as np
import pytest

from disn_b200 import synth
from oracle import disn_oracle as orc
from oracle import tc_emulator as te

pytestmark = pytest.mark.gpu

MODES = ("bf16x3", "f16f8")
BOUND = {"bf16x3": {"max": 5.5e-6, "rms": 8e-7}, "f16f8": {"max": 7.5e-6, "rms": 1.2e-6}}
FP32_BOUND = 3.2e-7
RMS_MIN_COUNT = 4096
HS_BYTES, W_TILE, W8_TILE = 32768, 16384, 8192
STAGES_PER_STREAM = 33
LAYER_POS = (0, 1, 9, 25)          # first stage of each tensor layer within a stream (point_tc.cu kLayerPos)


def _scaled_heads(W, s):
    from tests.test_gpu_configs import _scaled_heads as f
    return f(W, s)


def _engine(W, precision, max_batch=2):
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision=precision, max_batch=max_batch)
    eng.load_weights(W)
    return eng


@pytest.fixture(scope="module", params=MODES)
def tc(request, he_weights):
    eng = _engine(he_weights, request.param)
    yield request.param, eng
    eng.close()


def _stats(got, ref, div):
    d = np.abs(np.asarray(got, np.float64).reshape(-1) - np.asarray(ref, np.float64).reshape(-1)) / div
    return float(d.max()), float(np.sqrt(np.mean(d * d))), d.size


def _check(mode, case, pairs, div=orc.SDF_WEIGHT):
    """pairs: name -> (kernel, emulation); prints and bounds max and RMS of |kernel - emulation| / div."""
    bound = BOUND[mode]
    bad = []
    for name, (got, ref) in pairs.items():
        mx, rms, n = _stats(got, ref, div)
        print("tc-emulated %-6s %-34s %-6s max %.2e rms %.2e (n=%d)" % (mode, case, name, mx, rms, n))
        if not mx <= bound["max"] or (n >= RMS_MIN_COUNT and not rms <= bound["rms"]):
            bad.append((name, mx, rms))
    assert not bad, (mode, case, bad, bound)


def _points_ex(eng, W, mode, case, pts, tm):
    """eval_points_ex vs the emulation on the kernel's own uv (checked against the float32 projection first)."""
    pred, uv, g, l = eng.eval_points_ex(pts, tm)
    uv32 = te.project_f32(pts, tm, eng.cfg.clamp_max)
    assert (np.abs(uv - uv32) <= 4 * np.spacing(np.maximum(np.abs(uv32), np.float32(1)))).all(), case
    pmap, gbias = eng.get_encoded(6), eng.get_encoded(7)
    emu = te.emulate(W, pts, tm, pmap, gbias, mode, uv=uv, clamp_max=eng.cfg.clamp_max)
    _check(mode, case, {"pred": (pred, emu["pred"]), "global": (g, emu["global"]), "local": (l, emu["local"])})
    return emu


# --------------------------------------------------------------------------------------------------- packing
def _sw128(row, chunk):
    return (row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4)


def _sw64(row, chunk):
    return (row >> 3) * 512 + (row & 7) * 64 + ((chunk ^ ((row >> 1) & 3)) << 4)


def _unpack(s, l):
    """Byte offsets in the packed image of element (k, n) of tensor layer l of stream s: (16-bit tile offset, 8-bit
    tile offset), each [K, N], relative to the half-stage base (tiles are added by the caller)."""
    K, N = te.LAYER_K[l], te.LAYER_N[l]
    k = np.arange(K)[:, None]
    n = np.arange(N)[None, :]
    t, kk, nb, half, nl = k // 64, k % 64, n // 256, (n % 256) // 128, n % 128
    pos = s * STAGES_PER_STREAM + LAYER_POS[l] + t * (N // 256) + nb
    base = (2 * pos + half) * HS_BYTES
    return base + _sw128(nl, kk // 8) + (kk % 8) * 2, base + W_TILE + _sw64(nl, kk // 16) + kk % 16


def _bits16(image, off):
    return (image[off].astype(np.uint16) | (image[off + 1].astype(np.uint16) << 8))


@pytest.mark.parametrize("scale", [1.0, 2.0 ** -6, 2.0 ** 10])
@pytest.mark.parametrize("mode", MODES)
def test_packed_weights_and_scales_equal_the_emulation_bit_for_bit(he_weights, mode, scale):
    """The packed half-stage images (un-swizzled with the SW128 / SW64 offsets) and the activation-scale table equal the
    emulation's operands exactly, and the layout covers every byte of the image once."""
    import ctypes as C

    import torch
    from disn_b200 import _lib
    W = he_weights if scale == 1.0 else _scaled_heads(he_weights, scale)
    lib = _lib.load_test()
    eng = _engine(W, mode, max_batch=1)
    try:
        image = np.zeros(2 * 2 * STAGES_PER_STREAM * HS_BYTES, np.uint8)
        act = np.zeros((2, 4, 2), np.float32)
        prec = _lib.PREC_BF16X3 if mode == "bf16x3" else _lib.PREC_F16F8
        _lib.check(lib.disn_debug_tc_weights(eng._h, prec, image.size, image.ctypes.data_as(C.c_void_p),
                                             act.ctypes.data_as(C.c_void_p)))
    finally:
        eng.close()
    np.testing.assert_array_equal(act, te.act_scales(W))
    ops = te.weight_operands(W, mode)
    bits = lambda t: t.view(torch.int16 if t.element_size() == 2 else torch.uint8).numpy().view(
        np.uint16 if t.element_size() == 2 else np.uint8)
    seen = np.zeros(image.size, np.int32)
    for s in range(2):
        for l in range(4):
            o16, o8 = _unpack(s, l)
            if mode == "bf16x3":
                fields = {"hi": (o16, 2), "lo": (o16 + W_TILE, 2)}
            else:
                fields = {"h": (o16, 2), "e1": (o8, 1), "e2": (o8 + W8_TILE, 1)}
            for name, (off, width) in fields.items():
                got = _bits16(image, off) if width == 2 else image[off]
                np.testing.assert_array_equal(got, bits(ops[s][l][name]), err_msg="%s stream %d layer %d" % (name, s, l))
                for b in range(width):
                    np.add.at(seen, (off + b).reshape(-1), 1)
    assert (seen == 1).all()


# --------------------------------------------------------------------------------------------------- eval_points_ex
@pytest.mark.parametrize("n", [1, 63, 64, 65, 4099, 20000])
def test_eval_points_tiles_and_ring_edges(tc, he_weights, n):
    """B = 2 with different images and cameras.  N = 4099 gives 130 tiles (at most one per CTA on 132 SMs); N = 20000
    gives 626 tiles: uneven tile counts per CTA and many wraps of the weight ring."""
    mode, eng = tc
    eng.encode(synth.synthetic_images(2, seed=77))
    tm = np.concatenate([synth.DEMO_TRANS_MAT, synth.synthetic_trans_mats(1, seed=78)], axis=0)
    pts = np.random.default_rng(1000 + n).uniform(-1, 1, size=(2, n, 3)).astype(np.float32)
    _points_ex(eng, he_weights, mode, "points N=%d" % n, pts, tm)


def _points_on_pixels(tm, uv_target, rng):
    """Points whose projection through tm is uv_target [M,2] in float64: a random depth, then the 3x3 system solved."""
    T = np.asarray(tm, np.float64).reshape(4, 3)
    p0 = rng.uniform(-0.8, 0.8, size=(len(uv_target), 3))
    q2 = p0 @ T[:3, 2] + T[3, 2]
    q = np.stack([uv_target[:, 0] * q2, uv_target[:, 1] * q2, q2], axis=1)
    return np.linalg.solve(T[:3].T[None], (q - T[3])[..., None])[..., 0].astype(np.float32)


def test_gather_at_borders_and_integer_pixels(tc, he_weights):
    """Points projecting onto integer pixels (both taps of an axis on one texel: the floor and the weights at their
    edges), onto the clamped borders u or v = 0 and 136 (the far taps fall outside the 137 x 137 map) and beyond them."""
    mode, eng = tc
    eng.encode(synth.synthetic_images(2, seed=79))
    tm = np.concatenate([synth.DEMO_TRANS_MAT, synth.synthetic_trans_mats(1, seed=80)], axis=0)
    rng = np.random.default_rng(81)
    edge = np.array([-7.0, -0.5, 0.0, 0.5, 1.0, 68.0, 135.0, 135.5, 136.0, 136.5, 150.0])
    grid = np.stack(np.meshgrid(edge, edge, indexing="ij"), axis=-1).reshape(-1, 2)
    pts = []
    for b in range(2):
        ints = rng.integers(0, 137, size=(2048, 2)).astype(np.float64)
        pts.append(_points_on_pixels(tm[b], np.concatenate([np.tile(grid, (8, 1)), ints], axis=0), rng))
    pts = np.stack(pts)
    emu = _points_ex(eng, he_weights, mode, "gather borders", pts, tm)
    u = emu["uv"]
    assert (u == 0).any() and (u == 136).any() and (u == np.round(u)).mean() > 0.3   # the edges were reached


# --------------------------------------------------------------------------------------------------- grid mode
def test_grid_mode_sampled_points(tc, he_weights):
    """eval_grid at sdf_res 40 and a z-slab of it: 8000 (4000) sampled points against the emulation on the reference's
    grid coordinates (orc.grid_points), with the result divided by sdf_weight like the grid path."""
    mode, eng = tc
    imgs = synth.synthetic_images(1, seed=82)
    eng.encode(imgs)
    tm, sp = synth.DEMO_TRANS_MAT, np.array([[-1.0, -0.9, -0.8, 1.0, 0.7, 0.9]])
    R = 41
    pmap, gbias = eng.get_encoded(6), eng.get_encoded(7)
    allpts = orc.grid_points(sp[0], R)
    rng = np.random.default_rng(83)
    for z0, z1, n in ((0, R, 8000), (17, 29, 4000)):
        grid = eng.eval_grid(sp, tm, R - 1, z0=z0, z1=z1).reshape(-1)
        idx = rng.choice(grid.size, n, replace=False)
        pts = allpts[z0 * R * R + idx][None]
        emu = te.emulate(he_weights, pts, tm, pmap, gbias, mode, out_div=orc.SDF_WEIGHT, clamp_max=eng.cfg.clamp_max)
        _check(mode, "grid res 40 z [%d, %d)" % (z0, z1), {"pred": (grid[idx], emu["pred"][0])}, div=1.0)


# --------------------------------------------------------------------------------------------------- activation range
@pytest.mark.parametrize("scale", [2.0 ** -6, 2.0 ** -3, 1.0, 2.0 ** 6, 2.0 ** 10])
@pytest.mark.parametrize("mode", MODES)
def test_activation_range(he_weights, mode, scale):
    """The same function with the internal activations scaled by `scale` (test_gpu_configs._scaled_heads).  At the small
    scales the e5m2 residual operands underflow; the emulation reproduces which ones."""
    W = _scaled_heads(he_weights, scale)
    eng = _engine(W, mode, max_batch=1)
    try:
        eng.encode(synth.synthetic_images(1, seed=84))
        pts = np.random.default_rng(85).uniform(-1, 1, size=(1, 8192, 3)).astype(np.float32)
        _points_ex(eng, W, mode, "activations x 2^%d" % round(np.log2(scale)), pts, synth.DEMO_TRANS_MAT)
    finally:
        eng.close()


def test_f16f8_fp16_guard_edges(he_weights):
    """The largest fp16 A operand placed (through the emulation) in [65504, 65520), where it rounds to 65504: the call
    succeeds and matches; placed above 65520, where it rounds to +inf: the call raises "fp16 range".  N % 64 == 0, so
    every activation the kernel folds into its range guard belongs to a real point."""
    from disn_b200._lib import DisnError
    img, tm = synth.synthetic_images(1, seed=86), synth.DEMO_TRANS_MAT
    pts = np.random.default_rng(87).uniform(-1, 1, size=(1, 1024, 3)).astype(np.float32)
    eng = _engine(he_weights, "f16f8", max_batch=1)
    try:
        def emulate_at(s):
            W = _scaled_heads(he_weights, s)
            eng.load_weights(W)
            eng.encode(img)
            return W, te.emulate(W, pts, tm, eng.get_encoded(6), eng.get_encoded(7), "f16f8",
                                 uv=te.project_f32(pts, tm, eng.cfg.clamp_max))

        s = 1.0
        for _ in range(4):                 # the activations scale with s up to rounding: converge on the window
            W, emu = emulate_at(s)
            if 65504.0 <= emu["act_max"] < 65520.0:
                break
            s *= 65512.0 / emu["act_max"]
        assert 65504.0 <= emu["act_max"] < 65520.0 and not emu["overflow"], emu["act_max"]
        _points_ex(eng, W, "f16f8", "fp16 guard: max %.1f" % emu["act_max"], pts, tm)

        W, emu = emulate_at(s * 65536.0 / 65512.0)
        assert emu["act_max"] >= 65520.0 and emu["overflow"], emu["act_max"]
        with pytest.raises(DisnError, match="fp16 range"):
            eng.eval_points_ex(pts, tm)
    finally:
        eng.close()


# --------------------------------------------------------------------------------------------------- fp32 path
def test_fp32_path_matches_the_float64_restatement(he_weights):
    """point_fp32 against the float64 restatement ("exact" mode) of the same device encoder products."""
    eng = _engine(he_weights, "fp32")
    try:
        eng.encode(synth.synthetic_images(2, seed=88))
        tm = np.concatenate([synth.DEMO_TRANS_MAT, synth.synthetic_trans_mats(1, seed=89)], axis=0)
        pts = np.random.default_rng(90).uniform(-1, 1, size=(2, 4099, 3)).astype(np.float32)
        pred, _, g, l = eng.eval_points_ex(pts, tm)
        ref = te.emulate(he_weights, pts, tm, eng.get_encoded(6), eng.get_encoded(7), "exact", clamp_max=eng.cfg.clamp_max)
    finally:
        eng.close()
    for name, got, want in (("pred", pred, ref["pred"]), ("global", g, ref["global"]), ("local", l, ref["local"])):
        mx, rms, n = _stats(got, want, orc.SDF_WEIGHT)
        print("tc-emulated fp32   %-34s %-6s max %.2e rms %.2e (n=%d)" % ("vs float64 restatement", name, mx, rms, n))
        assert mx <= FP32_BOUND, (name, mx)
