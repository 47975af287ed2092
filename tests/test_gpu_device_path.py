"""GPU tests of the path bench.py times: device pointers, a caller's stream, z-slabs and the cross-process slab gather.

bench.py's run_ours binds the engine to a torch stream (disn_set_stream), encodes from a device image (disn_encode with
DISN_DEVICE_PTR), writes the grid into a device tensor or, on N GPUs, each rank's z-slab into rank 0's HBM through CUDA IPC
(disn_shared_alloc / disn_shared_open), and for config 4 meshes that device grid.  The DISN_DEVICE_PTR branches are code
paths of their own: asynchronous, in the caller's layout, with the f16f8 overflow status reported only at the next
synchronising call.  Both paths reach the same kernels, none of which uses atomics, so on the same encoder products the
device path must give the bits of the host path, which test_gpu_parity.py / test_gpu_configs.py hold to the float64
oracle; a few thousand grid points per configuration are also compared with the oracle directly, so that a wrong device
encode cannot hide behind an equally wrong host one.

Every engine here runs on a non-default torch stream, as in bench.py (handle 0 would mean "the context's own stream")."""
import contextlib
import gc
import multiprocessing
import queue
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from disn_b200 import sharding, synth
from oracle import disn_oracle as orc

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
FP32_TOL = 1e-5                 # test_gpu_parity.py: fp32 CUDA-core path, on pred / 10
TC_TOL = 1e-4                   # tensor-core modes, same unit
BENCH_CONFIGS = {0: (1, 64), 2: (8, 128), 1: (1, 256)}          # bench.py CONFIGS: batch, sdf_res
SLEEP_CYCLES = 200_000_000      # torch.cuda._sleep: ~0.1 s at the H100's 1.98 GHz boost clock, longer when clocked down
NAN = float("nan")


@contextlib.contextmanager
def _engine(weights, precision="f16f8", max_batch=8):
    """An Engine with `weights`, bound to a fresh non-default torch stream; restored to its own stream and closed on
    exit."""
    from disn_b200.engine import Engine
    stream = torch.cuda.Stream(DEV)
    eng = Engine(device=0, precision=precision, max_batch=max_batch)
    try:
        eng.set_stream(stream.cuda_stream)
        try:
            eng.load_weights(weights)
            yield eng, stream
        finally:
            eng.set_stream(None)
    finally:
        eng.close()


@pytest.fixture(scope="module")
def ctx(he_weights):
    with _engine(he_weights) as (eng, stream):
        yield eng, stream


def _dev(a):
    """Host array -> device tensor on the current torch stream."""
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _nan(shape):
    return torch.full(shape, NAN, dtype=torch.float32, device=DEV)


def _host(t, stream):
    """Device tensor -> numpy, ordered after everything enqueued on `stream`."""
    with torch.cuda.stream(stream):
        return t.cpu().numpy()


def _images(B, size, seed):
    if size == 137:
        return synth.synthetic_images(B, seed=seed)
    return np.random.default_rng(seed).random((B, size, size, 3), dtype=np.float32)


def _config_inputs(cfg):
    """bench.py's inputs of a config: images, one trans_mat per image and (for the batch) a distinct box per image."""
    B, res = BENCH_CONFIGS[cfg]
    imgs = _oracle_images()[:B]
    if B == 1:
        return imgs, synth.DEMO_TRANS_MAT.copy(), synth.DEMO_SDF_PARAMS.copy(), res
    tm = synth.synthetic_trans_mats(B, seed=4321)
    sp = np.tile(synth.DEMO_SDF_PARAMS, (B, 1)) * np.linspace(0.8, 1.0, B)[:, None]
    return imgs, tm, sp, res


def _oracle_images():
    return synth.synthetic_images(8, seed=2024)


ORACLE_IMAGES = (0, 5)          # the images of _oracle_images() the float64 oracle encodes (config 2 samples image 5)


@pytest.fixture(scope="module")
def oracle_enc(he_weights):
    """float64 oracle encoder products of two images (~10 s per image on the host)."""
    return orc.encode(_oracle_images()[list(ORACLE_IMAGES)], he_weights, dtype=np.float64)


def _slice_enc(enc, i):
    return SimpleNamespace(resized_ref_img=enc.resized_ref_img[i:i + 1], img_embedding=enc.img_embedding[i:i + 1],
                           maps=[m[i:i + 1] for m in enc.maps], vgg_end_points=None)


def _grid_points_at(sdf_params, R, flat_idx):
    """The reference's float32 grid points (create_sdf.py:246-255) at flat (z,y,x) indices, x fastest."""
    axes = [np.linspace(sdf_params[a], sdf_params[3 + a], num=R) for a in range(3)]
    ix, iy, iz = flat_idx % R, (flat_idx // R) % R, flat_idx // (R * R)
    return np.stack([axes[0][ix], axes[1][iy], axes[2][iz]], axis=1).astype(np.float32)


def _assert_bitwise(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.count_nonzero(~((got == want) | (np.isnan(got) & np.isnan(want))))
    if bad:
        d = np.abs(got.astype(np.float64) - want)
        raise AssertionError("%s: %d of %d values differ from the host path (max |diff| %.3e, %d NaN where the host "
                             "path has a number)" % (what, bad, got.size, np.nanmax(d) if np.isfinite(d).any() else NAN,
                                                     np.count_nonzero(np.isnan(got) & ~np.isnan(want))))


# ---- 1. encoding from device memory ------------------------------------------------------------------------------------
def _products(eng):
    return [eng.get_encoded(w) for w in range(9)]


def test_encode_device_equals_host_encode_through_every_graph_stage(ctx, he_weights):
    """encode_device == encode() on the same host images, all nine encoder products, bit for bit.  Four calls per
    (B, size) with a new image each run the encoder's eager warm-up, graph capture and replay stages; alternating 137² and
    224² inputs then catches a replay that reads a stale input or replays the graph of the other shape.  The host
    references come from two other engines that each only ever see one input size, so their graphs cannot be stale."""
    eng, stream = ctx
    eng.set_precision("f16f8")
    seed = 700
    with _engine(he_weights) as (ref137, _), _engine(he_weights) as (ref224, _):
        refs = {137: ref137, 224: ref224}
        for B in (1, 8):
            for step, size in enumerate([137] * 4 + [224] * 4 + [137, 224, 137, 224]):
                imgs = _images(B, size, seed)
                seed += 1
                refs[size].encode(imgs)
                want = _products(refs[size])
                with torch.cuda.stream(stream):
                    img_d = _dev(imgs)
                    eng.encode_device(img_d.data_ptr(), B, size, size, 3)
                    got = _products(eng)      # get_encoded synchronises the stream the copy above was enqueued on
                for w, (g, r) in enumerate(zip(got, want)):
                    _assert_bitwise(g, r, "B=%d, %d² input, call %d, encoder product %d" % (B, size, step, w))


# ---- 2. grids into device tensors: bench configs, every precision --------------------------------------------------------
_oracle_cache = {}


def _oracle_samples(cfg, enc, W):
    """(image, flat indices, float64 oracle SDF) at 3 000 random grid points of one image of the config."""
    if cfg not in _oracle_cache:
        imgs, tm, sp, res = _config_inputs(cfg)
        R = res + 1
        b = 0 if len(imgs) == 1 else ORACLE_IMAGES[1]
        idx = np.random.default_rng(950 + cfg).choice(R ** 3, size=3000, replace=False)
        pts = _grid_points_at(sp[b], R, idx)[None]
        ref = orc.decode(_slice_enc(enc, ORACLE_IMAGES.index(b)), pts, pts, tm[b:b + 1], W, dtype=np.float64)
        _oracle_cache[cfg] = (b, idx, ref["pred_sdf"].reshape(-1) / orc.SDF_WEIGHT)
    return _oracle_cache[cfg]


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "f16f8"])
@pytest.mark.parametrize("cfg", [0, 2, 1])
def test_eval_grid_device_equals_host_grid_and_oracle(ctx, he_weights, oracle_enc, cfg, precision):
    """bench.py configs 0 (65³), 2 (8 × 129³, a camera and box per image) and 1 (257³): the grid eval_grid_device writes
    into a torch tensor == eval_grid on the same encoder products, bitwise; one image against the float64 oracle."""
    eng, stream = ctx
    imgs, tm, sp, res = _config_inputs(cfg)
    B, R = len(imgs), res + 1
    eng.set_precision(precision)
    with torch.cuda.stream(stream):
        img_d, tm_d, out = _dev(imgs), _dev(tm), _nan((B, R, R, R))
        eng.encode_device(img_d.data_ptr(), B, 137, 137, 3)
        eng.eval_grid_device(sp, tm_d.data_ptr(), res, 0, R, out.data_ptr())
    got = _host(out, stream)
    want = eng.eval_grid(sp, tm, res)
    _assert_bitwise(got, want, "config %d, %s" % (cfg, precision))
    b, idx, ref = _oracle_samples(cfg, oracle_enc, he_weights)
    err = float(np.abs(got[b].reshape(-1)[idx] - ref).max())
    assert err <= (FP32_TOL if precision == "fp32" else TC_TOL), (cfg, precision, err)


# ---- 3. z-slabs at the offsets the sharded run uses ----------------------------------------------------------------------
RES_SLAB = 256
R_SLAB = RES_SLAB + 1
GUARD = 4096                    # NaN floats before and after the peer buffer


def _two_image_inputs():
    imgs = synth.synthetic_images(2, seed=3100)
    tm = synth.synthetic_trans_mats(2, seed=3200)
    sp = np.array([[-1.0, -1.0, -1.0, 1.0, 1.0, 1.0], [-0.9, -1.0, -0.8, 1.0, 0.85, 0.95]])
    return imgs, tm, sp


@pytest.fixture(scope="module")
def grid257(ctx):
    """The single-image f16f8 257³ host grid of bench.py config 1's inputs."""
    eng, _ = ctx
    imgs, tm, sp, _ = _config_inputs(1)
    eng.set_precision("f16f8")
    eng.encode(imgs)
    grid = eng.eval_grid(sp, tm, RES_SLAB)
    assert np.isfinite(grid).all()
    return imgs, tm, sp, grid


@pytest.mark.parametrize("world", [2, 3, 8])
def test_z_slabs_land_at_the_sharded_offsets(ctx, grid257, world):
    """Peer layout: every "rank" writes eval_grid_device(z0, z1) at base + z0*R*R*4 of one R³ buffer with NaN guard bands,
    which must then hold the whole grid bit for bit and leave the guards NaN.  Gather layout: a rank's [1, max_planes, R, R]
    slab; a short slab leaves its unused last plane NaN."""
    eng, stream = ctx
    imgs, tm, sp, full = grid257
    R = R_SLAB
    bounds = sharding.z_bounds(R, world)
    mp = sharding.max_planes(R, world)
    assert any(bounds[r + 1] - bounds[r] < mp for r in range(world))     # a short slab is exercised
    eng.set_precision("f16f8")
    with torch.cuda.stream(stream):
        img_d, tm_d = _dev(imgs), _dev(tm)
        eng.encode_device(img_d.data_ptr(), 1, 137, 137, 3)
        peer = _nan((2 * GUARD + R ** 3,))
        base = peer.data_ptr() + GUARD * 4
        slabs = [_nan((1, mp, R, R)) for _ in range(world)]
        for r in reversed(range(world)):
            z0, z1 = sharding.slab(R, world, r)
            eng.eval_grid_device(sp, tm_d.data_ptr(), RES_SLAB, z0, z1, base + z0 * R * R * 4)
            eng.eval_grid_device(sp, tm_d.data_ptr(), RES_SLAB, z0, z1, slabs[r].data_ptr())
    h = _host(peer, stream)
    assert np.isnan(h[:GUARD]).all() and np.isnan(h[GUARD + R ** 3:]).all(), "a slab was written outside the grid"
    _assert_bitwise(h[GUARD:GUARD + R ** 3].reshape(1, R, R, R), full, "peer layout, world %d" % world)
    gathered = [_host(s, stream)[0] for s in slabs]
    for r, g in enumerate(gathered):
        n = bounds[r + 1] - bounds[r]
        _assert_bitwise(g[:n], full[0, bounds[r]:bounds[r + 1]], "gather layout, world %d, rank %d" % (world, r))
        assert np.isnan(g[n:]).all(), "rank %d of %d wrote past its %d planes" % (r, world, n)
    _assert_bitwise(sharding.unpack_gather_list(gathered, R, world, np.empty((R, R, R), np.float32))[None], full,
                    "unpacked gather, world %d" % world)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_two_image_z_slabs_use_the_slab_stride(ctx, world):
    """B = 2: the slab is [B, z1-z0, R, R] with per-image stride (z1-z0)*R*R, equal to the host slab, and nothing is
    written past its end."""
    eng, stream = ctx
    imgs, tm, sp = _two_image_inputs()
    R = R_SLAB
    eng.set_precision("f16f8")
    with torch.cuda.stream(stream):
        img_d, tm_d = _dev(imgs), _dev(tm)
        eng.encode_device(img_d.data_ptr(), 2, 137, 137, 3)
    for r in range(world):
        z0, z1 = sharding.slab(R, world, r)
        n = 2 * (z1 - z0) * R * R
        with torch.cuda.stream(stream):
            buf = _nan((n + GUARD,))
            eng.eval_grid_device(sp, tm_d.data_ptr(), RES_SLAB, z0, z1, buf.data_ptr())
        got = _host(buf, stream)
        want = eng.eval_grid(sp, tm, RES_SLAB, z0=z0, z1=z1)
        assert np.isnan(got[n:]).all(), "rank %d of %d wrote past its slab" % (r, world)
        _assert_bitwise(got[:n].reshape(2, z1 - z0, R, R), want, "B=2 slab [%d, %d), world %d" % (z0, z1, world))


# ---- 4. explicit points on the device path --------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 63, 64, 65, 4099])
def test_eval_points_device_equals_host(ctx, n):
    """eval_points_device (B = 2, pts_rot != pts, uv out) == eval_points(pts, tm, pts_rot, want_uv=True), bitwise; also
    with pts_rot_ptr == pts_ptr and with pts_rot_ptr = 0 (both mean "rotated points = points")."""
    eng, stream = ctx
    rng = np.random.default_rng(4400 + n)
    pts = rng.uniform(-1.3, 1.3, size=(2, n, 3)).astype(np.float32)         # some project outside the image: clamped
    rot = rng.uniform(-1, 1, size=(2, n, 3)).astype(np.float32)
    tm = synth.synthetic_trans_mats(2, seed=4500 + n)
    imgs = synth.synthetic_images(2, seed=4600 + n)
    for precision in ("fp32", "bf16x3", "f16f8"):
        eng.set_precision(precision)
        with torch.cuda.stream(stream):
            img_d, pts_d, rot_d, tm_d = _dev(imgs), _dev(pts), _dev(rot), _dev(tm)
            eng.encode_device(img_d.data_ptr(), 2, 137, 137, 3)
            outs = {k: (_nan((2, n, 1)), _nan((2, n, 2))) for k in ("rot", "same", "none")}
            for k, rp in (("rot", rot_d.data_ptr()), ("same", pts_d.data_ptr()), ("none", 0)):
                pred_d, uv_d = outs[k]
                eng.eval_points_device(pts_d.data_ptr(), tm_d.data_ptr(), 2, n, pred_d.data_ptr(), uv_d.data_ptr(), rp)
        want = {"rot": eng.eval_points(pts, tm, rot, want_uv=True), "same": eng.eval_points(pts, tm, want_uv=True)}
        want["none"] = want["same"]
        for k, (pred_d, uv_d) in outs.items():
            _assert_bitwise(_host(pred_d, stream), want[k][0], "pred, N=%d, %s, pts_rot %s" % (n, precision, k))
            _assert_bitwise(_host(uv_d, stream), want[k][1], "uv, N=%d, %s, pts_rot %s" % (n, precision, k))
        assert not np.array_equal(want["rot"][0], want["same"][0])        # pts_rot really changes the prediction


# ---- 5. the caller's stream is really used --------------------------------------------------------------------------------
def test_kernels_run_on_the_callers_stream(ctx):
    """On stream S: a ~0.1 s GPU sleep, out.fill_(NaN), eval_grid_device(out), clone.  Had the library launched on any
    stream other than S, its kernel would finish during the sleep and the fill would leave NaN.  The stream must still be
    busy when the library call returns (it did not synchronise S).  Then the same on a second torch stream, then on the
    engine's own stream again; last, encode A / grid / encode B / grid back to back without a host synchronisation."""
    eng, stream = ctx
    res, R = 64, 65
    tm, sp = synth.DEMO_TRANS_MAT, synth.DEMO_SDF_PARAMS
    img_a, img_b = synth.synthetic_images(1, seed=5100), synth.synthetic_images(1, seed=5200)
    eng.set_precision("f16f8")
    eng.encode(img_b)
    want_b = eng.eval_grid(sp, tm, res)
    eng.encode(img_a)
    want_a = eng.eval_grid(sp, tm, res)        # also leaves this box's axis tables resident: no upload below
    with torch.cuda.stream(stream):
        a_d, b_d, tm_d, warm = _dev(img_a), _dev(img_b), _dev(tm), _nan((1, R, R, R))
        for _ in range(3):                     # the device-path calls below only replay and launch
            eng.encode_device(a_d.data_ptr(), 1, 137, 137, 3)
            eng.eval_grid_device(sp, tm_d.data_ptr(), res, 0, R, warm.data_ptr())
    stream.synchronize()

    def sleep_fill_eval(s):
        with torch.cuda.stream(s):
            out = torch.empty((1, R, R, R), dtype=torch.float32, device=DEV)
            torch.cuda._sleep(SLEEP_CYCLES)
            out.fill_(NAN)
            eng.eval_grid_device(sp, tm_d.data_ptr(), res, 0, R, out.data_ptr())
            busy = not s.query()
            got = out.clone()
            return busy, got.cpu().numpy()

    busy, got = sleep_fill_eval(stream)
    assert busy, "the sleep had ended when eval_grid_device returned: the library synchronised the caller's stream"
    _assert_bitwise(got, want_a, "grid on the caller's stream")
    other = torch.cuda.Stream(DEV)
    try:
        eng.set_stream(other.cuda_stream)
        busy, got = sleep_fill_eval(other)
        assert busy
        _assert_bitwise(got, want_a, "grid on a second caller stream")
        eng.set_stream(None)                   # back to the context's own stream
        with torch.cuda.stream(stream):
            out = _nan((1, R, R, R))
        stream.synchronize()
        eng.eval_grid_device(sp, tm_d.data_ptr(), res, 0, R, out.data_ptr())
        eng.synchronize()
        _assert_bitwise(_host(out, stream), want_a, "grid on the engine's own stream")
    finally:
        eng.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):
        buf1, buf2 = _nan((1, R, R, R)), _nan((1, R, R, R))
        torch.cuda._sleep(SLEEP_CYCLES)
        eng.encode_device(a_d.data_ptr(), 1, 137, 137, 3)
        eng.eval_grid_device(sp, tm_d.data_ptr(), res, 0, R, buf1.data_ptr())
        eng.encode_device(b_d.data_ptr(), 1, 137, 137, 3)
        eng.eval_grid_device(sp, tm_d.data_ptr(), res, 0, R, buf2.data_ptr())
        busy = not stream.query()
    stream.synchronize()
    assert busy, "a device-path call synchronised the caller's stream"
    _assert_bitwise(_host(buf1, stream), want_a, "back to back, image A")
    _assert_bitwise(_host(buf2, stream), want_b, "back to back, image B")


# ---- 6. asynchronous status -------------------------------------------------------------------------------------------------
def _scaled_heads(W, s):
    """Same function, internal activations of both point MLPs scaled by s: W1,b1 and every later bias (and the
    image-feature rows of fold2/conv1) times s, the linear output layer's weights times 1/s (as in test_gpu_configs.py)."""
    out = dict(W)
    for scope in ("sdfprediction", "sdfprediction_imgfeat"):
        g = lambda n: np.asarray(W["%s/%s" % (scope, n)], np.float64)
        out["%s/fold1/conv1/weights" % scope] = (g("fold1/conv1/weights") * s).astype(np.float32)
        for l in ("fold1/conv1", "fold1/conv2", "fold1/conv3", "fold2/conv1", "fold2/conv2"):
            out["%s/%s/biases" % (scope, l)] = (g(l + "/biases") * s).astype(np.float32)
        w = g("fold2/conv1/weights").copy()
        w[..., 512:, :] *= s                      # rows fed by the (unscaled) image features
        out["%s/fold2/conv1/weights" % scope] = w.astype(np.float32)
        out["%s/fold2/conv5/weights" % scope] = (g("fold2/conv5/weights") / s).astype(np.float32)
    return out


def test_device_path_status_is_reported_at_the_next_synchronise(he_weights):
    """f16f8 activations beyond the fp16 range: eval_grid_device / eval_points_device return, the next synchronize()
    raises "fp16 range"; afterwards bf16x3 on the same weights and f16f8 on normal weights succeed, equal the host path,
    and synchronize() stays quiet (the status does not stick).  Mis-shaped calls raise before launching anything."""
    from disn_b200._lib import DisnError
    res, R, n = 16, 17, 500
    imgs = synth.synthetic_images(1, seed=6100)
    tm, sp = synth.DEMO_TRANS_MAT, synth.DEMO_SDF_PARAMS
    pts = np.random.default_rng(6200).uniform(-1, 1, size=(1, n, 3)).astype(np.float32)
    with _engine(_scaled_heads(he_weights, 2.0 ** 17), "f16f8", max_batch=2) as (eng, stream):
        with torch.cuda.stream(stream):
            img_d, tm_d, pts_d = _dev(imgs), _dev(tm), _dev(pts)
            grid_d, pred_d = _nan((1, R, R, R)), _nan((1, n, 1))
            eng.encode_device(img_d.data_ptr(), 1, 137, 137, 3)
            eng.eval_grid_device(sp, tm_d.data_ptr(), res, 0, R, grid_d.data_ptr())
            eng.eval_points_device(pts_d.data_ptr(), tm_d.data_ptr(), 1, n, pred_d.data_ptr())
        with pytest.raises(DisnError, match="fp16 range"):
            eng.synchronize()
        eng.synchronize()

        for precision, weights in (("bf16x3", None), ("f16f8", he_weights)):
            eng.set_precision(precision)
            if weights is not None:
                eng.load_weights(weights)
            with torch.cuda.stream(stream):
                eng.encode_device(img_d.data_ptr(), 1, 137, 137, 3)
                eng.eval_grid_device(sp, tm_d.data_ptr(), res, 0, R, grid_d.data_ptr())
                eng.eval_points_device(pts_d.data_ptr(), tm_d.data_ptr(), 1, n, pred_d.data_ptr())
            eng.synchronize()
            _assert_bitwise(_host(grid_d, stream), eng.eval_grid(sp, tm, res), "grid after the overflow, " + precision)
            _assert_bitwise(_host(pred_d, stream), eng.eval_points(pts, tm), "points after the overflow, " + precision)
            eng.synchronize()

        before, launches = _host(grid_d, stream), eng.launch_count
        sp2, tm2_d = np.repeat(sp, 2, 0), _dev(np.repeat(tm, 2, 0))
        with pytest.raises(DisnError, match="batch differs"):
            eng.eval_grid_device(sp2, tm2_d.data_ptr(), res, 0, R, grid_d.data_ptr())
        with pytest.raises(DisnError, match="batch differs"):
            eng.eval_points_device(pts_d.data_ptr(), tm2_d.data_ptr(), 2, n // 2, pred_d.data_ptr())
        for z0, z1 in ((0, R + 1), (-1, 5), (9, 4)):
            with pytest.raises(DisnError, match="z range"):
                eng.eval_grid_device(sp, tm_d.data_ptr(), res, z0, z1, grid_d.data_ptr())
        assert eng.launch_count == launches
        eng.synchronize()
        _assert_bitwise(_host(grid_d, stream), before, "output after the refused calls")


# ---- 7. config 4's tail on device memory ------------------------------------------------------------------------------------
def test_config4_marching_cubes_of_the_device_grid(ctx):
    """bench.py config 4: the f16f8 513³ grid from eval_grid_device, meshed in place (marching_cubes with device_ptr) ==
    the mesh of the host grid passed as a host array, vertices and faces bit for bit, at iso 0 and at the bench's iso (the
    median of the field)."""
    eng, stream = ctx
    imgs, tm, sp, _ = _config_inputs(1)
    res, R = 512, 513
    eng.set_precision("f16f8")
    with torch.cuda.stream(stream):
        img_d, tm_d, grid_d = _dev(imgs), _dev(tm), _nan((R, R, R))
        eng.encode_device(img_d.data_ptr(), 1, 137, 137, 3)
        eng.eval_grid_device(sp, tm_d.data_ptr(), res, 0, R, grid_d.data_ptr())
        iso_med = float(grid_d.median().item())
    host = eng.eval_grid(sp, tm, res)[0]
    _assert_bitwise(_host(grid_d, stream), host, "513³ grid")
    faces = {}
    for iso in (0.0, iso_med):
        vd, fd = eng.marching_cubes(None, sp[0], iso, device_ptr=grid_d.data_ptr(), R=R)
        vh, fh = eng.marching_cubes(host, sp[0], iso)
        _assert_bitwise(vd, vh, "mesh vertices, iso %g" % iso)
        np.testing.assert_array_equal(fd, fh, err_msg="mesh faces, iso %g" % iso)
        faces[iso] = len(fh)
    assert faces[iso_med] > 1000, faces


# ---- 8. the peer-store gather across processes --------------------------------------------------------------------------------
RES_PEER = 128
PEER_TIMEOUT_S = 600


def _peer_rank(rank, world, handles, reports):
    """One rank of the peer-store gather in its own process: open rank 0's buffer, encode the image, store this rank's
    z-slab into it with eval_grid_device, synchronise, unmap, report."""
    try:
        from disn_b200.engine import Engine
        R = RES_PEER + 1
        device = rank % torch.cuda.device_count()
        imgs, tm, sp, _ = _config_inputs(1)
        stream = torch.cuda.Stream(torch.device("cuda", device))
        eng = Engine(device=device, precision="f16f8", max_batch=1)
        try:
            eng.set_stream(stream.cuda_stream)
            try:
                eng.load_weights(synth.make_weights(seed=7, init="he"))
                ptr = eng.shared_open(handles.get(timeout=PEER_TIMEOUT_S))
                try:
                    with torch.cuda.stream(stream):
                        img_d = torch.from_numpy(imgs).to(stream.device)
                        tm_d = torch.from_numpy(tm).to(stream.device)
                        eng.encode_device(img_d.data_ptr(), 1, 137, 137, 3)
                        z0, z1 = sharding.slab(R, world, rank)
                        eng.eval_grid_device(sp, tm_d.data_ptr(), RES_PEER, z0, z1, ptr + z0 * R * R * 4)
                    eng.synchronize()
                finally:
                    eng.shared_close(ptr, owner=False)
            finally:
                eng.set_stream(None)
        finally:
            eng.close()
        reports.put((rank, None))
    except BaseException as e:          # reported to rank 0, which fails the test with it
        reports.put((rank, "%s: %s" % (type(e).__name__, e)))


class _DeviceArray:
    """A raw device float32 buffer as a torch tensor (__cuda_array_interface__), to fill it from torch."""
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "strides": None,
                                        "version": 2}


@pytest.fixture(scope="module")
def spawn():
    """multiprocessing's spawn context.  Spawning also starts multiprocessing's resource tracker, a child of this process
    that would outlive the test run; it is stopped and waited for when the module ends."""
    yield multiprocessing.get_context("spawn")
    gc.collect()                # the ranks' queues unregister their semaphores while the tracker still runs
    from multiprocessing import resource_tracker
    stop = getattr(resource_tracker._resource_tracker, "_stop", None)
    if stop is not None:
        stop()


@pytest.mark.parametrize("world", [2, 3])
def test_peer_store_gather_across_processes(ctx, spawn, world):
    """bench.py's multi-GPU gather without NCCL: rank 0 (this process) shared_alloc's the R³ grid (R = 129) and sends the
    IPC handle to `world - 1` spawned ranks (device rank % device_count); each stores its z-slab into it with
    eval_grid_device.  The fetched buffer must equal this process's own single-process grid bitwise."""
    eng, stream = ctx
    imgs, tm, sp, _ = _config_inputs(1)
    R = RES_PEER + 1
    eng.set_precision("f16f8")
    eng.encode(imgs)
    want = eng.eval_grid(sp, tm, RES_PEER)
    ptr, handle = eng.shared_alloc(R ** 3 * 4)
    handles, reports = spawn.Queue(), spawn.Queue()
    procs = [spawn.Process(target=_peer_rank, args=(r, world, handles, reports), daemon=True) for r in range(1, world)]
    try:
        with torch.cuda.stream(stream):
            torch.as_tensor(_DeviceArray(ptr, R ** 3), device=DEV).fill_(NAN)
        stream.synchronize()
        for p in procs:
            p.start()
        for _ in procs:
            handles.put(handle)
        with torch.cuda.stream(stream):
            img_d, tm_d = _dev(imgs), _dev(tm)
            eng.encode_device(img_d.data_ptr(), 1, 137, 137, 3)
            z0, z1 = sharding.slab(R, world, 0)
            eng.eval_grid_device(sp, tm_d.data_ptr(), RES_PEER, z0, z1, ptr + z0 * R * R * 4)
        eng.synchronize()
        errors, done, deadline, silent_since = [], set(), time.monotonic() + PEER_TIMEOUT_S, None
        while len(done) < len(procs):
            try:
                rank, err = reports.get(timeout=1.0)
            except queue.Empty:
                now = time.monotonic()
                silent = [r for r, p in enumerate(procs, 1) if p.exitcode is not None and r not in done]
                silent_since = (silent_since or now) if silent else None
                if now > deadline or (silent and now - silent_since > 10.0):     # a report may still be in the pipe
                    pytest.fail("ranks %s did not report within %s s (exit codes %s)" % (
                        sorted(set(range(1, world)) - done), PEER_TIMEOUT_S if now > deadline else 10,
                        [p.exitcode for p in procs]))
                continue
            done.add(rank)
            if err:
                errors.append("rank %d: %s" % (rank, err))
        assert not errors, "; ".join(errors)
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0, (p.name, p.exitcode)
        got = eng.fetch(ptr, (1, R, R, R))
        _assert_bitwise(got, want, "peer-store gather, world %d" % world)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
            if p.pid is not None:
                p.join(timeout=30)
        eng.shared_close(ptr, owner=True)
