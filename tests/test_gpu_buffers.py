"""GPU tests of buffer ownership on one context: a call that grows one persistent buffer must leave every other buffer
intact, a buffer that grew and is reused must give the same results, and contexts are destroyed cleanly.  Each test
builds its own Engine, because what is tested is the order of calls on one context."""
import numpy as np
import pytest

from disn_b200 import synth
from disn_b200.engine import Engine

pytestmark = pytest.mark.gpu

BOX = [-1, -1, -1, 1, 1, 1]


@pytest.fixture
def eng(he_weights):
    e = Engine(device=0, precision="fp32")
    e.load_weights(he_weights)
    e.encode(synth.synthetic_images(1))
    yield e
    e.close()


def _pts(n, seed=0, batch=1):
    return np.random.default_rng(seed).uniform(-1, 1, (batch, n, 3)).astype(np.float32)


def _same(a, b):
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


def test_decoder_entry_points_survive_a_larger_nn_distance(eng):
    """eval_points_ex / point_img_feat / eval_features stage through the decoder scratch; a first, large nn_distance
    grows the nn scratch and must not release or overwrite it."""
    tm = synth.DEMO_TRANS_MAT
    pts = _pts(1000)
    rng = np.random.default_rng(1)
    gfeat = rng.standard_normal((1, 1024)).astype(np.float32)
    pfeat = rng.standard_normal((1, 1000, 1472)).astype(np.float32)

    def decoder_calls():
        return eng.eval_points_ex(pts, tm), eng.point_img_feat(pts, tm), eng.eval_features(pts, gfeat, pfeat)

    before = decoder_calls()
    d1, i1, d2, i2 = eng.nn_distance(_pts(4096, 2, batch=2), _pts(4096, 3, batch=2))
    assert d1.shape == (2, 4096) and np.isfinite(d1).all() and np.isfinite(d2).all()
    after = decoder_calls()
    for b, a in zip(before, after):
        _same(b, a)


def test_eval_points_grow_then_reuse(eng):
    tm = synth.DEMO_TRANS_MAT
    small = _pts(10)
    first = eng.eval_points(small, tm, want_uv=True)
    big = eng.eval_points(_pts(100_000, 5), tm)
    assert big.shape == (1, 100_000, 1) and np.isfinite(big).all()
    _same(first, eng.eval_points(small, tm, want_uv=True))


def test_eval_grid_grow_then_reuse(eng):
    tm = synth.DEMO_TRANS_MAT
    first = eng.eval_grid(synth.DEMO_SDF_PARAMS, tm, 16)
    big = eng.eval_grid(synth.DEMO_SDF_PARAMS, tm, 64)
    assert big.shape == (1, 65, 65, 65)
    np.testing.assert_array_equal(first, eng.eval_grid(synth.DEMO_SDF_PARAMS, tm, 16))


def test_marching_cubes_after_a_larger_clean(eng):
    small = eng.eval_grid(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 16)[0]
    iso = float(np.median(small))
    first = eng.marching_cubes(small, BOX, iso)
    noise = np.random.default_rng(7).standard_normal((65, 65, 65)).astype(np.float32)
    v, f = eng.marching_cubes(noise, BOX, 0.0)
    assert len(f) > 10 * len(first[1])
    eng.load_mesh(v, f)
    cv, cf = eng.clean_mesh(0.5, 0.0)
    assert 0 < len(cf) <= len(f)
    _same(first, eng.marching_cubes(small, BOX, iso))


def test_close_twice_and_a_second_context(he_weights):
    pts = _pts(300)
    e1 = Engine(device=0, precision="fp32")
    e1.load_weights(he_weights)
    e1.encode(synth.synthetic_images(1))
    want = e1.eval_points(pts, synth.DEMO_TRANS_MAT)
    e1.close()
    e1.close()
    e2 = Engine(device=0, precision="fp32")
    try:
        e2.load_weights(he_weights)
        e2.encode(synth.synthetic_images(1))
        np.testing.assert_array_equal(want, e2.eval_points(pts, synth.DEMO_TRANS_MAT))
    finally:
        e2.close()
