"""GPU tests of the indexed grid evaluation and the coarse-to-fine grid (DESIGN.md §4.9): indexed values equal the dense
grid bit for bit, the device refinement equals its numpy twin oracle/adaptive_oracle.py on the dense device grid, the
adaptive mesh of exact distance fields equals the dense mesh, large grids, and the argument checks."""
import ctypes as C

import numpy as np
import pytest

from disn_b200 import _lib, synth
from disn_b200._lib import DISN_DEVICE_PTR, DisnError
from disn_b200.engine import Engine
from oracle import adaptive_oracle as ao
from tests.test_mesh_sdf_cpu import analytic_mesh

pytestmark = pytest.mark.gpu

PRECS = ("fp32", "bf16x3", "f16f8")
BOX = [-1.0, -1.0, -1.0, 1.0, 1.0, 1.0]
BOXES = np.array([BOX, [-0.8, -0.9, -1.0, 0.9, 1.0, 0.7]], np.float64)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(seed=7, init="he")


@pytest.fixture(scope="module")
def demo_img(golden):
    return (golden["demo_input"]["img_u8"].astype(np.float32) / np.float32(255.))[None]


@pytest.fixture(scope="module")
def engines(weights):
    made = {}

    def get(prec):
        if prec not in made:
            eng = Engine(device=0, precision=prec, max_batch=2)
            eng.load_weights(weights)
            made[prec] = eng
        return made[prec]
    yield get
    for eng in made.values():
        eng.close()


def diag(fn, *args):
    lib = _lib.load_test()
    rc = getattr(lib, fn)(*args)
    if rc != 0:
        raise DisnError("%s (rc=%d)" % (lib.disn_last_error().decode("utf-8", "replace"), rc))


def adaptive_mask(eng, first, n):
    out = np.empty(n, np.uint8)
    diag("disn_adaptive_mask", eng._h, first, n, out.ctypes.data_as(C.c_void_p))
    return out.astype(bool)


def median_iso(eng, res=64):
    """The synthetic He-weight network need not cross 0: mesh at the median of its grid, as bench.py does."""
    return float(np.median(eng.eval_grid(BOX, synth.DEMO_TRANS_MAT, res)))


def adaptive_from_field(eng, field_ptr, res, box, iso=0.0, band=1.0):
    bb = (C.c_double * 6)(*box)
    grid = C.c_void_p()
    counts = np.zeros(5, np.int64)
    nl = C.c_int32(0)
    diag("disn_adaptive_from_field", eng._h, C.c_void_p(field_ptr), res, bb, float(iso), float(band), DISN_DEVICE_PTR,
         C.byref(grid), counts.ctypes.data_as(C.c_void_p), C.byref(nl))
    return int(grid.value), [int(v) for v in counts[:nl.value]]


# ---- 1. indexed evaluation == dense evaluation, bit for bit ----------------------------------------------------------
@pytest.mark.parametrize("res", [64, 256])
@pytest.mark.parametrize("prec", PRECS)
def test_indexed_equals_dense(engines, prec, res):
    eng = engines(prec)
    tm = synth.synthetic_trans_mats(2)
    eng.encode(synth.synthetic_images(2))
    R = res + 1
    dense = eng.eval_grid(BOXES, tm, res).reshape(2, -1)
    rng = np.random.default_rng(res)
    subsets = [rng.choice(R ** 3, 100_003, replace=False), rng.choice(R ** 3, 77, replace=False),
               np.array([R ** 3 - 1, 0, R ** 3 - 1], np.int64)]
    if res == 64:
        subsets.append(rng.permutation(R ** 3))                # every point, shuffled
    for image in (0, 1):
        for idx in subsets:
            got = eng.eval_grid_indexed(BOXES[image], tm[image], res, idx, image=image)
            np.testing.assert_array_equal(bits(got), bits(dense[image][idx]))


# ---- 2. the device refinement == the numpy twin on the dense device grid ---------------------------------------------
@pytest.mark.parametrize("res", [128, 256])
@pytest.mark.parametrize("prec", ["fp32", "f16f8"])
def test_refinement_equals_oracle(engines, demo_img, prec, res):
    eng = engines(prec)
    eng.encode(demo_img)
    R = res + 1
    dense = eng.eval_grid(BOX, synth.DEMO_TRANS_MAT, res)[0]
    iso = float(np.median(dense))
    ptr, counts = eng.eval_grid_adaptive(BOX, synth.DEMO_TRANS_MAT[0], res, iso=iso, band=1.0)
    grid = eng.fetch(ptr, (R, R, R))
    mask = adaptive_mask(eng, 0, R ** 3).reshape(R, R, R)
    want_mask, want_counts, want = ao.refine(dense, BOX, iso=iso, band=1.0)
    assert counts == want_counts and sum(counts) < R ** 3
    np.testing.assert_array_equal(mask, want_mask)
    np.testing.assert_array_equal(bits(grid), bits(want))
    nv, nf = eng.marching_cubes(None, BOX, iso, device_ptr=ptr, R=R, fetch=False)
    assert nv > 0 and nf > 0


# ---- 3. exact distance fields: the adaptive mesh is the dense mesh -----------------------------------------------------
@pytest.mark.parametrize("kind", ["torus", "sphere"])
def test_mesh_sdf_fields_mesh_identical(engines, kind):
    eng = engines("fp32")
    res, R = 256, 257
    v, f = analytic_mesh(kind, 15)
    field = eng.field_buffer(R)
    eng.mesh_sdf(res, bbox=BOX, verts=v, faces=f, device_ptr=field)
    dense = eng.marching_cubes(None, BOX, 0.0, device_ptr=field, R=R)
    ptr, counts = adaptive_from_field(eng, field, res, BOX, iso=0.0, band=1.0)
    assert sum(counts) < R ** 3 // 4
    got = eng.marching_cubes(None, BOX, 0.0, device_ptr=ptr, R=R)
    assert len(dense[1]) > 0
    np.testing.assert_array_equal(bits(got[0]), bits(dense[0]))
    np.testing.assert_array_equal(got[1], dense[1])
    mask = adaptive_mask(eng, 0, R ** 3)
    np.testing.assert_array_equal(bits(eng.fetch(ptr, (R ** 3,))[mask]), bits(eng.fetch(field, (R ** 3,))[mask]))


# ---- 4. res 512 and 1024 ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("res", [512, 1024])
def test_large_grids_match_dense_slabs(engines, demo_img, res):
    eng = engines("f16f8")
    eng.encode(demo_img)
    R = res + 1
    iso = median_iso(eng)
    ptr, counts = eng.eval_grid_adaptive(BOX, synth.DEMO_TRANS_MAT[0], res, iso=iso)
    assert len(counts) == 5 and sum(counts) < R ** 3
    for z0 in (0, R // 2 - 4, R - 8):
        dense = eng.eval_grid(BOX, synth.DEMO_TRANS_MAT, res, z0, z0 + 8)[0].reshape(-1)
        got = eng.fetch(ptr + z0 * R * R * 4, (8 * R * R,))
        mask = adaptive_mask(eng, z0 * R * R, 8 * R * R)
        assert mask.any()
        np.testing.assert_array_equal(bits(got[mask]), bits(dense[mask]))
    nv, nf = eng.marching_cubes(None, BOX, iso, device_ptr=ptr, R=R, fetch=False)
    assert nv > 0 and nf > 0


# ---- 5. argument checks -------------------------------------------------------------------------------------------------
def test_errors(weights, engines, demo_img):
    fresh = Engine(device=0, precision="fp32")
    try:
        fresh.load_weights(weights)
        with pytest.raises(DisnError, match="disn_encode"):
            fresh.eval_grid_adaptive(BOX, synth.DEMO_TRANS_MAT[0], 16)
        with pytest.raises(DisnError, match="disn_encode"):
            fresh.eval_grid_indexed(BOX, synth.DEMO_TRANS_MAT[0], 16, [0, 1])
    finally:
        fresh.close()
    eng = engines("fp32")
    eng.encode(demo_img)
    tm = synth.DEMO_TRANS_MAT[0]
    for image in (1, -1):
        with pytest.raises(DisnError, match="image outside"):
            eng.eval_grid_adaptive(BOX, tm, 16, image=image)
        with pytest.raises(DisnError, match="image outside"):
            eng.eval_grid_indexed(BOX, tm, 16, [0], image=image)
    for res in (0, -3):
        with pytest.raises(DisnError, match="sdf_res"):
            eng.eval_grid_adaptive(BOX, tm, res)
        with pytest.raises(DisnError, match="sdf_res"):
            eng.eval_grid_indexed(BOX, tm, res, [0])
    for iso in (np.nan, np.inf, -np.inf):
        with pytest.raises(DisnError, match="iso"):
            eng.eval_grid_adaptive(BOX, tm, 16, iso=iso)
    for band in (np.nan, -1.0, -np.inf):
        with pytest.raises(DisnError, match="band"):
            eng.eval_grid_adaptive(BOX, tm, 16, band=band)
    with pytest.raises(DisnError, match="outside"):
        eng.eval_grid_indexed(BOX, tm, 16, [0, 17 ** 3])
    # device indices are checked on the device: the call returns, the next synchronize() reports the bad index
    import torch
    d_idx = torch.tensor([0, 17 ** 3, 5], dtype=torch.int32, device="cuda:0")
    d_tm = torch.from_numpy(np.ascontiguousarray(tm, np.float32)).to("cuda:0")
    d_out = torch.empty(3, dtype=torch.float32, device="cuda:0")
    torch.cuda.synchronize()
    eng.eval_grid_indexed_device(BOX, d_tm.data_ptr(), 16, d_idx.data_ptr(), 3, d_out.data_ptr())
    with pytest.raises(DisnError, match="outside"):
        eng.synchronize()
    # band = +inf is valid and gives the dense grid; the context is still usable after the errors
    R = 65
    ptr, counts = eng.eval_grid_adaptive(BOX, tm, 64, band=np.inf)
    assert sum(counts) == R ** 3 and adaptive_mask(eng, 0, R ** 3).all()
    np.testing.assert_array_equal(bits(eng.fetch(ptr, (R, R, R))), bits(eng.eval_grid(BOX, synth.DEMO_TRANS_MAT, 64)[0]))
    # a resolution no power of two divides: one level, the dense grid
    ptr, counts = eng.eval_grid_adaptive(BOX, tm, 63)
    assert counts == [64 ** 3]
    np.testing.assert_array_equal(bits(eng.fetch(ptr, (64, 64, 64))), bits(eng.eval_grid(BOX, synth.DEMO_TRANS_MAT, 63)[0]))


# ---- the driver flag ----------------------------------------------------------------------------------------------------
def test_driver_adaptive_flag(weights, engines, demo_img, tmp_path):
    """FLAGS.adaptive: same output name; band = inf writes the dense run's OBJ byte for byte, band 1 a non-empty mesh."""
    from disn_b200 import create_sdf as drv
    batch = {"img": demo_img, "trans_mat": synth.DEMO_TRANS_MAT.copy(),
             "sdf_params": np.asarray(synth.DEMO_SDF_PARAMS, np.float64).reshape(1, 6).copy(),
             "cat_id": ["demo"], "obj_nm": ["obj"], "view_id": [0]}
    eng = engines("fp32")
    eng.encode(demo_img)
    iso = median_iso(eng)
    objs = {}
    for name, kw in (("dense", {}), ("band_inf", {"adaptive": True, "adaptive_band": float("inf")}),
                     ("band_1", {"adaptive": True})):
        drv.configure(drv.default_flags(sdf_res=64, iso=iso, log_dir=str(tmp_path / name), precision="fp32", **kw))
        (path,) = drv.create(weights, [batch])
        assert path.endswith("demo_obj_00.obj")
        with open(path, "rb") as fh:
            objs[name] = fh.read()
    assert objs["band_inf"] == objs["dense"]
    assert b"\nf " in objs["band_1"]
