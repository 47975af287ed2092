"""GPU tests of the coarse-to-fine mesher (disn_mesh_grid_adaptive, DESIGN.md §4.10): on given fields and on the network in
all three precisions its mesh equals marching cubes of the dense adaptive grid bit for bit (vertices, faces, order, level
counts) and the numpy twin oracle/adaptive_mesh_oracle.py; cleaning and the driver's OBJ files are unchanged; res 2048
runs and its vertices recompute from the network; argument errors and the f16f8 overflow leave the context usable."""
import ctypes as C
import json

import numpy as np
import pytest

from disn_b200 import synth
from disn_b200._lib import DisnError
from disn_b200.engine import Engine
from oracle import adaptive_mesh_oracle as amo
from tests.test_adaptive_mesh_cpu import make_field
from tests.test_gpu_adaptive import BOX, bits, demo_img, diag, engines, median_iso, weights  # noqa: F401
from tests.test_mesh_sdf_cpu import analytic_mesh

pytestmark = pytest.mark.gpu


def from_field(eng, fn, F, res, box, iso, band, *out):
    """a diagnostic that reads host field F (staged by the library)"""
    a = np.ascontiguousarray(F, np.float32)
    diag(fn, eng._h, a.ctypes.data_as(C.c_void_p), res, (C.c_double * 6)(*box), float(iso), float(band), 0, *out)


def dense_from_field(eng, F, res, box, iso, band):
    """disn_adaptive_from_field + disn_mc_run: the dense adaptive grid's mesh and level counts"""
    grid = C.c_void_p()
    counts = np.zeros(5, np.int64)
    nl = C.c_int32(0)
    from_field(eng, "disn_adaptive_from_field", F, res, box, iso, band, C.byref(grid), counts.ctypes.data_as(C.c_void_p),
               C.byref(nl))
    v, f = eng.marching_cubes(None, box, iso, device_ptr=int(grid.value), R=res + 1)
    return v, f, [int(c) for c in counts[:nl.value]]


def mesh_from_field(eng, F, res, box, iso, band):
    counts = np.zeros(5, np.int64)
    nl = C.c_int32(0)
    nv, nf = C.c_int64(eng._mesh_verts), C.c_int64(eng._mesh_faces)
    try:
        from_field(eng, "disn_mesh_adaptive_from_field", F, res, box, iso, band, counts.ctypes.data_as(C.c_void_p),
                   C.byref(nl), C.byref(nv), C.byref(nf))
    finally:
        eng._mesh_verts, eng._mesh_faces = nv.value, nf.value
    v, f = eng.fetch_mesh()
    return v, f, [int(c) for c in counts[:nl.value]]


def same(a, b):
    assert a[0].shape == b[0].shape and a[1].shape == b[1].shape
    np.testing.assert_array_equal(bits(a[0]), bits(b[0]))
    np.testing.assert_array_equal(a[1], b[1])


# ---- 1. given fields: the mesher equals adaptive_from_field + mc_run, and the twin ------------------------------------
@pytest.mark.parametrize("res,kind,band", [(64, "noise", 0.5), (64, "smooth", 0.0), (64, "smooth", np.inf),
                                           (128, "noise", 1.0), (128, "smooth", 2.0), (256, "smooth", 1.0),
                                           (512, "smooth", 1.0), (96, "ties", 0.0), (96, "subnormal", 0.0)])
def test_from_field_equals_dense_path(engines, res, kind, band):
    eng = engines("fp32")
    R = res + 1
    F = make_field(kind, BOX, R, seed=res)
    iso = {"ties": 0.25, "subnormal": 0.0}.get(kind, float(np.median(F[::4, ::4, ::4])))
    want = dense_from_field(eng, F, res, BOX, iso, band)
    assert len(want[1]) > 0
    got = mesh_from_field(eng, F, res, BOX, iso, band)
    assert got[2] == want[2] and sum(got[2]) <= R ** 3
    same(got, want)
    if res <= 128:
        twin = amo.mesh(F, BOX, iso=iso, band=band)
        assert twin[2] == want[2]
        same(got, twin)


def test_exact_distance_field(engines):
    eng = engines("fp32")
    res, R = 256, 257
    v, f = analytic_mesh("torus", 15)
    F, _ = eng.mesh_sdf(res, bbox=BOX, verts=v, faces=f)
    want = dense_from_field(eng, F, res, BOX, 0.0, 1.0)
    got = mesh_from_field(eng, F, res, BOX, 0.0, 1.0)
    assert got[2] == want[2] and sum(got[2]) < R ** 3 // 4 and len(want[1]) > 0
    same(got, want)


# ---- 2. the network in every precision -----------------------------------------------------------------------------
@pytest.mark.parametrize("prec,res", [("fp32", 256), ("bf16x3", 256), ("f16f8", 256), ("f16f8", 512), ("f16f8", 1024)])
def test_network_equals_dense_path(engines, demo_img, prec, res):
    eng = engines(prec)
    eng.encode(demo_img)
    R = res + 1
    iso = median_iso(eng)
    tm = synth.DEMO_TRANS_MAT[0]
    grid, counts = eng.eval_grid_adaptive(BOX, tm, res, iso=iso)
    want = eng.marching_cubes(None, BOX, iso, device_ptr=grid, R=R)
    got = eng.mesh_grid_adaptive(BOX, tm, res, iso=iso)
    assert got[2] == counts and len(want[1]) > 0
    same(got, want)


def test_clean_and_driver_objs(weights, engines, demo_img, tmp_path, monkeypatch):
    eng = engines("fp32")
    eng.encode(demo_img)
    iso = median_iso(eng)
    tm = synth.DEMO_TRANS_MAT[0]
    grid, _ = eng.eval_grid_adaptive(BOX, tm, 128, iso=iso)
    eng.marching_cubes(None, BOX, iso, device_ptr=grid, R=129, fetch=False)
    want = eng.clean_mesh(0.5, 0.3)
    eng.mesh_grid_adaptive(BOX, tm, 128, iso=iso, fetch=False)
    same(eng.clean_mesh(0.5, 0.3), want)

    from disn_b200 import create_sdf as drv
    imgs = np.concatenate([demo_img, demo_img[:, ::-1].copy()])
    batch = {"img": imgs, "trans_mat": np.concatenate([synth.DEMO_TRANS_MAT] * 2),
             "sdf_params": np.asarray([synth.DEMO_SDF_PARAMS] * 2, np.float64).reshape(2, 6),
             "cat_id": ["demo", "demo"], "obj_nm": ["a", "b"], "view_id": [0, 1]}
    for res in (64, 128):
        for clean in (False, True):
            objs = {}
            for name, keep in (("grid", True), ("surface", False)):
                monkeypatch.setattr(drv, "SURFACE_MESH_MIN_RES", 1 if name == "surface" else 10 ** 9)
                drv.configure(drv.default_flags(sdf_res=res, iso=iso, log_dir=str(tmp_path / ("%s%d%d" % (name, res, clean))),
                                                precision="fp32", adaptive=True, keep_dist=keep, clean_smallparts=clean,
                                                batch_size=2))
                paths = drv.create(weights, [batch])
                assert len(paths) == 2
                objs[name] = [open(p, "rb").read() for p in paths]
            assert objs["grid"] == objs["surface"]
            assert all(b"\nf " in o for o in objs["surface"])


# ---- 3. res 2048 ---------------------------------------------------------------------------------------------------------
def test_res_2048_vertices_recompute(engines, demo_img):
    eng = engines("f16f8")
    eng.encode(demo_img)
    res, R = 2048, 2049
    iso = median_iso(eng)
    tm = synth.DEMO_TRANS_MAT[0]
    (nv, nf), counts = eng.mesh_grid_adaptive(BOX, tm, res, iso=iso, fetch=False)
    held = C.c_int64(0)
    diag("disn_mesh_adaptive_bytes", eng._h, C.byref(held))
    ms = np.zeros(3, np.float32)
    diag("disn_mesh_adaptive_phase_ms", eng._h, ms.ctypes.data_as(C.c_void_p))
    info = {"res": res, "level_counts": counts, "evaluated": sum(counts), "verts": nv, "faces": nf,
            "bytes_held": held.value, "phase_ms": [float(m) for m in ms]}
    print("res 2048:", json.dumps(info))
    assert len(counts) == 5 and nv > 0 and nf > 0
    verts, faces = eng.fetch_mesh()
    rng = np.random.default_rng(2048)
    sel = np.sort(rng.choice(nv, 10_000, replace=False))
    edges = np.empty(nv, np.int64)
    diag("disn_mesh_adaptive_edges", eng._h, 0, nv, edges.ctypes.data_as(C.c_void_p))
    assert (np.diff(edges) > 0).all()
    e = edges[sel]
    a, q = e % 3, e // 3
    idx = np.stack([q % R, (q // R) % R, q // (R * R)], axis=1)
    idx1 = idx + np.eye(3, dtype=np.int64)[a]
    ax = [np.linspace(BOX[k], BOX[3 + k], num=R).astype(np.float32) for k in range(3)]
    pts = np.concatenate([np.stack([ax[k][i[:, k]] for k in range(3)], axis=1) for i in (idx, idx1)])[None]
    pred = eng.eval_points(pts, synth.DEMO_TRANS_MAT).reshape(-1).astype(np.float32) / np.float32(10)
    v0, v1 = pred[:len(sel)], pred[len(sel):]
    iso32 = np.float32(iso)
    assert ((v0 < iso32) != (v1 < iso32)).all()
    lo = np.asarray(BOX[:3], np.float64)
    h = (np.asarray(BOX[3:], np.float64) - lo) / np.float64(R - 1)
    t = (np.float64(iso32) - v0.astype(np.float64)) / (v1.astype(np.float64) - v0.astype(np.float64))
    pos = lo[None, :] + idx.astype(np.float64) * h[None, :]
    rows = np.arange(len(sel))
    pos[rows, a] = pos[rows, a] + t * h[a]
    np.testing.assert_array_equal(bits(pos.astype(np.float32)), bits(verts[sel]))


# ---- 4. errors ------------------------------------------------------------------------------------------------------------
def test_errors_leave_context_usable(weights, engines, demo_img, tmp_path):
    from tests.test_gpu_configs import _scaled_heads
    eng = engines("fp32")
    eng.encode(demo_img)
    tm = synth.DEMO_TRANS_MAT[0]
    for image in (1, -1):
        with pytest.raises(DisnError, match="image outside"):
            eng.mesh_grid_adaptive(BOX, tm, 16, image=image)
    for res in (0, -3, 2049, 4096):
        with pytest.raises(DisnError, match="sdf_res"):
            eng.mesh_grid_adaptive(BOX, tm, res)
    with pytest.raises(DisnError, match="sdf_res"):       # odd: the dense grid, beyond its size limit
        eng.mesh_grid_adaptive(BOX, tm, 1291)
    for iso in (np.nan, np.inf):
        with pytest.raises(DisnError, match="iso"):
            eng.mesh_grid_adaptive(BOX, tm, 16, iso=iso)
    for band in (np.nan, -1.0):
        with pytest.raises(DisnError, match="band"):
            eng.mesh_grid_adaptive(BOX, tm, 16, band=band)
    # odd res: the dense grid, as eval_grid_adaptive + marching cubes
    iso = median_iso(eng)
    grid, counts = eng.eval_grid_adaptive(BOX, tm, 63, iso=iso)
    want = eng.marching_cubes(None, BOX, iso, device_ptr=grid, R=64)
    eng.mesh_grid_adaptive(BOX, tm, 64, iso=iso, fetch=False)
    ms = np.zeros(3, np.float32)
    diag("disn_mesh_adaptive_phase_ms", eng._h, ms.ctypes.data_as(C.c_void_p))
    got = eng.mesh_grid_adaptive(BOX, tm, 63, iso=iso)
    assert got[2] == counts == [64 ** 3]
    same(got, want)
    # the odd-res call ran no surface mesher: its diagnostics refuse instead of describing the previous call
    with pytest.raises(DisnError, match="no coarse-to-fine mesh"):
        diag("disn_mesh_adaptive_phase_ms", eng._h, ms.ctypes.data_as(C.c_void_p))
    with pytest.raises(DisnError, match="no coarse-to-fine mesh"):
        diag("disn_mesh_adaptive_edges", eng._h, 0, 1, np.zeros(1, np.int64).ctypes.data_as(C.c_void_p))
    # f16f8 overflow is loud, empties the resident mesh in the library and in Python alike, and does not stick
    fresh = Engine(device=0, precision="f16f8")
    try:
        fresh.load_weights(weights)
        fresh.encode(demo_img)
        small = fresh.mesh_grid_adaptive(BOX, tm, 16, iso=median_iso(fresh))
        assert len(small[1]) > 0
        fresh.load_weights(_scaled_heads(weights, 2.0 ** 17))
        fresh.encode(demo_img)
        with pytest.raises(DisnError, match="fp16 range"):
            fresh.mesh_grid_adaptive(BOX, tm, 128, iso=0.0)
        v, f = fresh.fetch_mesh()
        assert v.shape == (0, 3) and f.shape == (0, 3)
        fresh.write_mesh_obj(str(tmp_path / "after_overflow.obj"))      # the library's counts, not Python's
        with open(tmp_path / "after_overflow.obj") as fh:
            head = fh.read(4096)
        assert "Number of vertices: 0\n" in head and "Number of faces: 0\n" in head
        fresh.load_weights(weights)
        fresh.encode(demo_img)
        iso = median_iso(fresh)
        v, f, _ = fresh.mesh_grid_adaptive(BOX, tm, 64, iso=iso)
        assert len(f) > 0 and np.isfinite(v).all()
    finally:
        fresh.close()
