"""GPU tests of the small-part cleaning (disn_mesh_load / disn_mesh_clean, Engine.load_mesh / clean_mesh) against the CPU
twin oracle/mesh_clean_oracle.py, bit for bit: faces, vertices, per-face component labels, component and kept counts."""
import os

import numpy as np
import pytest

from disn_b200 import synth
from disn_b200._lib import DisnError
from disn_b200.create_sdf import read_obj, write_obj
from oracle import mc_oracle
from oracle import mesh_clean_oracle as mco
from tests.test_mesh_clean_cpu import hand_meshes

pytestmark = pytest.mark.gpu

BOX = [-1, -1, -1, 1, 1, 1]
# composite field: (centre, radius, survives).  The medium sphere has (0.2/0.3)^2 = 0.44 of the large one's vertices
# (> 0.3); the tiny ones ~3 %; the far one enough vertices but a centre 0.89 from the origin (>= 0.5).
SPHERES = [((-0.25, -0.1, 0.0), 0.3, True), ((0.25, 0.2, 0.1), 0.2, True), ((0.1, 0.5, -0.5), 0.05, False),
           ((-0.6, 0.5, 0.5), 0.05, False), ((-0.5, -0.6, -0.5), 0.05, False), ((0.65, -0.45, -0.4), 0.22, False)]


@pytest.fixture(scope="module")
def cases():
    return hand_meshes()


@pytest.fixture(scope="module")
def predicted_grid(engine):
    """The 257^3 grid of the synthetic He-scaled network on the demo image and camera, left in HBM, and its median."""
    engine.encode(synth.synthetic_images(1))
    ptr = engine.eval_grid_resident(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 256)
    grid = engine.fetch(ptr, (257, 257, 257))
    return grid, float(np.median(grid))


def _clean(engine, d=0.5, n=0.3):
    """clean the resident mesh -> (verts, faces, labels, counts)"""
    v, f, labels = engine.clean_mesh(d, n, want_labels=True)
    return v, f, labels, engine.last_clean


def _check(got, want):
    v, f, labels, c = got
    np.testing.assert_array_equal(f, want["faces"])
    np.testing.assert_array_equal(v, want["verts"])
    np.testing.assert_array_equal(labels, want["labels"])
    assert (c.n_components, c.n_kept, c.n_verts, c.n_faces) == (want["n_components"], want["n_kept"], len(want["verts"]),
                                                                len(want["faces"]))


def _same(a, b):
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


@pytest.mark.parametrize("name", sorted(hand_meshes()))
def test_hand_built_meshes_match_oracle(engine, cases, name):
    v, f, d, n, expected = cases[name]
    engine.load_mesh(v, f)
    want = mco.clean(v, f, d, n)
    _check(_clean(engine, d, n), want)
    assert (want["n_components"], want["n_kept"]) == expected


@pytest.mark.parametrize("R", [17, 40])
@pytest.mark.parametrize("num_thresh", [0.0, 0.3])
def test_random_field_meshes_match_oracle(engine, R, num_thresh):
    """normal-noise fields: thousands of components, union-find under contention"""
    sdf = np.random.default_rng(R).standard_normal((R, R, R)).astype(np.float32)
    v, f = engine.marching_cubes(sdf, BOX, 0.0)
    want = mco.clean(v, f, 0.5, num_thresh)
    assert want["n_components"] > (20 if R == 17 else 500)
    _check(_clean(engine, 0.5, num_thresh), want)


def test_composite_spheres_known_survivors(engine):
    R = 97
    ax = np.linspace(-1, 1, R)
    z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
    sdf = np.min([np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) - r for c, r, _ in SPHERES], axis=0)
    sdf = sdf.astype(np.float32)
    v, f = engine.marching_cubes(sdf, BOX, 0.0)
    got = _clean(engine)
    want = mco.clean(v, f)
    _check(got, want)
    assert want["n_components"] >= len(SPHERES)
    out_v = got[0].astype(np.float64)
    h = 2.0 / (R - 1)
    for c, r, survives in SPHERES:
        on = np.abs(np.linalg.norm(v - np.asarray(c), axis=1) - r) < h
        kept = np.abs(np.linalg.norm(out_v - np.asarray(c), axis=1) - r) < h
        assert on.sum() > 0
        assert kept.sum() == (on.sum() if survives else 0), (c, r)
    assert want["n_kept"] == 2 and len(out_v) == sum(
        (np.abs(np.linalg.norm(v - np.asarray(c), axis=1) - r) < h).sum() for c, r, s in SPHERES if s)


def test_predicted_grid_resident_equals_upload_and_oracle(engine, predicted_grid):
    grid, iso = predicted_grid
    ptr = engine.eval_grid_resident(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 256)
    v, f = engine.marching_cubes(None, BOX, iso, device_ptr=ptr, R=257)
    assert len(f) > 10 ** 5
    resident = _clean(engine)                                  # resident path: the mesh never left HBM before cleaning
    want = mco.clean(v, f)
    _check(resident, want)
    print("257^3 predicted grid: %d verts, %d faces, %d components, %d kept -> %d verts, %d faces"
          % (len(v), len(f), want["n_components"], want["n_kept"], len(want["verts"]), len(want["faces"])))
    engine.marching_cubes(None, BOX, iso, device_ptr=ptr, R=257, fetch=False)
    _same(_clean(engine), resident)                            # second run: bit-identical
    engine.load_mesh(v, f)                                     # upload path of the same mesh
    _same(_clean(engine), resident)


def test_write_mesh_obj_writes_the_cleaned_mesh(engine, cases, tmp_path):
    v, f, d, n, _ = cases["threshold_10x0.3"]
    engine.load_mesh(v, f)
    counts = engine.clean_mesh(d, n, fetch=False)
    assert counts.n_faces == 10 and counts.n_kept == 2
    p, q = str(tmp_path / "gpu.obj"), str(tmp_path / "ref.obj")
    engine.write_mesh_obj(p)
    want = mco.clean(v, f, d, n)
    write_obj(q, want["verts"], want["faces"])
    assert open(p).read() == open(q).read()


def test_empty_context_and_errors(tmp_path):
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="fp32")
    try:
        v, f = eng.clean_mesh()                                # a fresh context holds the empty mesh
        assert v.shape == (0, 3) and f.shape == (0, 3) and eng.last_clean.n_components == 0
        assert eng.mesh_counts() == (0, 0)
        tri = np.array([[0, 0, 0], [0.25, 0, 0], [0, 0.25, 0]], np.float32)
        eng.load_mesh(tri, [[0, 1, 2], [0, 2, 1]])
        with pytest.raises(DisnError, match="outside"):
            eng.load_mesh(tri, [[0, 1, 3]])
        with pytest.raises(DisnError, match="outside"):
            eng.load_mesh(tri, [[0, -1, 2]])
        assert eng.mesh_counts() == (3, 2)                    # a refused upload leaves the mesh loaded before
        eng.load_mesh(tri * np.float32(2 ** 29), [[0, 1, 2]])  # max|v| * n_verts = 3 * 2^27 ... below 2^30
        eng.clean_mesh()
        big = tri * np.float32(2 ** 31)                        # 2^29 * 3 >= 2^30
        eng.load_mesh(big, [[0, 1, 2]])
        with pytest.raises(DisnError, match="2\\^30"):
            eng.clean_mesh()
        assert eng.mesh_counts() == (3, 1)                    # refused after the synchronisation: still resident
        nan = tri.copy()
        nan[1, 0] = np.nan
        eng.load_mesh(nan, [[0, 1, 2]])
        with pytest.raises(DisnError, match="2\\^30"):
            eng.clean_mesh()
        eng.load_mesh(tri, [[0, 1, 2]])
        p = str(tmp_path / "t.obj")
        eng.write_mesh_obj(p)                                  # the loaded mesh is the resident one
        rv, rf = read_obj(p)
        np.testing.assert_array_equal(rv, tri)
        np.testing.assert_array_equal(rf, [[0, 1, 2]])
    finally:
        eng.close()


def _roundtrip(path, verts, faces):
    write_obj(path, verts, faces)
    return read_obj(path)


def test_create_sdf_clean_smallparts_flag(he_weights, tmp_path):
    from disn_b200 import create_sdf as cs
    from disn_b200.engine import Engine
    imgs = synth.synthetic_images(2, seed=41)
    batch = {"img": imgs, "trans_mat": synth.synthetic_trans_mats(2, seed=42),
             "sdf_params": np.tile(synth.DEMO_SDF_PARAMS, (2, 1)), "cat_id": ["02691156", "03001627"],
             "obj_nm": ["a", "b"], "view_id": [0, 23]}
    eng = Engine(device=0, precision="f16f8", max_batch=2)
    try:
        eng.load_weights(he_weights)
        eng.encode(imgs)
        grid = eng.eval_grid(batch["sdf_params"], batch["trans_mat"], 24)
    finally:
        eng.close()
    iso = float(np.median(grid))
    out = {}
    for clean in (True, False):
        F = cs.default_flags(sdf_res=24, log_dir=str(tmp_path / ("log%d" % clean)), iso=iso, batch_size=2,
                             precision="f16f8")
        if clean:
            F.clean_smallparts = True
        cs.configure(F)
        out[clean] = cs.create(he_weights, [batch])
    removed = 0
    for b in range(2):
        rv, rf = mc_oracle.marching_cubes(grid[b], batch["sdf_params"][b], iso)
        want = mco.clean(rv, rf)
        removed += len(rf) - len(want["faces"])
        for clean, (wv, wf) in ((True, (want["verts"], want["faces"])), (False, (rv, rf))):
            gv, gf = read_obj(out[clean][b])
            ev, ef = _roundtrip(str(tmp_path / ("ref%d%d.obj" % (clean, b))), wv, wf)
            np.testing.assert_array_equal(gf, ef)
            np.testing.assert_array_equal(gv, ev)
    assert removed > 0


def test_clean_meshes_and_separate_single_mesh(cases, tmp_path):
    from disn_b200 import clean_smallparts as cl
    cat = "03001627"
    src, tar = tmp_path / "src", tmp_path / "tar"
    (src / cat).mkdir(parents=True)
    meshes = {"03001627_two_00.obj": cases["two_closed"][:2], "03001627_thr_01.obj": cases["threshold_10x0.3"][:2],
              "03001627_far_02.obj": cases["far_part_dropped_by_dist"][:2],
              "03001627_rnd_03.obj": mc_oracle.marching_cubes(
                  np.random.default_rng(5).standard_normal((20, 20, 20)).astype(np.float32), BOX, 0.0)}
    for name, (v, f) in meshes.items():
        write_obj(str(src / cat / name), v, f)
    cl.clean_meshes({"chair": cat}, str(src), str(tar), thread_n=3)
    for name in meshes:
        sv, sf = read_obj(str(src / cat / name))
        want = mco.clean(sv, sf, 0.5, 0.3)
        ev, ef = _roundtrip(str(tmp_path / "ref.obj"), want["verts"], want["faces"])
        gv, gf = read_obj(str(tar / cat / name))
        np.testing.assert_array_equal(gf, ef)
        np.testing.assert_array_equal(gv, ev)

    v, f = cases["degenerate"][:2]
    write_obj(str(tmp_path / "d.obj"), v, f)
    cl.separate_single_mesh(str(tmp_path / "d.obj"), str(tmp_path / "sep"))
    labels = mco.clean(v, f)["labels"]
    wv, wf = read_obj(str(tmp_path / "sep.obj"))
    np.testing.assert_array_equal(wf, f)
    assert len(wv) == len(v)
    parts = sorted(p for p in os.listdir(tmp_path) if p.startswith("sep_"))
    assert parts == ["sep_%d.obj" % i for i in range(labels.max() + 1)]
    for i in range(labels.max() + 1):
        pv, pf = read_obj(str(tmp_path / ("sep_%d.obj" % i)))
        used = np.unique(f[labels == i])
        assert len(pf) == (labels == i).sum() and len(pv) == len(used)
        np.testing.assert_array_equal(pv[pf], v[f[labels == i]])
