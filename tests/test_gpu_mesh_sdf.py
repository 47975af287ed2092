"""GPU tests of the signed distance field (disn_mesh_sdf, Engine.mesh_sdf) against the CPU twin
oracle/mesh_sdf_oracle.py, bit for bit, on a zoo of closed meshes, holes, polygon soups and boxes."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

from disn_b200 import synth
from disn_b200._lib import DisnError
from oracle import mc_oracle
from oracle import mesh_sdf_oracle as so
from tests.test_mesh_sdf_cpu import CUBE_F, CUBE_V, analytic_mesh, holed_sphere

pytestmark = pytest.mark.gpu

BOX = [-1, -1, -1, 1, 1, 1]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def soup():
    """Two interpenetrating cubes, a duplicated face, a zero-area face (collinear corners), a repeated-vertex face and a
    stray triangle crossing both cubes."""
    v2 = CUBE_V * np.float32(0.6) + np.float32(0.55)
    v = np.concatenate([CUBE_V, v2, [[0.1, 0.1, 0.5], [0.5, 0.5, 0.5], [0.9, 0.9, 0.5]], [[-0.2, 0.5, 0.5],
                        [1.4, 0.3, 0.9], [1.3, 1.3, 0.2]]]).astype(np.float32)
    f = np.concatenate([CUBE_F, CUBE_F + 8, CUBE_F[:1], [[16, 17, 18], [3, 3, 5], [19, 20, 21]]]).astype(np.int32)
    return v, f


def zoo():
    sph = analytic_mesh("sphere", 13)
    hv, hf, _ = holed_sphere()
    return {
        "cube": (CUBE_V, CUBE_F, None, 0.0),
        "sphere": (*sph, None, 0.0),
        "torus": (*analytic_mesh("torus", 15), None, 0.0),
        "holed_sphere_s0": (hv, hf, None, 0.0),
        "holed_sphere_s015": (hv, hf, None, 0.15),
        "soup": (*soup(), None, 0.0),
        "crosses_box": (*sph, [-0.3, -0.8, -0.5, 0.9, 0.8, 0.4], 0.0),
        "non_cubic_box": (*analytic_mesh("torus", 15), [-0.9, -0.8, -0.35, 0.85, 0.9, 0.3], 0.02),
    }


ZOO = zoo()


@pytest.mark.parametrize("name", sorted(ZOO))
def test_zoo_full_grid_bit_exact_res32(engine, name):
    v, f, bbox, sigma = ZOO[name]
    got, gb = engine.mesh_sdf(32, bbox=bbox, sigma=sigma, verts=v, faces=f)
    want, wb = so.mesh_sdf(v, f, 32, bbox=bbox, sigma=sigma)
    assert gb == wb
    np.testing.assert_array_equal(bits(got), bits(want))
    if name == "holed_sphere_s0":
        assert (got[got != 0] > 0).all()                     # the hole leaks: no negative point off the surface


def _band_and_samples(R, d_band, n, seed):
    rng = np.random.default_rng(seed)
    band = np.nonzero(np.isfinite(d_band))[0]
    band = rng.choice(band, min(len(band), 4000), replace=False)
    return np.union1d(band, rng.choice(R ** 3, n, replace=False))


@pytest.mark.parametrize("name,res", [(n, 64) for n in ("sphere", "torus", "holed_sphere_s015", "soup", "non_cubic_box")]
                         + [(n, 128) for n in ("sphere", "torus", "soup", "crosses_box")])
def test_zoo_sign_everywhere_and_distance_on_band_and_samples(engine, name, res):
    """Sign (exterior mask) at every grid point; distance bit for bit on 4000 points of the two-cell band and 3000
    random points."""
    v, f, bbox, sigma = ZOO[name]
    got, gb = engine.mesh_sdf(res, bbox=bbox, sigma=sigma, verts=v, faces=f)
    R = res + 1
    ext = so.sign_from_band(v, f, res, gb, sigma)
    g = got.reshape(-1)
    np.testing.assert_array_equal(np.signbit(g), ~ext)
    band = so.band_distance(v, f, gb, R, 2.0 * (gb[3] - gb[0]) / res)
    idx = _band_and_samples(R, band, 3000, res)
    want = so.unsigned_distance(v, f, so.grid_points(gb, R)[idx])
    np.testing.assert_array_equal(bits(np.abs(g[idx])), bits(want))


def _exact_distance_by_candidates(verts, faces, pts, d_bound):
    """Brute-force d of pts restricted to faces whose centroid ball can reach within d_bound (+ slack) of the point:
    a face farther than that cannot be nearer than d_bound; a d_bound that is too small leaves the true nearest face out
    and the result above d_bound, so the check stays a check."""
    v = verts.astype(np.float64)
    tri = v[faces]
    cen = tri.mean(axis=1)
    rad = np.linalg.norm(tri - cen[:, None], axis=2).max()
    tree = cKDTree(cen)
    lists = tree.query_ball_point(pts.astype(np.float64), d_bound.astype(np.float64) * (1 + 1e-6) + rad + 1e-6)
    pi = np.repeat(np.arange(len(pts)), [len(x) for x in lists])
    fi = np.concatenate([np.asarray(x, np.int64) for x in lists])
    P = pts.astype(np.float64)
    d2 = so.tri_dist2([P[pi, i] for i in range(3)], *[[tri[fi, k, i] for i in range(3)] for k in range(3)])
    best = np.full(len(pts), np.inf)
    np.fmin.at(best, pi, d2)
    return np.sqrt(best).astype(np.float32)


@pytest.fixture(scope="module")
def predicted_mesh(engine):
    """Marching cubes of the config-1 predicted 257^3 grid at its median (~8e5 faces)."""
    engine.encode(synth.synthetic_images(1))
    ptr = engine.eval_grid_resident(synth.DEMO_SDF_PARAMS, synth.DEMO_TRANS_MAT, 256)
    grid = engine.fetch(ptr, (257, 257, 257))
    iso = float(np.median(grid))
    v, f = engine.marching_cubes(None, BOX, iso, device_ptr=ptr, R=257)
    return v, f, ptr, iso


def test_predicted_mesh_257_distances_at_samples(engine, predicted_mesh):
    v, f, _, _ = predicted_mesh
    assert len(f) > 10 ** 5
    got, gb = engine.mesh_sdf(256)
    R = 257
    rng = np.random.default_rng(7)
    g = got.reshape(-1)
    near = np.nonzero(np.abs(g) < 4 * (gb[3] - gb[0]) / 256)[0]
    idx = np.concatenate([rng.choice(near, 19800, replace=False), rng.choice(R ** 3, 200, replace=False)])
    pts = so.grid_points(gb, R)[idx]
    want = _exact_distance_by_candidates(v, f, pts, np.abs(g[idx]))
    np.testing.assert_array_equal(bits(np.abs(g[idx])), bits(want))
    print("257^3 predicted mesh: %d faces, phases %s" % (len(f), engine.mesh_sdf_phase_ms()))


def test_closed_mesh_257_sign_against_winding_number(engine):
    v, f = analytic_mesh("torus", 65)
    got, gb = engine.mesh_sdf(256, verts=v, faces=f)
    rng = np.random.default_rng(8)
    idx = rng.choice(257 ** 3, 1500, replace=False)
    g = got.reshape(-1)[idx]
    w = so.winding_number(v, f, so.grid_points(gb, 257)[idx])
    off = np.abs(g) > 1e-6
    np.testing.assert_array_equal((g < 0)[off], (np.abs(w) > 0.5)[off])


def test_deterministic_and_resident_chain_equals_upload(engine, predicted_mesh):
    v, f, ptr, iso = predicted_mesh
    engine.marching_cubes(None, BOX, iso, device_ptr=ptr, R=257, fetch=False)      # the mesh stays in HBM
    a, ba = engine.mesh_sdf(128)
    b, bb = engine.mesh_sdf(128)
    np.testing.assert_array_equal(bits(a), bits(b))
    c, bc = engine.mesh_sdf(128, verts=v, faces=f)
    assert ba == bb == bc
    np.testing.assert_array_equal(bits(a), bits(c))


def test_round_trip_through_marching_cubes(engine):
    import torch
    v, f = analytic_mesh("sphere", 65)
    res = 128
    out = torch.empty((res + 1,) * 3, dtype=torch.float32, device="cuda:0")
    none, bb = engine.mesh_sdf(res, verts=v, faces=f, device_ptr=out.data_ptr())
    assert none is None
    torch.cuda.synchronize()
    host, bh = engine.mesh_sdf(res)
    np.testing.assert_array_equal(bits(out.cpu().numpy()), bits(host))
    v2, f2 = engine.marching_cubes(None, bb, 0.0, device_ptr=out.data_ptr(), R=res + 1)
    iou = engine.iou(v, f, v2, f2, dim=110)
    cd = float(engine.chamfer_x1000(v[None], v2[None])[0])
    print("round trip: IoU %.5f, Chamfer x1000 %.3e" % (iou, cd))
    assert iou >= 0.99
    # Chamfer of the two vertex clouds: the 65^3 mesh's vertex spacing dominates it (0.177 for the same mesh against
    # marching cubes of the analytic sphere field on this 129^3 grid), so the bound leaves only ~40 % for the field
    assert cd < 0.25


def test_errors_leave_the_context_usable():
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="fp32")
    try:
        with pytest.raises(DisnError, match="no resident mesh"):
            eng.mesh_sdf(8)
        eng.load_mesh(CUBE_V, np.zeros((0, 3), np.int32))
        with pytest.raises(DisnError, match="no resident mesh"):
            eng.mesh_sdf(8)
        nan = CUBE_V.copy()
        nan[3, 1] = np.nan
        with pytest.raises(DisnError, match="non-finite"):
            eng.mesh_sdf(8, verts=nan, faces=CUBE_F)
        inf = CUBE_V.copy()
        inf[0, 2] = np.inf
        with pytest.raises(DisnError, match="non-finite"):
            eng.mesh_sdf(8, verts=inf, faces=CUBE_F)
        eng.load_mesh(CUBE_V, CUBE_F)
        for kw, msg in [(dict(res=0), "res >= 1"), (dict(res=-3), "res >= 1"), (dict(res=1290), "32-bit"),
                        (dict(res=8, bbox=[0, 0, 0, 1, 0, 1]), "min must be below max"),
                        (dict(res=8, bbox=[0, 0, 0, 1, 1, np.nan]), "min must be below max"),
                        (dict(res=8, sigma=-0.1), "sigma"), (dict(res=8, sigma=np.nan), "sigma"),
                        (dict(res=8, sigma=np.inf), "sigma"), (dict(res=8, expand_rate=0.0), "expand_rate")]:
            with pytest.raises(DisnError, match=msg):
                eng.mesh_sdf(**kw)
            got, _ = eng.mesh_sdf(8)                      # the context still works
            assert (got < 0).sum() > 0
        flat = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
        with pytest.raises(DisnError, match="min must be below max"):
            eng.mesh_sdf(8, verts=flat * 0, faces=[[0, 1, 2]])       # a single point: no automatic box
        got, bb = eng.mesh_sdf(8, verts=CUBE_V, faces=CUBE_F)
        want, wb = so.mesh_sdf(CUBE_V, CUBE_F, 8)
        assert bb == wb
        np.testing.assert_array_equal(bits(got), bits(want))
    finally:
        eng.close()


def test_create_one_sdf_writes_dist_and_samples(tmp_path):
    from disn_b200 import create_point_sdf_grid as cpsg
    from disn_b200.create_sdf import write_obj
    v, f = analytic_mesh("sphere", 25)
    obj, dist = str(tmp_path / "m.obj"), str(tmp_path / "m.dist")
    write_obj(obj, v, f)
    grid, bbox = cpsg.create_one_sdf("ignored", 32, 1.2, dist, obj, 0, g=0.0)
    s = cpsg.get_sdf(dist, 32)
    from disn_b200.create_sdf import read_obj
    rv, rf = read_obj(obj)
    want, wb = so.mesh_sdf(rv, rf, 32)
    np.testing.assert_array_equal(bits(s["value"]), bits(want))
    np.testing.assert_array_equal(s["param"], np.float32(wb))
    np.random.seed(0)
    pts, flag = cpsg.sample_sdf("02691156", 2000, 0.1, 0.0, s, 32)
    assert len(pts) == 2000 and not flag                     # the origin is inside the sphere
    cpsg.main(["--obj", obj, "--res", "16", "--out", str(tmp_path / "c.dist"), "--samples", "400", "--seed", "1"])
    z = np.load(str(tmp_path / "c_samples.npz"))
    assert z["sdf_pt_val"].shape == (400, 4)
