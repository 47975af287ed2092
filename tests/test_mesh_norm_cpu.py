"""CPU tests of the twins of the surface-sample normalisation and the field samplers (oracle/mesh_norm_oracle.py), which
the GPU path reproduces bit for bit: exact areas, area-proportional picks, samples inside their triangles, the reference's
own get_normalize_mesh (tests/golden/normalize_ref.npz), the host sample_sdf on golden and band-edge fields, and the whole
chain at res 32 on the CPU twins."""
import numpy as np
import pytest
from scipy import stats

from disn_b200 import create_point_sdf_grid as cpsg
from disn_b200.create_sdf import read_obj_parts
from oracle import mc_oracle
from oracle import mesh_norm_oracle as no
from oracle import mesh_sdf_oracle as so

TRI_V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0], [0, 3, 0], [0, 0, 4], [0.5, 0.5, 0]], np.float32)


def test_exact_areas_and_quantisation():
    f = np.array([[0, 1, 2], [0, 3, 4], [0, 1, 3], [0, 5, 1], [1, 2, 6]], np.int32)     # 0.5, 3, 0 (collinear), 2, 0
    a = no.face_areas(TRI_V, f)
    np.testing.assert_array_equal(a, [0.5, 3.0, 0.0, 2.0, 0.0])
    s = no.part_scan(TRI_V, f)
    assert s["shift"] == 62 - 4                     # a_max * n_faces = 15 = 0.9375 * 2^4
    q = np.rint(np.ldexp(a, s["shift"])).astype(np.int64)
    assert s["q"] == [int(q.sum())] and q[0] * 6 == q[1] and q[2] == q[4] == 0
    assert s["q"][0] < 2 ** 63


def test_amounts_are_exact_integers():
    assert no.amounts([1, 1, 1]) == [5461, 5461, 5461]
    assert no.amounts([3, 1]) == [12288, 4096]
    assert no.amounts([2 ** 61, 2 ** 61 - 1]) == [8192, 8191]
    assert no.amounts([5, 0]) == [16384, 0]


def _draws(n, seed):
    np.random.seed(seed)
    return cpsg.surface_draws([n])


def test_picks_proportional_to_area_chi_square():
    f = np.array([[0, 1, 2], [0, 3, 4], [0, 5, 1]], np.int32)        # areas 0.5, 3, 2
    scan = no.part_scan(TRI_V, f)
    _, face = no.sample(TRI_V, f, scan, [16384], _draws(16384, 1))
    obs = np.bincount(face, minlength=3)
    exp = 16384 * np.array([0.5, 3, 2]) / 5.5
    assert stats.chisquare(obs, exp).pvalue > 1e-3


def test_zero_area_faces_never_picked():
    f = np.array([[0, 1, 3], [0, 1, 2], [0, 1, 3], [1, 2, 6], [0, 3, 4], [1, 2, 6]], np.int32)
    scan = no.part_scan(TRI_V, f)
    zero = scan["areas"] == 0
    assert zero.sum() == 4
    d = _draws(5000, 2)
    d[:3, 0] = [0.0, 1.0 - 2.0 ** -53, 0.5 / 3.5]        # both ends and the boundary between the two faces with area
    _, face = no.sample(TRI_V, f, scan, [5000], d)
    assert not zero[face].any() and set(face[:2]) == {1, 4}


def test_samples_inside_their_triangles():
    v = np.random.default_rng(4).standard_normal((30, 3)).astype(np.float32)
    f = np.random.default_rng(5).integers(0, 30, (40, 3)).astype(np.int32)
    scan = no.part_scan(v, f)
    pts, face = no.sample(v, f, scan, [4000], _draws(4000, 3))
    t = v.astype(np.float64)[f[face]]
    e1, e2, d = t[:, 1] - t[:, 0], t[:, 2] - t[:, 0], pts - t[:, 0]
    g = np.stack([np.einsum("ij,ij->i", x, y) for x, y in ((e1, e1), (e1, e2), (e2, e2), (d, e1), (d, e2))])
    den = g[0] * g[2] - g[1] * g[1]
    b1 = (g[2] * g[3] - g[1] * g[4]) / den
    b2 = (g[0] * g[4] - g[1] * g[3]) / den
    ok = den > 1e-12 * (g[0] * g[2])
    tol = 1e-9
    assert (b1[ok] >= -tol).all() and (b2[ok] >= -tol).all() and (b1[ok] + b2[ok] <= 1 + tol).all()
    resid = np.linalg.norm(d - b1[:, None] * e1 - b2[:, None] * e2, axis=1)
    assert (resid[ok] < 1e-9 * (1 + np.abs(t).max())).all()


def test_twin_against_the_reference_get_normalize_mesh(golden):
    g = golden["normalize_ref"]
    names = sorted({k[:-len("_meta")] for k in g.files if k.endswith("_meta")})
    assert len(names) == 3
    for name in names:
        v, f, pid = g[name + "_verts"], g[name + "_faces"], g[name + "_part_ids"]
        P, seed = (int(x) for x in g[name + "_meta"])
        scan = no.part_scan(v, f, pid, P)
        amts = no.amounts(scan["q"])
        assert amts == g[name + "_amounts"].tolist(), name
        np.random.seed(seed)
        c, m, pts, out = no.normalize(v, f, pid, P, amts, cpsg.surface_draws(amts))
        # fixed-point centroid vs np.mean: rint(p * 2^32) moves each term by <= 2^-33, the float64 mean and the final
        # roundings of both by a few 2^-53 * max|p| * log2(N) -- bound 2^-33 + 2^-44 max|p|
        maxabs = np.abs(pts).max()
        bc = 2.0 ** -33 + 2.0 ** -44 * maxabs
        dc = np.abs(c - g[name + "_centroid"]).max()
        assert dc <= bc, (name, dc, bc)
        bm = np.sqrt(3) * bc + 2.0 ** -50 * m
        assert abs(m - float(g[name + "_m"])) <= bm, name
        ref = g[name + "_out_verts"]
        rel = np.abs(v.astype(np.float64) - c).max() / m
        bound = (bc + rel * bm) / m
        err = np.abs(out.astype(np.float64) - ref)
        assert (err <= np.spacing(np.abs(ref).astype(np.float32)) + bound).all(), name


@pytest.mark.parametrize("case", ["centred_plane", "shifted_car", "chair_iso", "short_band"])
def test_band_twin_equals_host_sample_sdf_on_golden(golden, case):
    from tests.golden.make_golden_sample_sdf import CASES
    g = golden["sample_sdf"]
    _, _, _, cat, n, bw, iso, seed = [c for c in CASES if c[0] == case][0]
    res = int(g["res"])
    val = g[case + "_value"]
    np.random.seed(seed)
    host, _ = cpsg.sample_sdf(cat, n, bw, iso, {"param": g["param"], "value": val}, res)
    np.random.seed(seed)
    twin = no.sample_sdf(n, bw, iso, g["param"], res, val)
    np.testing.assert_array_equal(twin.view(np.uint32), host.view(np.uint32))
    np.testing.assert_array_equal(twin.view(np.uint32), g[case + "_samples"].view(np.uint32))


@pytest.mark.parametrize("iso", [0.0, 0.003])
def test_band_twin_on_band_edges(iso):
    """Values exactly on, one ulp below and one ulp above every band edge: float32(0.03) >= 0.1 * 0.30 is True under numpy
    2's float32 comparison and False in float64."""
    bw = 0.1
    edges = no.band_edges(bw)
    assert np.float32(0.03) >= np.float32(bw * 0.30) and not float(np.float32(0.03)) >= bw * 0.30
    e = np.unique(edges.reshape(-1))
    d = np.concatenate([e, np.nextafter(e, np.float32(-1)), np.nextafter(e, np.float32(1)), [np.float32(0.03)]])
    vals = (d + np.float32(iso)).astype(np.float32)
    res = 6
    field = np.resize(vals, (res + 1) ** 3).astype(np.float32).reshape(res + 1, res + 1, res + 1)
    params = np.float32([-1, -1, -1, 1, 1, 1])
    lists = no.band_lists(field, iso, edges)
    dis = field.reshape(-1) - iso
    for b, (lo, hi) in enumerate(edges):
        np.testing.assert_array_equal(lists[b], np.argwhere((dis >= lo) & (dis < hi))[:, 0])
    for seed in (0, 1):
        np.random.seed(seed)
        host, _ = cpsg.sample_sdf("", 200, bw, iso, {"param": params, "value": field}, res)
        np.random.seed(seed)
        twin = no.sample_sdf(200, bw, iso, params, res, field)
        np.testing.assert_array_equal(twin.view(np.uint32), host.view(np.uint32))


def test_strided_twin_equals_the_reference_index_formula():
    res, reduce = 16, 3
    R = res + 1
    v = np.random.default_rng(6).standard_normal((R, R, R)).astype(np.float32)
    n = res // reduce + 1
    zv, yv, xv = np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij")
    idx = (xv * reduce + yv * R * reduce + zv * R * R * reduce).reshape(-1)
    np.testing.assert_array_equal(no.strided(v, reduce).reshape(-1), v.reshape(-1)[idx])


def test_read_obj_parts_splits_by_material(tmp_path):
    p = tmp_path / "m.obj"
    p.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nv 0 0 1\nf 1 2 3\nusemtl b\nf 1 2 4\nusemtl a\nf 1/1 3/1 4/1\n"
                 "usemtl b\nf 2 3 4\n")
    v, f, pid, names = read_obj_parts(str(p))
    assert names == [None, "b", "a"] and pid.tolist() == [0, 1, 2, 1] and f.tolist()[2] == [0, 2, 3]
    q = tmp_path / "n.obj"
    q.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3\n")
    assert read_obj_parts(str(q))[3] == [None]


def test_whole_chain_on_the_cpu_twins():
    """raw mesh -> twin normalisation -> twin field at res 32 -> twin marching cubes at 0.003 -> host sample_sdf."""
    ax = np.linspace(-1, 1, 21)
    z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
    f = np.sqrt((np.sqrt((x - 0.2) ** 2 + y * y) - 0.45) ** 2 + z * z) - 0.2
    v, fc = mc_oracle.marching_cubes(f.astype(np.float32), [-1, -1, -1, 1, 1, 1], 0.0)
    v = (v * np.float32(5) + np.float32(3)).astype(np.float32)
    scan = no.part_scan(v, fc)
    amts = no.amounts(scan["q"])
    np.random.seed(9)
    c, m, pts, nv = no.normalize(v, fc, None, 1, amts, cpsg.surface_draws(amts))
    assert np.abs((pts - c) / m).max() <= 1.0 + 1e-12
    assert np.linalg.norm(nv.astype(np.float64), axis=1).max() < 1.01
    grid, bbox = so.mesh_sdf(nv, fc, 32)
    mv, mf = mc_oracle.marching_cubes(grid, bbox, 0.003)
    assert len(mf) > 100
    samples, insideout = cpsg.sample_sdf("02691156", 2000, 0.1, 0.003, {"param": np.float32(bbox), "value": grid}, 32)
    assert samples.shape == (2000, 4) and np.abs(samples[:, 3] - np.float32(0.003)).max() < 0.1 + 1e-6
    assert insideout                                        # the torus hole: the point nearest the origin is outside
