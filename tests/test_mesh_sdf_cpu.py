"""CPU tests of the signed-distance twin oracle/mesh_sdf_oracle.py against methods that share none of its code: hand-
derived distances, the closed-form box distance, a dense barycentric search, the generalised winding number, and the
reference's own sample_sdf / check_insideout (golden)."""
import numpy as np
import pytest

from disn_b200 import create_point_sdf_grid as cpsg
from oracle import mc_oracle
from oracle import mesh_sdf_oracle as so

CUBE_V = np.array([[x, y, z] for z in (0, 1) for y in (0, 1) for x in (0, 1)], np.float32)
CUBE_F = np.array([[0, 2, 1], [1, 2, 3], [4, 5, 6], [5, 7, 6], [0, 1, 4], [1, 5, 4], [2, 6, 3], [3, 6, 7],
                   [0, 4, 2], [2, 4, 6], [1, 3, 5], [3, 7, 5]], np.int32)


def analytic_mesh(kind, R):
    """Closed MC meshes of analytic fields on [-1,1]^3 (outward winding)."""
    ax = np.linspace(-1, 1, R)
    z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
    r = np.sqrt(x * x + y * y + z * z)
    if kind == "sphere":
        f = r - 0.62
    elif kind == "torus":
        f = np.sqrt((np.sqrt(x * x + y * y) - 0.5) ** 2 + z * z) - 0.22
    elif kind == "nested_shells":                   # two outward spheres, one inside the other
        v1, f1 = mc_oracle.marching_cubes((r - 0.7).astype(np.float32), [-1, -1, -1, 1, 1, 1], 0.0)
        v2, f2 = mc_oracle.marching_cubes((r - 0.35).astype(np.float32), [-1, -1, -1, 1, 1, 1], 0.0)
        return np.concatenate([v1, v2]), np.concatenate([f1, f2 + len(v1)]).astype(np.int32)
    else:
        raise ValueError(kind)
    return mc_oracle.marching_cubes(f.astype(np.float32), [-1, -1, -1, 1, 1, 1], 0.0)


def cavity_shell(R):
    """max(r - 0.7, 0.35 - r): the inner surface faces inwards and encloses a cavity that no grid path reaches."""
    ax = np.linspace(-1, 1, R)
    z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
    r = np.sqrt(x * x + y * y + z * z)
    return mc_oracle.marching_cubes(np.maximum(r - 0.7, 0.35 - r).astype(np.float32), [-1, -1, -1, 1, 1, 1], 0.0)


def _d(p, a, b, c):
    pp = [np.array([[v]], np.float64) for v in p]
    return float(np.sqrt(so.tri_dist2(pp, *[[np.array([[v]], np.float64) for v in q] for q in (a, b, c)])[0, 0]))


def test_single_triangle_voronoi_regions():
    a, b, c = (0.0, 0.0, 0.0), (2.0, 0.0, 0.0), (0.0, 2.0, 0.0)
    cases = [((-1.0, -1.0, 0.0), np.sqrt(2.0)),            # vertex a
             ((3.0, -1.0, 0.0), np.sqrt(2.0)),             # vertex b
             ((-1.0, 3.0, 1.0), np.sqrt(3.0)),             # vertex c
             ((1.0, -2.0, 0.0), 2.0),                      # edge ab
             ((-3.0, 1.0, 4.0), 5.0),                      # edge ac
             ((2.0, 2.0, 0.0), np.sqrt(2.0)),              # edge bc
             ((0.5, 0.5, -3.0), 3.0)]                      # face
    for p, want in cases:
        assert _d(p, a, b, c) == pytest.approx(want, rel=1e-15), p


def test_degenerate_triangle_counts_as_segments():
    a, b, c = (0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (3.0, 0.0, 0.0)     # collinear: the segment [0, 3]
    assert _d((2.0, 1.0, 0.0), a, b, c) == 1.0
    assert _d((4.0, 0.0, 0.0), a, b, c) == 1.0
    assert _d((1.0, 1.0, 1.0), a, a, a) == pytest.approx(np.sqrt(3.0), rel=1e-15)


def test_unit_cube_closed_form():
    bbox = [-0.5, -0.45, -0.55, 1.5, 1.4, 1.6]
    g, _ = so.mesh_sdf(CUBE_V, CUBE_F, 20, bbox=bbox)
    p = so.grid_points(bbox, 21).astype(np.float64)
    outside = np.linalg.norm(p - np.clip(p, 0, 1), axis=1)
    inside = (p > 0).all(1) & (p < 1).all(1)
    exact = np.where(inside, -np.minimum(p, 1 - p).min(axis=1), outside)
    got = g.reshape(-1).astype(np.float64)
    assert np.abs(np.abs(got) - np.abs(exact)).max() < 1e-7
    off = np.abs(exact) > 1e-6
    np.testing.assert_array_equal(np.sign(got[off]), np.sign(exact[off]))


def test_random_pairs_against_dense_barycentric_search():
    rng = np.random.default_rng(1)
    n = 60
    tri = rng.uniform(-1, 1, (n, 3, 3))
    p = rng.uniform(-2, 2, (n, 3))
    k = 400
    u, v = np.meshgrid(np.arange(k + 1), np.arange(k + 1), indexing="ij")
    m = u + v <= k
    u, v = u[m] / k, v[m] / k
    for i in range(n):
        a, b, c = tri[i]
        q = a[None] + u[:, None] * (b - a)[None] + v[:, None] * (c - a)[None]
        dense = np.linalg.norm(q - p[i][None], axis=1).min()
        got = _d(p[i], a, b, c)
        assert got <= dense + 1e-12
        assert dense - got < 3.0 / k * max(np.linalg.norm(b - a), np.linalg.norm(c - a)), i


def _winding_subset(v, f, bbox, res, step=5):
    """grid indices (every step-th point), their winding-number inside flags and band distances"""
    pts = so.grid_points(bbox, res + 1)
    sel = np.arange(0, len(pts), step)
    inside = np.abs(so.winding_number(v, f, pts[sel])) > 0.5
    return sel, inside


@pytest.mark.parametrize("kind,R,res", [("sphere", 25, 32), ("torus", 29, 40), ("nested_shells", 25, 33)])
def test_sign_of_closed_meshes_equals_winding_number(kind, R, res):
    v, f = analytic_mesh(kind, R)
    assert mc_oracle.is_closed_manifold(f)
    bbox = so.auto_bbox(v)
    ext = so.sign_from_band(v, f, res, bbox)
    d = so.band_distance(v, f, bbox, res + 1, 1e-6)          # exact up to 1e-6, inf beyond
    sel, inside = _winding_subset(v, f, bbox, res)
    off = d[sel] > 1e-6
    np.testing.assert_array_equal(~ext[sel][off], inside[off])
    assert inside.sum() > 100


def test_enclosed_cavity_is_interior():
    """The flood fill cannot reach a cavity: its points are negative although their winding number is 0."""
    v, f = cavity_shell(25)
    bbox, res = so.auto_bbox(v), 32
    ext = so.sign_from_band(v, f, res, bbox)
    p = so.grid_points(bbox, res + 1).astype(np.float64)
    r = np.linalg.norm(p, axis=1)
    assert not ext[r < 0.3].any() and not ext[(r > 0.4) & (r < 0.65)].any() and ext[r > 0.75].all()


def test_line_through_shared_edge_and_vertex_is_blocked():
    """Octahedron |x|+|y|+|z| = 0.5 on a grid of step 0.125: z-lines through (0.25, 0.25) meet the shared edge
    (0.5,0,0)-(0,0.5,0) in z = 0 exactly at a grid point, x-lines through (y, z) = (0, 0) meet the shared vertices."""
    V = np.array([[0.5, 0, 0], [-0.5, 0, 0], [0, 0.5, 0], [0, -0.5, 0], [0, 0, 0.5], [0, 0, -0.5]], np.float32)
    F = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]], np.int32)
    bbox, res = [-1, -1, -1, 1, 1, 1], 16
    R = res + 1
    G = so.axes(bbox, R)[0]
    i = {float(x): n for n, x in enumerate(G)}
    bits = so.blocked_edges(V, F, bbox, R)
    idx = lambda x, y, z: (i[z] * R + i[y]) * R + i[x]
    assert bits[idx(0.25, 0.25, 0.0)] & 4 and bits[idx(0.25, 0.25, -0.125)] & 4        # both z-edges at the edge point
    assert bits[idx(0.5, 0.0, 0.0)] & 1 and bits[idx(0.375, 0.0, 0.0)] & 1            # both x-edges at the vertex
    g, _ = so.mesh_sdf(V, F, res, bbox=bbox)
    p = so.grid_points(bbox, R).astype(np.float64)
    l1 = np.abs(p).sum(axis=1)
    got = g.reshape(-1)
    assert (got[l1 < 0.5 - 1e-9] < 0).all() and (got[l1 > 0.5 + 1e-9] > 0).all()
    assert (got[np.abs(l1 - 0.5) < 1e-9] == 0).all()                                   # on the surface: -0.0


def holed_sphere():
    v, f = analytic_mesh("sphere", 25)
    c = v[f].mean(axis=1)
    keep = ~((c[:, 2] > 0.55) & (np.hypot(c[:, 0], c[:, 1]) < 0.12))       # a hole of radius ~0.12 at the top
    return v, f[keep], 0.12


def test_hole_leaks_at_zero_sigma_and_closes_at_hole_radius():
    v, f, hole = holed_sphere()
    bbox, res = so.auto_bbox(v), 32
    pts = so.grid_points(bbox, res + 1)
    sig = 1.25 * hole
    d = so.band_distance(v, f, bbox, res + 1, sig)
    ext0 = so.sign_from_band(v, f, res, bbox, 0.0)
    assert ext0[d > 0].all()                                                # the interior leaks out: no negative d > 0
    ext = so.sign_from_band(v, f, res, bbox, sig)
    sel, inside = _winding_subset(v, f, bbox, res, step=3)
    away = (d[sel] > sig) & (np.linalg.norm(pts[sel] - np.array([0, 0, 0.62]), axis=1) > 3 * hole)
    np.testing.assert_array_equal(~ext[sel][away], inside[away])
    assert inside[away].sum() > 200


def test_auto_bbox_is_cube_around_the_aabb():
    v = np.array([[0, 0, 0], [2, 1, 0.5], [1, -1, 0]], np.float32)
    bb = so.auto_bbox(v, 1.2)
    assert bb == pytest.approx([1 - 1.2, -1.2, 0.25 - 1.2, 1 + 1.2, 1.2, 0.25 + 1.2], abs=1e-15)


@pytest.mark.parametrize("case", ["centred_plane", "shifted_car", "chair_iso", "short_band"])
def test_sample_sdf_and_check_insideout_match_reference(golden, case):
    g = golden["sample_sdf"]
    res = int(g["res"])
    seed = {"centred_plane": 3, "shifted_car": 4, "chair_iso": 5, "short_band": 6}[case]
    args = {"centred_plane": ("02691156", 4000, 0.1, 0.0), "shifted_car": ("02958343", 3001, 0.1, 0.0),
            "chair_iso": ("03001627", 2000, 0.05, 0.01), "short_band": ("04530566", 1000, 0.3, 0.0)}[case]
    np.random.seed(seed)
    pts, flag = cpsg.sample_sdf(args[0], args[1], args[2], args[3],
                                {"param": g["param"], "value": g[case + "_value"]}, res)
    np.testing.assert_array_equal(pts, g[case + "_samples"])
    assert pts.dtype == g[case + "_samples"].dtype
    assert bool(flag) == bool(g[case + "_insideout"])


def test_get_sdf_reads_the_dist_layout(tmp_path, golden):
    from disn_b200.engine import write_dist
    d = golden["dist_roundtrip"]
    fn = str(tmp_path / "x.dist")
    write_dist(fn, int(d["res"]), d["bbox"], d["values"])
    s = cpsg.get_sdf(fn, int(d["res"]))
    np.testing.assert_array_equal(s["param"], np.float32(d["bbox"]))
    np.testing.assert_array_equal(s["value"].reshape(-1), d["values"])
    with pytest.raises(ValueError):
        cpsg.get_sdf(fn, int(d["res"]) + 1)
