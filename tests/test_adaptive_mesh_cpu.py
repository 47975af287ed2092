"""CPU tests of the coarse-to-fine mesher's numpy twin (oracle/adaptive_mesh_oracle.py, DESIGN.md §4.10): built from the
refinement's states and evaluated values only, its mesh equals marching cubes of the dense adaptive grid bit for bit on
smooth, noise, exact distance, tied and subnormal fields, every crossing cell lies in the candidate set K, and without
rule (ii) noise fields lose triangles, without rule (iii) the subnormal field does."""
import numpy as np
import pytest

from oracle import adaptive_mesh_oracle as amo
from oracle import adaptive_oracle as ao
from oracle import mc_oracle
from tests.test_adaptive_cpu import exact_field, grid_xyz

BANDS = [0.0, 0.5, 1.0, 2.0, np.inf]
BOXES = {"cube": [-1, -1, -1, 1, 1, 1], "non_cubic": [-0.9, -0.7, -0.8, 0.8, 0.9, 0.6]}


def make_field(kind, box, R, seed=0):
    if kind == "noise":
        return np.random.default_rng(seed).standard_normal((R, R, R)).astype(np.float32)
    if kind == "smooth":
        x, y, z = grid_xyz(box, R)
        return (np.sin(3.1 * x) * np.cos(2.3 * y) + np.sin(1.7 * z + 0.4) * 0.8 - 0.1 * x * y).astype(np.float32)
    if kind == "subnormal":                           # -2^-149 (the fill's halves round to -0) around a ball of +1
        x, y, z = grid_xyz(box, R)
        F = np.full((R, R, R), -np.float32(2.0 ** -149), np.float32)
        F[np.sqrt((x - 0.5) ** 2 + (y - 0.5) ** 2 + (z - 0.5) ** 2) < 0.3] = 1
        return F
    if kind == "ties":                                # values on a coarse quantum: iso equals many of them
        x, y, z = grid_xyz(box, R)
        return (np.round((np.sqrt(x * x + y * y + z * z) - 0.5) * 8) / 8).astype(np.float32)
    return exact_field(kind, box, R)


def crossing_cells(g, iso):
    inside = g < np.float32(iso)
    C = g.shape[0] - 1
    case = np.zeros((C, C, C), np.int64)
    for k in range(8):
        dx, dy, dz = k & 1, (k >> 1) & 1, (k >> 2) & 1
        case |= inside[dz:dz + C, dy:dy + C, dx:dx + C].astype(np.int64) << k
    return (case != 0) & (case != 255)


def check(field, box, iso, band):
    F = np.ascontiguousarray(field, np.float32)
    _, counts, dense_grid = ao.refine(F, box, iso=iso, band=band)
    want = mc_oracle.marching_cubes(dense_grid, box, iso)
    v, f, got_counts, K = amo.mesh(F, box, iso=iso, band=band, want_K=True)
    assert got_counts == counts
    assert v.shape == want[0].shape and f.shape == want[1].shape
    np.testing.assert_array_equal(v.view(np.uint32), want[0].view(np.uint32))
    np.testing.assert_array_equal(f, want[1])
    assert not (crossing_cells(dense_grid, iso) & ~K).any(), "a crossing cell of the dense adaptive grid is not in K"
    return len(want[1]), K


@pytest.mark.parametrize("band", BANDS)
@pytest.mark.parametrize("res", [2, 6, 24, 48, 64, 7])
@pytest.mark.parametrize("kind", ["smooth", "noise", "sphere", "torus"])
def test_twin_equals_dense_adaptive_mesh(kind, res, band):
    box = BOXES["cube"]
    F = make_field(kind, box, res + 1, seed=res)
    iso = float(np.median(F)) if kind in ("smooth", "noise") else 0.0
    check(F, box, iso, band)


@pytest.mark.parametrize("band", BANDS)
@pytest.mark.parametrize("kind", ["smooth", "sphere", "noise"])
def test_non_cubic_box(kind, band):
    box = BOXES["non_cubic"]
    F = make_field(kind, box, 49, seed=3)
    check(F, box, float(np.median(F)) if kind != "sphere" else 0.0, band)


@pytest.mark.parametrize("band", BANDS)
@pytest.mark.parametrize("res", [24, 64])
def test_iso_ties(res, band):
    box = BOXES["cube"]
    F = make_field("ties", box, res + 1)
    assert (F == np.float32(0.25)).any()
    check(F, box, 0.25, band)


@pytest.mark.parametrize("iso", [1.0, 0.3, -2.0])
def test_band0_one_ulp(iso):
    """band 0: inactive blocks with corners one ulp from iso.  In the normal range the fill keeps their side here (the
    margin rule (iii) still adds these blocks); test_rule_iii_subnormal_corners is the field where it must."""
    res, R = 48, 49
    rng = np.random.default_rng(11)
    iso32 = np.float32(iso)
    below, above = np.nextafter(iso32, np.float32(-np.inf)), np.nextafter(iso32, np.float32(np.inf))
    F = np.where(rng.random((R, R, R)) < 0.5, below, above).astype(np.float32)
    F[:, :, : R // 2] = below                       # half the volume one ulp below iso, no crossing inside it
    F[rng.random((R, R, R)) < 0.01] = np.float32(iso - 1.0)
    n, K = check(F, BOXES["cube"], iso, 0.0)
    assert n > 0


@pytest.mark.parametrize("res", [24, 48])
def test_rule_iii_subnormal_corners(res):
    """band 0, iso 0: inactive blocks with every corner at -2^-149 fill some points with -0, which marching cubes sees
    outside (-0 < 0 is false) while the corners are inside.  Those crossing cells are found only through rule (iii)."""
    box = BOXES["cube"]
    F = make_field("subnormal", box, res + 1)
    n, K = check(F, box, 0.0, 0.0)
    assert n > 0
    partial = amo.mesh(F, box, iso=0.0, band=0.0, rule_iii=False)
    assert len(partial[1]) < n


def test_negative_control_rule_ii():
    """Without rule (ii) (the boundary layer of inactive blocks toward active neighbours) noise fields lose triangles."""
    box = BOXES["cube"]
    lost = 0
    for seed in range(4):
        F = make_field("noise", box, 49, seed=seed)
        iso = float(np.median(F))
        full = amo.mesh(F, box, iso=iso, band=0.5)
        part = amo.mesh(F, box, iso=iso, band=0.5, rule_ii=False)
        assert len(part[1]) <= len(full[1])
        lost += len(full[1]) - len(part[1])
    assert lost > 0
