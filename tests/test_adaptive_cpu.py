"""CPU tests of the coarse-to-fine grid's numpy twin (oracle/adaptive_oracle.py): on exact distance fields the mesh of the
adaptive grid equals the dense grid's, the stride rule, band = inf, and the fill rule at a T-junction."""
import numpy as np
import pytest

from oracle import adaptive_oracle as ao
from oracle import mc_oracle


def grid_xyz(bbox, R):
    ax = [np.linspace(bbox[a], bbox[3 + a], R) for a in range(3)]
    z, y, x = np.meshgrid(ax[2], ax[1], ax[0], indexing="ij")
    return x, y, z


def exact_field(kind, bbox, R):
    """Exact signed distance fields (1-Lipschitz) in float64, rounded once to float32."""
    x, y, z = grid_xyz(bbox, R)
    if kind == "sphere":
        f = np.sqrt(x * x + y * y + z * z) - 0.55
    elif kind == "torus":
        f = np.sqrt((np.sqrt(x * x + y * y) - 0.5) ** 2 + z * z) - 0.2
    elif kind == "slabs":             # two parallel slabs thinner than the coarse stride, 0.12 apart
        w = 0.012
        f = np.minimum(np.abs(z - 0.13) - w, np.abs(z - 0.25) - w)
    elif kind == "box":
        q = np.abs(np.stack([x, y, z])) - np.array([0.5, 0.3, 0.4])[:, None, None, None]
        f = np.linalg.norm(np.maximum(q, 0), axis=0) + np.minimum(q.max(axis=0), 0)
    else:
        raise ValueError(kind)
    return f.astype(np.float32)


CASES = {   # name: (field kind, bbox, iso)
    "sphere": ("sphere", [-1, -1, -1, 1, 1, 1], 0.0),
    "torus": ("torus", [-1, -1, -1, 1, 1, 1], 0.0),
    "slabs": ("slabs", [-1, -1, -1, 1, 1, 1], 0.0),
    "box_iso": ("box", [-1, -1, -1, 1, 1, 1], 0.07),
    "sphere_non_cubic": ("sphere", [-0.9, -0.7, -0.8, 0.8, 0.9, 0.6], 0.0),
}


def same_mesh(a, b):
    return a[0].shape == b[0].shape and a[1].shape == b[1].shape and np.array_equal(a[0].view(np.uint32),
                                                                                    b[0].view(np.uint32)) \
        and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("R", [65, 129])
@pytest.mark.parametrize("name", sorted(CASES))
def test_exact_fields_mesh_identical_band1(name, R):
    kind, bbox, iso = CASES[name]
    f = exact_field(kind, bbox, R)
    mask, counts, g = ao.refine(f, bbox, iso=iso, band=1.0)
    assert sum(counts) == mask.sum() < R ** 3
    assert len(counts) == 1 + 4                       # coarse lattice + levels 16, 8, 4, 2
    np.testing.assert_array_equal(g[mask].view(np.uint32), f[mask].view(np.uint32))
    dense = mc_oracle.marching_cubes(f, bbox, iso)
    assert len(dense[1]) > 0
    assert same_mesh(mc_oracle.marching_cubes(g, bbox, iso), dense)
    # every sign-changing edge of the dense grid has both ends evaluated
    for ax in range(3):
        a = [slice(None)] * 3
        b = [slice(None)] * 3
        a[ax], b[ax] = slice(0, -1), slice(1, None)
        cross = (f[tuple(a)] < iso) != (f[tuple(b)] < iso)
        assert (mask[tuple(a)][cross] & mask[tuple(b)][cross]).all()


def test_evaluated_fraction_shrinks_with_resolution():
    bbox = [-1, -1, -1, 1, 1, 1]
    frac = [ao.refine(exact_field("sphere", bbox, R), bbox)[0].mean() for R in (65, 129)]
    assert frac[1] < frac[0] < 0.6


@pytest.mark.parametrize("R", [33, 65])
def test_band_inf_evaluates_everything(R):
    bbox = [-1, -1, -1, 1, 1, 1]
    f = exact_field("torus", bbox, R)
    mask, counts, g = ao.refine(f, bbox, band=np.inf)
    assert mask.all() and sum(counts) == R ** 3
    np.testing.assert_array_equal(g.view(np.uint32), f.view(np.uint32))


@pytest.mark.parametrize("res,s0", [(100, 4), (101, 1), (96, 16), (72, 8), (34, 2), (128, 16), (1, 1), (2, 2)])
def test_stride_rule(res, s0):
    assert ao.coarse_stride(res) == s0
    bbox = [-1, -1, -1, 1, 1, 1]
    f = exact_field("sphere", bbox, res + 1)
    mask, counts, g = ao.refine(f, bbox)
    n_levels = int(np.log2(s0))
    assert len(counts) == 1 + n_levels
    assert counts[0] == (res // s0 + 1) ** 3
    if s0 == 1:
        assert mask.all() and np.array_equal(g.view(np.uint32), f.view(np.uint32))
    else:
        assert sum(counts) == mask.sum()
        assert same_mesh(mc_oracle.marching_cubes(g, bbox), mc_oracle.marching_cubes(f, bbox))


def _lerp(t, a, b):
    return (np.float32(1) - np.float32(t)) * np.float32(a) + np.float32(t) * np.float32(b)


def _interp(F, o, s, p):
    """trilinear value at point p (z, y, x) of the block of size s at origin o: x, then y, then z."""
    t = [np.float32(p[k] - o[k]) / np.float32(s) for k in range(3)]
    c = [[_lerp(t[2], F[o[0] + s * kz, o[1] + s * ky, o[2]], F[o[0] + s * kz, o[1] + s * ky, o[2] + s])
          for ky in (0, 1)] for kz in (0, 1)]
    return _lerp(t[0], _lerp(t[1], c[0][0], c[0][1]), _lerp(t[1], c[1][0], c[1][1]))


def test_t_junction_fill_rule():
    """res 32: eight level-16 blocks; a small ball near the origin (grid units) makes only the block at the origin and its
    child at the origin active (band 0.5).  A point on the face that block shares with an inactive level-16 neighbour
    takes the value of the finest inactive child there, not the coarse neighbour's, and the whole fill equals a
    coarse-to-fine overwrite over the inactive blocks."""
    R, res = 33, 32
    bbox = [0, 0, 0, res, res, res]                 # h = 1 per axis
    x, y, z = grid_xyz(bbox, R)
    f = (np.sqrt((x - 3) ** 2 + (y - 3) ** 2 + (z - 3) ** 2) - 2).astype(np.float32)
    mask, counts, g, states = ao.refine(f, bbox, iso=0.0, band=0.5, want_states=True)
    st = dict(states)
    assert st[16][0, 0, 0] == 2 and (st[16].reshape(-1)[1:] == 1).all()
    # coarse-to-fine overwrite, block by block
    want = np.where(mask, f, np.float32(np.nan)).astype(np.float32)
    for s in sorted(st, reverse=True):
        for bz, by, bx in zip(*np.nonzero(st[s] == 1)):
            o = (bz * s, by * s, bx * s)
            for pz in range(o[0], o[0] + s + 1):
                for py in range(o[1], o[1] + s + 1):
                    for px in range(o[2], o[2] + s + 1):
                        if not mask[pz, py, px]:
                            want[pz, py, px] = _interp(f, o, s, (pz, py, px))
    np.testing.assert_array_equal(g.view(np.uint32), want.view(np.uint32))
    # the face x = 16 between block (0,0,0) (active, subdivided) and block (0,0,1) (inactive at level 16)
    assert st[8][0, 0, 0] == 2 and (st[8][:2, :2, :2].reshape(-1)[1:] == 1).all()
    p = (12, 4, 16)                       # on the face x = 16 of child (1, 0, 1), off every evaluated lattice
    assert not mask[p]
    fine, coarse = _interp(f, (8, 0, 8), 8, p), _interp(f, (0, 0, 16), 16, p)
    assert g[p] == fine != coarse
