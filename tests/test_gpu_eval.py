"""GPU tests of the evaluation path: disn_iou_views (one reference mesh against V views) equals V separate disn_iou calls
bit for bit, in counts and grids, and the CPU twin's grids; it refuses bad arguments before launching anything; and the
three evaluation drivers, on the GPU engine, reproduce the reference scripts' golden (tests/golden/eval_ref.npz):
Chamfer, F-score and IoU bit for bit, EMD within the bound of tests/test_gpu_emd.py."""
import ctypes as C
import re

import numpy as np
import pytest

from oracle import metrics_oracle as mo
from tests.test_eval_cpu import Fixture, cd_numbers
from tests.test_gpu_emd import COST_RTOL

pytestmark = pytest.mark.gpu


def _icosphere(r, c, level=2):
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1),
         (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
         (9, 8, 1)]
    v = [np.array(p, float) / np.linalg.norm(p) for p in v]
    for _ in range(level):
        mid, nf = {}, []

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[k] = len(v) - 1
            return mid[k]
        for a, b, cc in f:
            ab, bc, ca = m(a, b), m(b, cc), m(cc, a)
            nf += [(a, ab, ca), (b, bc, ab), (cc, ca, bc), (ab, bc, ca)]
        f = nf
    return (np.array(v) * r + np.array(c)).astype(np.float32), np.array(f, np.int32)


def _torus(nu, nv, R=0.5, r=0.2, c=(0, 0, 0)):
    """Parametric torus with 2 * nu * nv triangles."""
    u, w = np.meshgrid(np.arange(nu) * 2 * np.pi / nu, np.arange(nv) * 2 * np.pi / nv, indexing="ij")
    v = np.stack([(R + r * np.cos(w)) * np.cos(u), (R + r * np.cos(w)) * np.sin(u), r * np.sin(w)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    a, b = i * nv + j, ((i + 1) % nu) * nv + j
    cc, d = ((i + 1) % nu) * nv + (j + 1) % nv, i * nv + (j + 1) % nv
    f = np.concatenate([np.stack([a, b, cc], -1).reshape(-1, 3), np.stack([a, cc, d], -1).reshape(-1, 3)])
    return (v + np.array(c)).astype(np.float32), f.astype(np.int32)


def _views(n, seed):
    """n meshes of very different sizes: icospheres of 80..5120 faces, random soups, a single triangle, a mesh that
    leaves the voxel window."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        kind = k % 5
        if kind == 0:
            out.append(_icosphere(rng.uniform(0.2, 0.5), rng.uniform(-0.1, 0.1, 3), level=int(rng.integers(1, 5))))
        elif kind == 1:
            m = int(rng.integers(1, 60))
            out.append((rng.uniform(-0.8, 0.8, (3 * m, 3)).astype(np.float32), np.arange(3 * m, dtype=np.int32).reshape(m, 3)))
        elif kind == 2:
            out.append((np.array([[0, 0, 0], [0.3, 0, 0], [0, 0.3, 0.1]], np.float32), np.array([[0, 1, 2]], np.int32)))
        elif kind == 3:
            out.append(_torus(int(rng.integers(8, 40)), int(rng.integers(6, 20)), R=rng.uniform(0.3, 0.6)))
        else:
            out.append(_icosphere(0.6, (0.9, -0.8, 0.2), level=2))            # partly outside [-1.1, 1.3)
    return out


@pytest.fixture(scope="module")
def eng():
    from disn_b200.engine import Engine
    e = Engine(device=0, precision="fp32")
    yield e
    e.close()


def _check_against_pairs(eng, ref, views, dim, grids=True):
    got = eng.iou_views(ref[0], ref[1], views, dim=dim, want_grids=grids)
    for v, (vv, vf) in enumerate(views):
        one = eng.iou(ref[0], ref[1], vv, vf, dim=dim, want_grids=grids)
        if grids:
            _, inter, uni, o1, o2 = one
            np.testing.assert_array_equal(got[3][0], o1)
            np.testing.assert_array_equal(got[3][v + 1], o2, err_msg="view %d" % v)
        else:
            inter, uni = eng.iou(ref[0], ref[1], vv, vf, dim=dim, want_grids=True)[1:3]
        assert (int(got[1][v]), int(got[2][v])) == (inter, uni), v
        assert got[0][v] == inter / uni
    return got


@pytest.mark.parametrize("V,dim", [(1, 32), (3, 32), (24, 32), (1, 110), (3, 110), (24, 110)])
def test_iou_views_equals_separate_calls_and_the_twin(eng, V, dim):
    ref = _icosphere(0.45, (0.05, -0.02, 0.1), level=3)
    views = _views(V, seed=V * 1000 + dim)
    got = _check_against_pairs(eng, ref, views, dim)
    np.testing.assert_array_equal(got[3][0], mo.voxel_occupancy(ref[0], ref[1], dim))
    for v in range(min(V, 6)):
        np.testing.assert_array_equal(got[3][v + 1], mo.voxel_occupancy(*views[v], dim), err_msg="view %d" % v)


def test_iou_views_large_reference(eng):
    ref = _torus(640, 640, R=0.5, r=0.25)                                    # 819 200 faces
    assert len(ref[1]) >= 800_000
    _check_against_pairs(eng, ref, _views(3, seed=5) + [_torus(300, 200, R=0.48, r=0.26)], 110)
    _check_against_pairs(eng, ref, _views(24, seed=6), 110, grids=False)


def test_iou_views_dim_512(eng):
    ref = _torus(400, 300, R=0.5, r=0.25)
    _check_against_pairs(eng, ref, [_icosphere(0.5, (0, 0, 0), level=4), _views(2, seed=9)[1]], 512)


def _call(eng, ref_v, ref_f, verts, voff, faces, foff, dim=32, V=None, null=None):
    V = len(voff) - 1 if V is None else V
    inter, uni = np.zeros(max(V, 1), np.int64), np.zeros(max(V, 1), np.int64)
    args = [ref_v, ref_f, verts, voff, faces, foff, inter, uni]
    ptrs = [None if (null == i) else a.ctypes.data_as(C.c_void_p) for i, a in enumerate(args)]
    return eng.lib.disn_iou_views(eng._h, ptrs[0], len(ref_v), ptrs[1], len(ref_f), V, ptrs[2], ptrs[3], ptrs[4], ptrs[5],
                                  dim, ptrs[6], ptrs[7], None)


def test_iou_views_refuses_bad_arguments_before_launching(eng):
    from disn_b200._lib import load
    rv, rf = _icosphere(0.4, (0, 0, 0), level=1)
    a, b, c = _icosphere(0.3, (0, 0, 0), 1), _icosphere(0.2, (0.1, 0, 0), 1), _icosphere(0.35, (0, 0.1, 0), 1)
    verts = np.concatenate([a[0], b[0], c[0]])
    faces = np.concatenate([a[1], b[1], c[1]])
    voff = np.array([0, len(a[0]), len(a[0]) + len(b[0]), len(verts)], np.int64)
    foff = np.array([0, len(a[1]), len(a[1]) + len(b[1]), len(faces)], np.int64)
    assert _call(eng, rv, rf, verts, voff, faces, foff) == 0
    bad_faces = faces.copy()
    bad_faces[foff[1] + 4, 2] = len(b[0])                                  # view 1: id = its own vertex count
    neg = faces.copy()
    neg[foff[2], 0] = -1
    cases = [
        (dict(null=2), "null argument"),
        (dict(null=7), "null argument"),
        (dict(dim=1), r"dim in \[2,512\]"),
        (dict(dim=513), r"dim in \[2,512\]"),
        (dict(V=0), "V >= 1"),
        (dict(voff=voff + 1), "must be 0"),
        (dict(foff=np.array([0, foff[2], foff[1], foff[3]], np.int64)), "view 1: face_offsets decrease"),
        (dict(voff=np.array([0, voff[2], voff[1], voff[3]], np.int64)), "view 1: vert_offsets decrease"),
        (dict(foff=np.array([0, foff[1], foff[3], foff[3]], np.int64)), "view 2: no faces"),
        (dict(faces=bad_faces), "view 1: face index out of range"),
        (dict(faces=neg), "view 2: face index out of range"),
        (dict(ref_f=rf[:0]), "reference mesh has no faces"),
    ]
    for kw, msg in cases:
        args = dict(ref_v=rv, ref_f=rf, verts=verts, voff=voff, faces=faces, foff=foff)
        args.update(kw)
        before = eng.launch_count
        assert _call(eng, **args) == -2, msg
        assert re.search(msg, load().disn_last_error().decode()), (msg, load().disn_last_error())
        assert eng.launch_count == before, msg
    from disn_b200._lib import DisnError
    with pytest.raises(DisnError, match="view 1: no faces"):
        eng.iou_views(rv, rf, [a, (b[0], b[1][:0]), c])


# -------------------------------------------------------------------------------------------------------------- drivers
@pytest.fixture
def fx(golden, tmp_path):
    return Fixture(golden["eval_ref"], tmp_path / "fx")


@pytest.mark.parametrize("batch_size", ["view_num", 1])
def test_cd_emd_driver_on_the_gpu_matches_the_golden(fx, batch_size):
    bs = fx.view_num if batch_size == "view_num" else 1
    res, draws, _ = fx.cd_emd(bs)
    prefix = "cd_emd_bs%d" % bs
    fx.assert_draws(draws, prefix)
    objs, cats = cd_numbers(res)
    want_o, want_c = fx.g[prefix + "_obj"], fx.g[prefix + "_cat"]
    # columns: avg_cf, min_cf, arg_cf, avg_emd, min_emd, arg_emd
    np.testing.assert_array_equal(np.float32(objs[:, [0, 1, 2, 5]]), np.float32(want_o[:, [0, 1, 2, 5]]))
    np.testing.assert_allclose(objs[:, [3, 4]], want_o[:, [3, 4]], rtol=COST_RTOL, atol=1e-9)
    np.testing.assert_array_equal(np.float32(cats[:, 0]), np.float32(want_c[:, 0]))
    np.testing.assert_allclose(cats[:, 1], want_c[:, 1], rtol=COST_RTOL)


def test_f_score_driver_on_the_gpu_matches_the_golden(fx):
    fx.save_pnt()
    for path in ("computed", "cached"):
        _, _, lines = fx.f_score()
        assert lines == list(fx.g["f_score_%s_lines" % path]), path


def test_iou_driver_on_the_gpu_matches_the_golden(fx):
    _, draws, lines = fx.iou()
    fx.assert_draws(draws, "iou")
    assert lines == list(fx.g["iou_lines"])
