"""CPU tests of the small-part cleaning twin (oracle/mesh_clean_oracle.py) against a plain-Python breadth-first
restatement of postprocessing/clean_smallparts.py:38-54, plus the OBJ reader and the file naming of the mirror module."""
import os
from collections import defaultdict

import numpy as np
import pytest

from oracle import mesh_clean_oracle as mco


def _tetra(c, s):
    v = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], np.float64) * s + np.asarray(c, np.float64)
    return v, np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]])


def _octa(c, s):
    v = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float64) * s
    f = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]])
    return v + np.asarray(c, np.float64), f


def _strip(n, c):
    """triangle strip over n vertices (n-2 faces, one component of n vertices)"""
    v = np.array([[i / 32.0, (i % 2) / 16.0, 0.0] for i in range(n)]) + np.asarray(c, np.float64)
    return v, np.array([[i, i + 1, i + 2] for i in range(n - 2)])


def _join(*parts):
    vs, fs, off = [], [], 0
    for v, f in parts:
        vs.append(v)
        fs.append(np.asarray(f) + off)
        off += len(v)
    return np.concatenate(vs).astype(np.float32), np.concatenate(fs).astype(np.int32)


def hand_meshes():
    """name -> (verts, faces, dist_thresh, num_thresh, expected (n_components, n_kept))"""
    two = _join(_tetra((0.125, 0, 0), 0.125), _octa((-0.125, 0.0625, 0), 0.125))
    tri = np.array([[0.25, 0, 0], [0.75, 0.125, 0], [0.5, -0.125, 0]], np.float32)     # centroid (0.5, 0, 0) exactly
    v5 = np.array([[0, 0, 0], [0.25, 0, 0], [0, 0.25, 0], [0, -0.25, 0], [0, 0, 0.25], [0.5, 0.5, 0]], np.float32)
    unref = _tetra((0, 0.0625, 0), 0.25)
    uv = np.insert(unref[0], 2, [[0.9, 0.9, 0.9]], axis=0).astype(np.float32)
    uf = np.where(unref[1] >= 2, unref[1] + 1, unref[1]).astype(np.int32)
    return {
        "two_closed": (*two, 0.5, 0.3, (2, 2)),
        "small_part_dropped_by_num": (*two, 0.5, 0.7, (2, 1)),          # 4 > 6 * 0.7 fails
        "far_part_dropped_by_dist": (*_join(_octa((0.7, 0, 0), 0.125), _tetra((0, 0, 0.0625), 0.125)), 0.5, 0.3, (2, 1)),
        "threshold_10x0.3": (*_join(_strip(10, (-0.25, 0, 0)), _strip(3, (0, 0.25, 0)), _strip(4, (0, -0.25, 0))),
                             0.5, 0.3, (3, 2)),                             # 3 > 3.0 fails, 4 > 3.0 holds
        "norm_equals_dist": (tri, np.array([[0, 1, 2]], np.int32), 0.5, 0.3, (1, 0)),
        "norm_below_dist": (tri, np.array([[0, 1, 2]], np.int32), 0.5000001, 0.3, (1, 1)),
        "bowtie": (v5, np.array([[0, 1, 2], [0, 3, 4]], np.int32), 0.5, 0.3, (2, 2)),
        "three_faces_one_edge": (v5, np.array([[0, 1, 2], [0, 1, 3], [1, 0, 4]], np.int32), 0.5, 0.3, (1, 1)),
        "degenerate": (v5, np.array([[0, 1, 2], [1, 1, 2], [3, 3, 3], [4, 4, 5], [2, 1, 2]], np.int32), 0.5, 0.5, (3, 2)),
        "unreferenced_vertex": (uv, uf, 0.5, 0.3, (1, 1)),
        "all_dropped": (*two, 0.0, 0.3, (2, 0)),
        "no_faces": (two[0], np.zeros((0, 3), np.int32), 0.5, 0.3, (0, 0)),
        "empty": (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32), 0.5, 0.3, (0, 0)),
    }


def bfs_clean(verts, faces, dist_thresh, num_thresh):
    """clean_single_mesh restated with a breadth-first search over shared edges and float64 np.mean centroids."""
    faces = [tuple(int(x) for x in f) for f in faces]
    by_edge = defaultdict(list)
    for i, (a, b, c) in enumerate(faces):
        for x, y in ((a, b), (b, c), (c, a)):
            if x != y:
                by_edge[frozenset((x, y))].append(i)
    label = [-1] * len(faces)
    comps = []
    for s in range(len(faces)):
        if label[s] >= 0:
            continue
        label[s] = len(comps)
        members, todo = [s], [s]
        while todo:
            a, b, c = faces[todo.pop()]
            for x, y in ((a, b), (b, c), (c, a)):
                for g in by_edge.get(frozenset((x, y)), []) if x != y else []:
                    if label[g] < 0:
                        label[g] = len(comps)
                        members.append(g)
                        todo.append(g)
        comps.append(sorted({x for g in members for x in faces[g]}))
    counts = [len(c) for c in comps]
    keep = []
    for vs in comps:
        cen = np.mean(np.asarray(verts, np.float64)[vs], axis=0)
        keep.append(len(vs) > max(counts) * num_thresh and np.sqrt(np.sum(np.square(cen))) < dist_thresh)
    kf = [f for f, l in zip(faces, label) if keep[l]]
    used = sorted({x for f in kf for x in f})
    remap = {x: i for i, x in enumerate(used)}
    return dict(verts=np.asarray(verts, np.float32).reshape(-1, 3)[used].reshape(-1, 3),
                faces=np.array([[remap[x] for x in f] for f in kf], np.int32).reshape(-1, 3),
                labels=np.array(label, np.int32), n_components=len(comps), n_kept=int(sum(keep)))


def _assert_same(got, want):
    for k in ("verts", "faces", "labels"):
        assert got[k].shape == want[k].shape, k
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    assert (got["n_components"], got["n_kept"]) == (want["n_components"], want["n_kept"])


@pytest.mark.parametrize("name", sorted(hand_meshes()))
def test_oracle_matches_bfs_on_hand_built_meshes(name):
    v, f, d, n, expected = hand_meshes()[name]
    got = mco.clean(v, f, d, n)
    _assert_same(got, bfs_clean(v, f, d, n))
    assert (got["n_components"], got["n_kept"]) == expected


def test_hand_built_details():
    m = hand_meshes()
    got = mco.clean(*m["bowtie"][:4])
    assert list(got["counts"]) == [3, 3] and len(got["verts"]) == 5        # the shared vertex counts in both, kept once
    got = mco.clean(*m["degenerate"][:4])
    assert list(got["labels"]) == [0, 0, 1, 2, 0] and list(got["counts"]) == [3, 1, 2]
    got = mco.clean(*m["unreferenced_vertex"][:4])
    assert len(got["verts"]) == 4 and not (got["verts"] == np.float32(0.9)).all(axis=1).any()
    got = mco.clean(*m["threshold_10x0.3"][:4])
    assert list(got["counts"]) == [10, 3, 4] and len(got["faces"]) == 8 + 2
    assert mco.clean(*m["norm_equals_dist"][:4])["centroids"][0].tolist() == [0.5, 0.0, 0.0]


def _mc_mesh(R, seed):
    from oracle import mc_oracle
    sdf = np.random.default_rng(seed).standard_normal((R, R, R)).astype(np.float32)
    return mc_oracle.marching_cubes(sdf, [-1, -1, -1, 1, 1, 1], 0.0)


@pytest.mark.parametrize("num_thresh", [0.0, 0.3])
def test_oracle_matches_bfs_on_random_field_meshes(num_thresh):
    v, f = _mc_mesh(17, 17)
    got = mco.clean(v, f, 0.5, num_thresh)
    assert got["n_components"] > 20
    _assert_same(got, bfs_clean(v, f, 0.5, num_thresh))


def test_fixed_point_centroid_within_2pow32_of_mean():
    v, f = _mc_mesh(17, 17)
    got = mco.clean(v, f)
    for c in range(got["n_components"]):
        vs = np.unique(f[got["labels"] == c])
        assert len(vs) == got["counts"][c]
        assert np.abs(got["centroids"][c] - np.mean(v[vs].astype(np.float64), axis=0)).max() <= 2.0 ** -32


def test_coordinate_guard():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    mco.clean(v * np.float32(2 ** 28 - 1), [[0, 1, 2]])
    with pytest.raises(ValueError, match="2\\^30"):
        mco.clean(v * np.float32(2 ** 29), [[0, 1, 2]])
    with pytest.raises(ValueError):
        mco.clean(v, [[0, 1, 3]])


def test_read_obj_round_trips_write_obj(tmp_path):
    from disn_b200.create_sdf import read_obj, write_obj
    rng = np.random.default_rng(3)
    v = (rng.integers(-64, 65, (50, 3)) / 64.0).astype(np.float32)
    f = rng.integers(0, 50, (70, 3)).astype(np.int32)
    p = str(tmp_path / "m.obj")
    write_obj(p, v, f)
    rv, rf = read_obj(p)
    assert rv.dtype == np.float32 and rf.dtype == np.int32
    np.testing.assert_array_equal(rv, v)
    np.testing.assert_array_equal(rf, f)
    q = str(tmp_path / "t.obj")
    with open(q, "w") as fh:
        fh.write("# c\nmtllib x.mtl\nv 1 2 3\nv 4 5 6\nvn 0 0 1\nvt 0 0\nv 7 8 9\ng grp\nusemtl m\nf 1/1/1 2//1 3/2\nf 3 2 1\n")
    rv, rf = read_obj(q)
    assert rv.tolist() == [[1, 2, 3], [4, 5, 6], [7, 8, 9]] and rf.tolist() == [[0, 1, 2], [2, 1, 0]]
    with open(q, "w") as fh:
        fh.write("v 0 0 0\nv 1 0 0\nv 0 1 0\nv 1 1 0\nf 1 2 4 3\n")
    with pytest.raises(ValueError, match="triangle"):
        read_obj(q)
    write_obj(p, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    ev, ef = read_obj(p)
    assert ev.shape == (0, 3) and ef.shape == (0, 3)


def test_build_file_dict_naming(tmp_path):
    from disn_b200 import clean_smallparts as cl
    src, tar = tmp_path / "src", tmp_path / "tar"
    src.mkdir()
    names = ["03001627_abc_00.obj", "03001627_abc_01.obj", "03001627_def_07.obj"]
    for n in names:
        (src / n).write_text("")
    (src / "subdir_x_y").mkdir()                       # directories are skipped
    sd, td, sl, tl = cl.build_file_dict(str(src), str(tar))
    assert sorted(sl) == sorted(str(src / n) for n in names)
    assert [os.path.basename(t) for t in tl] == [os.path.basename(s) for s in sl]
    assert all(os.path.dirname(t) == str(tar) for t in tl)
    assert sorted(sd) == ["abc", "def"] and sorted(sd["abc"]) == [str(src / n) for n in names[:2]]
    assert sorted(td["def"]) == [str(tar / names[2])]
