"""GPU tests of the surface-sample normalisation (disn_mesh_part_areas / disn_mesh_normalize) against the CPU twin
oracle/mesh_norm_oracle.py bit for bit, of the band and strided field samplers against the host sample_sdf and numpy, and
of the per-object chain (create_sdf_obj, create_sdf) against its separately called steps."""
import os
import time

import numpy as np
import pytest

from disn_b200 import create_point_sdf_fullgrid as fullgrid
from disn_b200 import create_point_sdf_grid as cpsg
from disn_b200._lib import DisnError
from disn_b200.create_sdf import read_obj_parts
from oracle import mesh_norm_oracle as no
from tests.test_gpu_mesh_sdf import predicted_mesh, soup  # noqa: F401  (module fixture reused by import)
from tests.test_mesh_sdf_cpu import CUBE_F, CUBE_V, analytic_mesh

pytestmark = pytest.mark.gpu


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


def two_material():
    sv, sf = analytic_mesh("sphere", 21)
    tv, tf = analytic_mesh("torus", 25)
    v = np.concatenate([sv * np.float32(0.5) - np.float32(0.4), tv + np.float32(0.3)]).astype(np.float32)
    f = np.concatenate([sf, tf + len(sv)]).astype(np.int32)
    pid = np.concatenate([np.zeros(len(sf), np.int32), np.ones(len(tf), np.int32)])
    perm = np.random.default_rng(1).permutation(len(f))
    return v, f[perm], pid[perm], 2


def with_zero_area_faces():
    v, f = analytic_mesh("sphere", 17)
    z = np.stack([f[:, 0], f[:, 0], f[:, 1]], axis=1)[::3]              # repeated-vertex faces: zero area
    return v, np.concatenate([z[:40], f, z[40:]]).astype(np.int32)


def cases():
    tv, tf = analytic_mesh("torus", 33)
    return {
        "sphere": (*analytic_mesh("sphere", 33), None, 1),
        "torus_x7_offcentre": ((tv * np.float32(7) + np.float32([3.5, -2.0, 1.25])).astype(np.float32), tf, None, 1),
        "soup": (*soup(), None, 1),
        "two_material": two_material(),
        "zero_area_faces": (*with_zero_area_faces(), None, 1),
        "single_face": (np.array([[0.1, 0.2, 0.3], [1.5, 0.2, -0.4], [0.3, 2.0, 0.7]], np.float32),
                        np.array([[0, 1, 2]], np.int32), None, 1),
    }


CASES = cases()


def check_against_twin(eng, v, f, pid, P, seed):
    eng.load_mesh(v, f)
    q, s = eng.part_areas(pid, P)
    scan = no.part_scan(v, f, pid, P)
    assert q.tolist() == scan["q"] and s == scan["shift"]
    amts = no.amounts(q)
    np.random.seed(seed)
    draws = cpsg.surface_draws(amts)
    c, m, smp = eng.normalize_mesh(pid, P, amts, draws, want_samples=True)
    tc, tm, tp, tv = no.normalize(v, f, pid, P, amts, draws)
    np.testing.assert_array_equal(bits(smp), bits(tp))
    np.testing.assert_array_equal(bits(c), bits(tc))
    assert bits(np.float64(m)) == bits(np.float64(tm))
    gv, gf = eng.fetch_mesh()
    np.testing.assert_array_equal(bits(gv), bits(tv))
    np.testing.assert_array_equal(gf, f)
    return c, m, smp, gv


@pytest.mark.parametrize("name", sorted(CASES))
def test_normalize_bit_exact_against_twin(engine, name):
    v, f, pid, P = CASES[name]
    check_against_twin(engine, v, f, pid, P, 3)


def test_normalize_829k_marching_cubes_mesh(engine, predicted_mesh):  # noqa: F811
    v, f, _, _ = predicted_mesh
    assert len(f) > 5 * 10 ** 5
    check_against_twin(engine, v, f, None, 1, 4)


def test_normalize_6m_noise_mesh_deep_scan(engine):
    noise = np.random.default_rng(129).standard_normal((129, 129, 129)).astype(np.float32)
    v, f = engine.marching_cubes(noise, [-1, -1, -1, 1, 1, 1], 0.0)
    assert len(f) > 6 * 10 ** 6
    pid = (np.arange(len(f)) % 3 == 0).astype(np.int32)             # two interleaved parts
    check_against_twin(engine, v, f, pid, 2, 5)


def test_run_to_run_deterministic(engine):
    v, f, pid, P = CASES["two_material"]
    a = check_against_twin(engine, v, f, pid, P, 6)
    b = check_against_twin(engine, v, f, pid, P, 6)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(bits(np.asarray(x)), bits(np.asarray(y)))


def test_given_params_only_transform(engine):
    v, f, _, _ = CASES["sphere"]
    engine.load_mesh(v, f)
    c, m = engine.normalize_mesh(given=[0.25, -0.5, 1.0, 1.75])
    assert c.tolist() == [0.25, -0.5, 1.0] and m == 1.75
    np.testing.assert_array_equal(bits(engine.fetch_mesh()[0]), bits(no.transform(v, [0.25, -0.5, 1.0], 1.75)))


def test_errors_leave_mesh_and_context_usable():
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="fp32")
    try:
        with pytest.raises(DisnError, match="no resident mesh"):
            eng.part_areas()
        eng.load_mesh(CUBE_V, np.zeros((0, 3), np.int32))
        with pytest.raises(DisnError, match="no resident mesh"):
            eng.normalize_mesh(None, 1, [0], np.zeros((0, 3)))
        v, f = CUBE_V * np.float32(0.5), CUBE_F
        one = np.full((16384, 3), 0.5)

        def expect(msg, verts=v, faces=f, **kw):
            eng.load_mesh(verts, faces)
            before = eng.fetch_mesh()
            with pytest.raises(DisnError, match=msg):
                eng.normalize_mesh(**kw)
            after = eng.fetch_mesh()
            np.testing.assert_array_equal(bits(after[0]), bits(before[0]))
            np.testing.assert_array_equal(after[1], before[1])

        nan = v.copy()
        nan[2, 1] = np.nan
        expect("non-finite", verts=nan, amounts=[16384], draws=one)
        with pytest.raises(DisnError, match="non-finite"):
            eng.part_areas()
        expect("part id", part_ids=np.full(len(f), 2, np.int32), n_parts=2, amounts=[1, 1], draws=one[:2])
        expect("draws for", amounts=[16384], draws=one[:100])
        expect("negative", amounts=[-1], draws=one[:0])
        expect(r"\[0, 1\)", amounts=[16384], draws=np.full((16384, 3), 1.0))
        flat = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0]], np.float32)
        expect("zero area", verts=flat, faces=[[0, 1, 2]], amounts=[5], draws=one[:5])
        expect("no samples", verts=flat, faces=[[0, 1, 2]], amounts=[0], draws=one[:0])
        expect("2\\^30", verts=v * np.float32(1e6), amounts=[16384], draws=one)
        tri = np.array([[0.5, 0.25, 1.0], [1.5, 0.25, 1.0], [0.5, 1.25, 1.0]], np.float32)
        expect("m = 0", verts=tri, faces=[[0, 1, 2]], amounts=[8], draws=np.stack([np.full(8, 0.3), np.zeros(8),
                                                                                    np.zeros(8)], axis=1))
        expect("given", given=[0, 0, 0, 0.0])
        expect("given", given=[0, np.inf, 0, 1.0])
        # the context still normalises bit for bit
        check_against_twin(eng, v, f, None, 1, 7)
    finally:
        eng.close()


# ---- band and strided samplers -------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["centred_plane", "shifted_car", "chair_iso", "short_band"])
def test_band_sampler_equals_host_sample_sdf_on_golden(engine, golden, case):
    from tests.golden.make_golden_sample_sdf import CASES as SCASES
    g = golden["sample_sdf"]
    _, _, _, cat, n, bw, iso, seed = [c for c in SCASES if c[0] == case][0]
    res, val = int(g["res"]), g[case + "_value"]
    np.random.seed(seed)
    host, _ = cpsg.sample_sdf(cat, n, bw, iso, {"param": g["param"], "value": val}, res)
    np.random.seed(seed)
    dev = engine.band_samples(n, bw, iso, g["param"], res, sdf=val)
    np.testing.assert_array_equal(bits(dev), bits(host))
    np.testing.assert_array_equal(bits(dev), bits(g[case + "_samples"]))


def test_band_sampler_on_the_257_field_of_the_829k_mesh(engine, predicted_mesh):  # noqa: F811
    v, f, _, _ = predicted_mesh
    engine.load_mesh(v, f)
    ptr = engine.field_buffer(257)
    _, bbox = engine.mesh_sdf(256, device_ptr=ptr)
    field = engine.fetch(ptr, (257, 257, 257))
    params = np.float32(bbox)
    for iso, seed in ((0.003, 8), (0.0, 9)):
        np.random.seed(seed)
        t0 = time.perf_counter()
        host, flag = cpsg.sample_sdf("02691156", 32768, 0.1, iso, {"param": params, "value": field}, 256)
        t1 = time.perf_counter()
        np.random.seed(seed)
        dev = engine.band_samples(32768, 0.1, iso, params, 256, device_ptr=ptr)
        t2 = time.perf_counter()
        np.testing.assert_array_equal(bits(dev), bits(host))
        assert len(dev) == 32768
        print("257^3 band sampling: host %.1f ms, device %.1f ms (counts %s)" % ((t1 - t0) * 1e3, (t2 - t1) * 1e3,
                                                                             engine.last_band_counts.tolist()))
        idx = cpsg.insideout_index(256, params)
        assert bool(engine.fetch(ptr + 4 * idx, (1,))[0] > 0) == bool(flag)


@pytest.mark.parametrize("reduce", [1, 3, 8])
def test_strided_sampler_equals_numpy(engine, reduce):
    v, f, _, _ = CASES["torus_x7_offcentre"]
    engine.load_mesh(v, f)
    R = 65
    ptr = engine.field_buffer(R)
    _, bbox = engine.mesh_sdf(R - 1, device_ptr=ptr)
    field = engine.fetch(ptr, (R, R, R))
    want = no.strided(field, reduce)
    np.testing.assert_array_equal(bits(engine.sdf_strided(R, reduce, device_ptr=ptr)), bits(want))
    np.testing.assert_array_equal(bits(engine.sdf_strided(R, reduce, sdf=field)), bits(want))
    vals, flag = fullgrid.sample_sdf("02958343", 0, 0.1, 0.0, {"param": np.float32(bbox), "value": field}, R - 1, reduce,
                                     engine=engine)
    np.testing.assert_array_equal(bits(vals.reshape(-1)), bits(want.reshape(-1)))


def test_band_gather_errors():
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="fp32")
    try:
        k = np.zeros(4, np.int64)
        k[0] = 1
        ax = np.zeros(3 * 8, np.float32)
        ch = np.zeros(1, np.int64)
        import ctypes as C
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        out = np.zeros((1, 4), np.float32)
        from disn_b200._lib import check
        with pytest.raises(DisnError, match="band_count first"):
            check(eng.lib.disn_sdf_band_gather(eng._h, p(ax), p(ch), p(k), p(out)))
        field = np.linspace(-0.2, 0.2, 8 ** 3).astype(np.float32)
        counts = np.zeros(4, np.int64)
        edges = no.band_edges(0.1)
        check(eng.lib.disn_sdf_band_count(eng._h, p(field), 8, 0.0, p(edges), 0, p(counts)))
        ch[0] = counts[0]
        with pytest.raises(DisnError, match="outside band 0"):
            check(eng.lib.disn_sdf_band_gather(eng._h, p(ax), p(ch), p(k), p(out)))
        np.random.seed(1)
        dev = eng.band_samples(100, 0.1, 0.0, [-1, -1, -1, 1, 1, 1], 7, sdf=field)
        np.random.seed(1)
        want = no.sample_sdf(100, 0.1, 0.0, np.float32([-1, -1, -1, 1, 1, 1]), 7, field)
        np.testing.assert_array_equal(bits(dev), bits(want))
    finally:
        eng.close()


# ---- the per-object chain and the batch driver ----------------------------------------------------------------------
def write_raw_obj(path, v, f, pid, names=("body", "wheel")):
    """Raw OBJ with one usemtl run per maximal run of equal part ids (materials recur, as in ShapeNet models)."""
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as fh:
        for x in v:
            fh.write("v %.9g %.9g %.9g\n" % tuple(x))
        cur = None
        for tri, p in zip(f, pid):
            if p != cur:
                fh.write("usemtl %s\n" % names[p])
                cur = p
            fh.write("f %d/1 %d/1 %d/1\n" % tuple(tri + 1))


def raw_model():
    v, f, pid, _ = two_material()
    v = (v * np.float32(3.0) + np.float32([10.0, -4.0, 2.5])).astype(np.float32)
    return v, f, pid


def test_create_sdf_obj_equals_the_separate_steps(engine, tmp_path):
    v, f, pid = raw_model()
    cat, obj, res, iso = "02691156", "obj_a", 32, 0.003
    model = str(tmp_path / "mesh" / cat / obj / "model.obj")
    write_raw_obj(model, v, f, pid)
    # the separate steps, each through its file
    sep = tmp_path / "sep"
    sep.mkdir()
    np.random.seed(21)
    norm_obj, c, m = cpsg.get_normalize_mesh(model, str(sep), engine=engine)
    sdf_file, cube = str(sep / "isosurf.sdf"), str(sep / "isosurf.obj")
    cpsg.create_one_sdf(None, res, 1.2, sdf_file, norm_obj, 0, g=0.0, engine=engine)
    cpsg.create_one_cube_obj(None, iso, sdf_file, cube, engine=engine)
    cpsg.create_h5_sdf_pt(cat, str(sep / "ori_sample.npz"), sdf_file, str(sep / "isinsideout.txt"), cube, norm_obj, c, m,
                          res, 2000, 0.1, iso, 16384, True, engine=engine)
    # the chain
    np.random.seed(21)
    out = cpsg.create_sdf_obj(None, None, str(tmp_path / "mesh" / cat), str(tmp_path / "norm" / cat),
                              str(tmp_path / "sdf" / cat), obj + "\n", res, iso, 1.2, 0, True, True, 2000, 0.1, 16384, cat,
                              0.0, 1, False, engine=engine, keep_dist=True)
    chain_norm, chain_sdf = tmp_path / "norm" / cat / obj, tmp_path / "sdf" / cat / obj
    assert out == str(chain_sdf / "ori_sample.npz")
    for a, b in ((sep / "pc_norm.obj", chain_norm / "pc_norm.obj"), (sep / "isosurf.obj", chain_norm / "isosurf.obj"),
                 (sep / "isosurf.sdf", chain_sdf / "isosurf.sdf")):
        assert a.read_bytes() == b.read_bytes(), b.name
    za, zb = np.load(str(sep / "ori_sample.npz")), np.load(out)
    assert sorted(za.files) == sorted(zb.files) == ["norm_params", "pc_sdf_original", "pc_sdf_sample", "sdf_params"]
    for k in za.files:
        assert za[k].dtype == zb[k].dtype
        np.testing.assert_array_equal(za[k], zb[k])
    assert zb["norm_params"].dtype == np.float64 and zb["pc_sdf_sample"].shape == (2000, 4)
    assert os.path.exists(chain_sdf / "isinsideout.txt") == os.path.exists(sep / "isinsideout.txt")
    # the normalised mesh equals the twin's
    rv, rf, rp, names = read_obj_parts(model)
    np.random.seed(21)
    scan = no.part_scan(rv, rf, rp, len(names))
    amts = no.amounts(scan["q"])
    tc, tm, _, tv = no.normalize(rv, rf, rp, len(names), amts, cpsg.surface_draws(amts))
    nv, _, _, _ = read_obj_parts(str(chain_norm / "pc_norm.obj"))
    np.testing.assert_array_equal(bits(nv), bits(tv))
    np.testing.assert_array_equal(zb["norm_params"], np.concatenate([tc, [np.float32(tm)]]))
    # the fullgrid variant: the largest part with the grid run's norm_params
    fobj, fc, fm = fullgrid.get_normalize_mesh(model, out, cat, obj, str(tmp_path), engine=engine)
    big = int(np.argmax(scan["q"]))
    keep = rp == big
    used = np.unique(rf[keep])
    gv, _, _, _ = read_obj_parts(fobj)
    np.testing.assert_array_equal(bits(gv), bits(no.transform(rv[used], fc, fm)))


def test_batch_driver_on_a_two_category_tree(tmp_path):
    v, f, pid = raw_model()
    sv, sf = analytic_mesh("sphere", 21)
    tree = {"02958343": ["car_1", "car_2"], "03001627": ["chair_1"]}
    lst = tmp_path / "lst"
    lst.mkdir()
    for cat, objs in tree.items():
        (lst / (cat + "_test.lst")).write_text(objs[0] + "\n")
        (lst / (cat + "_train.lst")).write_text("".join(o + "\n" for o in objs[1:]))
        for o in objs:
            if o == "car_2":
                write_raw_obj(str(tmp_path / "mesh" / cat / o / "model.obj"), sv, sf, np.zeros(len(sf), np.int32))
            else:
                write_raw_obj(str(tmp_path / "mesh" / cat / o / "model.obj"), v, f, pid)
    args = ["--mesh_dir", str(tmp_path / "mesh"), "--lst_dir", str(lst), "--sdf_dir", str(tmp_path / "sdf"),
            "--norm_mesh_dir", str(tmp_path / "norm"), "--cats", "02958343", "03001627", "--res", "32",
            "--num_sample", "1000", "--seed", "3"]
    cpsg.main(args)
    for cat, objs in tree.items():
        for o in objs:
            for p in (tmp_path / "norm" / cat / o / "pc_norm.obj", tmp_path / "norm" / cat / o / "isosurf.obj"):
                assert p.stat().st_size > 1000, p
            z = np.load(str(tmp_path / "sdf" / cat / o / "ori_sample.npz"))
            assert z["pc_sdf_sample"].shape == (1000, 4) and z["norm_params"].shape == (4,)
            assert z["sdf_params"].dtype == np.float32
    stamp = os.path.getmtime(tmp_path / "sdf" / "03001627" / "chair_1" / "ori_sample.npz")
    raw_dirs = {"mesh_dir": str(tmp_path / "mesh"), "sdf_dir": str(tmp_path / "sdf"), "norm_mesh_dir": str(tmp_path / "norm")}
    done = cpsg.create_sdf(None, None, None, 1000, 0.1, 32, 1.2, {"chair": "03001627"}, raw_dirs, str(lst), 0.003, 16384,
                           version=1, skip_all_exist=True)
    assert done == [] and os.path.getmtime(tmp_path / "sdf" / "03001627" / "chair_1" / "ori_sample.npz") == stamp


def test_band_count_refuses_overlapping_or_nan_edges():
    """The four index lists share one buffer of R^3 entries, so the bands must be disjoint; the context stays usable."""
    import ctypes as C
    from disn_b200._lib import check
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="fp32")
    try:
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        field = np.linspace(-0.5, 0.5, 9 ** 3).astype(np.float32)
        counts = np.zeros(4, np.int64)

        def count(edges):
            e = np.ascontiguousarray(edges, np.float32).reshape(4, 2)
            check(eng.lib.disn_sdf_band_count(eng._h, p(field), 9, 0.0, p(e), 0, p(counts)))
            return counts.tolist()

        for bad, msg in [([[-1, 1]] * 4, "overlap"), ([[-1, 0], [-0.5, 0.5], [1, 2], [2, 3]], "bands 0 and 1 overlap"),
                         ([[-1, 0], [0, 1], [1, 2], [1.5, 1.6]], "bands 2 and 3 overlap"),
                         ([[-1, 0], [0, np.nan], [1, 2], [2, 3]], "NaN")]:
            with pytest.raises(DisnError, match=msg):
                count(bad)
        # touching and empty intervals are disjoint: every point lands in exactly one band
        assert sum(count([[-1, -0.25], [-0.25, 0], [0, 1], [0.5, 0.5]])) == 9 ** 3
        assert sum(count([[0.3, -0.3], [-1, 0], [0, 1], [5, 4]])) == 9 ** 3
        np.random.seed(2)
        dev = eng.band_samples(400, 0.3, 0.0, [-1, -1, -1, 1, 1, 1], 8, sdf=field)
        np.random.seed(2)
        np.testing.assert_array_equal(bits(dev), bits(no.sample_sdf(400, 0.3, 0.0, np.float32([-1, -1, -1, 1, 1, 1]), 8,
                                                                      field)))
    finally:
        eng.close()


def test_normalize_refuses_bad_part_counts_and_amounts_before_sizing():
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="fp32")
    try:
        v, f = CUBE_V * np.float32(0.5), CUBE_F
        eng.load_mesh(v, f)
        with pytest.raises(DisnError, match="n_parts <= n_faces"):
            eng.part_areas(np.zeros(len(f), np.int32), len(f) + 1)
        with pytest.raises(DisnError, match="n_parts <= n_faces"):
            eng.normalize_mesh(np.zeros(len(f), np.int32), 10 ** 6, [1] + [0] * (10 ** 6 - 1), np.full((1, 3), 0.5))
        with pytest.raises(DisnError, match="exceeds 2\\^31 - 1"):
            eng.normalize_mesh(None, 1, [2 ** 40], np.full((1, 3), 0.5))
        with pytest.raises(DisnError, match="draws for"):
            eng.normalize_mesh(None, 1, [16384], np.full((10, 3), 0.5))
        np.testing.assert_array_equal(bits(eng.fetch_mesh()[0]), bits(v))
        check_against_twin(eng, v, f, None, 1, 8)
    finally:
        eng.close()


def test_fetch_mesh_returns_the_vertices_of_a_mesh_without_faces(engine):
    v = np.random.default_rng(3).standard_normal((17, 3)).astype(np.float32)
    engine.load_mesh(v, np.zeros((0, 3), np.int32))
    gv, gf = engine.fetch_mesh()
    np.testing.assert_array_equal(bits(gv), bits(v))
    assert gf.shape == (0, 3)
