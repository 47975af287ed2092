"""GPU tests of the device OBJ reader (disn_obj_read / Engine.read_obj): every array and name bit for bit equal to
create_sdf.read_obj / read_obj_parts, the fallback to them for every file outside the reader's grammar, the C ABI's
refusals, and the drivers and mesh calls that now read through it."""
import ctypes as C
import lzma
import os
import warnings

import numpy as np
import pytest

from disn_b200 import _lib
from disn_b200 import clean_smallparts as csp
from disn_b200 import create_point_sdf_grid as cpsg
from disn_b200.create_sdf import read_obj, read_obj_parts, write_obj
from disn_b200.engine import Engine
from tests.test_gpu_mesh_norm import raw_model, write_raw_obj

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if isinstance(w, np.ndarray):
            assert g.dtype == w.dtype and g.shape == w.shape
            np.testing.assert_array_equal(bits(g), bits(w))
        else:
            assert g == w


def check_device(eng, path, parts=None):
    """Engine.read_obj takes the device path and equals the Python readers."""
    for p in ((False, True) if parts is None else (parts,)):
        before = eng.obj_fallbacks
        got = eng.read_obj(str(path), parts=p)
        assert eng.obj_fallbacks == before, "fell back on " + str(path)
        same(got, read_obj_parts(str(path)) if p else read_obj(str(path)))
        same(eng.fetch_mesh(), got[:2])


@pytest.fixture(scope="module")
def eng():
    e = Engine(device=0, precision="fp32")
    yield e
    e.close()


def write_g(path, v, f):
    write_obj(str(path), v, f)


def write_9g(path, v, f):
    cpsg.write_obj_exact(str(path), v, f)


def write_18e(path, v, f):
    with open(path, "w") as fh:
        np.savetxt(fh, v, fmt="v %.18e %.18e %.18e")
        np.savetxt(fh, np.asarray(f, np.int64) + 1, fmt="f %d %d %d")


WRITERS = {"g": write_g, "9g": write_9g, "18e": write_18e}


def mesh(eng, name):
    box = [-1, -1, -1, 1, 1, 1]
    if name == "empty":
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32)
    if name == "one_triangle":
        return np.float32([[0, 0, 0], [1, -0.0, 0], [0, 1e-7, -3.5]]), np.int32([[0, 1, 2]])
    R = {"sphere_33": 33, "noise_129": 129}[name]
    if name == "sphere_33":
        ax = np.linspace(-1, 1, R)
        z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
        field = (np.sqrt(x * x + y * y + z * z) - 0.6).astype(np.float32)
    else:
        field = np.random.default_rng(129).standard_normal((R, R, R)).astype(np.float32)
    return eng.marching_cubes(field, box, 0.0)


@pytest.mark.parametrize("name", ["empty", "one_triangle", "sphere_33", "noise_129"])
def test_three_formats_equal_the_python_reader(eng, tmp_path, name):
    v, f = mesh(eng, name)
    if name == "noise_129":
        assert len(f) > 6_000_000
    for fmt, writer in WRITERS.items():
        p = tmp_path / ("m_%s.obj" % fmt)
        writer(p, v, f)
        check_device(eng, p, parts=False if name == "noise_129" else None)
        if fmt != "18e":
            assert eng.obj_read_stats()["host_tokens"] == 0, fmt
        p.unlink()


def coord_token(rng):
    k = rng.integers(0, 12)
    x = float(rng.standard_normal() * 10.0 ** rng.integers(-8, 8))
    forms = ["%g" % x, "%.9g" % x, "%.17g" % x, "%.18e" % x, "%d" % int(x * 1000), "-0", "+0.0", "00%s" % ("%g" % abs(x)),
             "+%.3f" % abs(x), ".5", "7.", "%.3E" % x, "inf", "-Infinity", "nAn"]
    return forms[int(k) % len(forms)] if k < 11 else "%.25g" % x


def random_file(rng, path):
    """A valid file mixing every record type, line end and separator, i/j/k corners, leading zeros and signs, and faces
    that refer to vertices defined later."""
    seps = [" ", "\t", "\v", "\f", "\x1c", "\x1d", "\x1e", "\x1f", "  "]
    ends = ["\n", "\r\n", "\r"]
    nv = int(rng.integers(3, 60))
    recs = []
    for _ in range(nv):
        recs.append(["v"] + [coord_token(rng) for _ in range(3)] + (["1.0"] if rng.random() < 0.2 else []))
    for _ in range(int(rng.integers(0, 80))):
        idx = rng.integers(1, nv + 1, 3)
        corner = lambda i: rng.choice(["%d", "+%d", "0%d", "%d/1", "%d//3", "%d/2/3", "%d/"]) % i
        recs.append(["f"] + [corner(int(i)) for i in idx])
    for _ in range(int(rng.integers(0, 6))):
        recs.append(["usemtl"] + ([str(rng.choice(["a", "b", "mat_1", "A"]))] if rng.random() < 0.8 else []))
    for extra in (["#", "comment", "v", "1"], ["vt", "0.5", "0.5"], ["vn", "0", "0", "1"], ["g", "grp"], ["o", "x"],
                  ["s", "off"], ["mtllib", "x.mtl"], ["v1", "2"], ["#v"], []):
        if rng.random() < 0.5:
            recs.append(extra)
    order = rng.permutation(len(recs))
    text = ""
    for i in order:
        sep = lambda: str(rng.choice(seps))
        lead = sep() if rng.random() < 0.2 else ""
        text += lead + sep().join(recs[i]) + (sep() if rng.random() < 0.2 else "") + str(rng.choice(ends))
    if rng.random() < 0.5:
        text = text.rstrip("\r\n")
    with open(path, "w", newline="") as fh:
        fh.write(text)


def test_random_corpus_equals_the_python_reader(eng, tmp_path):
    rng = np.random.default_rng(11)
    for k in range(60):
        p = tmp_path / ("r%d.obj" % k)
        random_file(rng, p)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            check_device(eng, p)


def test_reference_demo_mesh(eng, tmp_path):
    p = tmp_path / "result.obj"
    with lzma.open(os.path.join(ROOT, "tests", "golden", "demo_result.obj.xz")) as src:
        p.write_bytes(src.read())
    check_device(eng, p)
    v, f = eng.fetch_mesh()
    assert v.shape == (82584, 3) and f.shape == (165196, 3)
    assert eng.obj_read_stats()["host_tokens"] == 0


def test_parts_are_numbered_by_first_face(eng, tmp_path):
    p = tmp_path / "m.obj"
    p.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nusemtl b\nusemtl a\nf 1 2 3\nusemtl b\nf 1 2 3\nusemtl a\nf 3 2 1\n"
                 "usemtl\nf 1 2 3\n")
    check_device(eng, p, parts=True)
    _, _, pid, names = eng.read_obj(str(p), parts=True)
    assert names == ["a", "b", ""] and pid.tolist() == [0, 1, 0, 2]
    p.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3\nusemtl m\nf 1 2 3\n")
    _, _, pid, names = eng.read_obj(str(p), parts=True)
    assert names == [None, "m"] and pid.tolist() == [0, 1]
    check_device(eng, p, parts=True)


def test_overflow_warns_as_the_cast_does(eng, tmp_path):
    p = tmp_path / "m.obj"
    p.write_text("v 1e39 1e400 -1e-400\nv 0 0 0\nv 1 1 1\nf 1 2 3\n")
    with pytest.warns(RuntimeWarning, match="overflow encountered in cast"):
        got = eng.read_obj(str(p))
    with pytest.warns(RuntimeWarning, match="overflow encountered in cast"):
        want = read_obj(str(p))
    same(got, want)
    assert eng.obj_read_stats()["overflows"] == 1


FALLBACKS = {
    "bom": b"\xef\xbb\xbfv 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3\n",
    "non_ascii_name": "v 0 0 0\nv 1 0 0\nv 0 1 0\nusemtl métal\nf 1 2 3\n".encode(),
    "underscore": b"v 1_0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3\n",
    "quad": b"v 0 0 0\nv 1 0 0\nv 0 1 0\nv 1 1 0\nf 1 2 3 4\n",
    "two_coordinates": b"v 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3\n",
    "index_zero": b"v 0 0 0\nv 1 0 0\nv 0 1 0\nf 0 2 3\n",
    "index_negative": b"v 0 0 0\nv 1 0 0\nv 0 1 0\nf -1 2 3\n",
    "index_past_v": b"v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 4\n",
    "empty_index": b"v 0 0 0\nv 1 0 0\nv 0 1 0\nf /2 2 3\n",
    "hex": b"v 0x1 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3\n",
}


def python_result(fn, path):
    try:
        return "ok", fn(path)
    except Exception as e:
        return "raise", (type(e), str(e))


@pytest.mark.parametrize("case", sorted(FALLBACKS) + ["missing"])
@pytest.mark.parametrize("parts", [False, True])
def test_fallback_inputs_give_the_python_result(eng, tmp_path, case, parts):
    p = str(tmp_path / "m.obj")
    if case != "missing":
        with open(p, "wb") as fh:
            fh.write(FALLBACKS[case])
    fn = read_obj_parts if parts else read_obj
    kind, want = python_result(fn, p)
    before = eng.obj_fallbacks
    gkind, got = python_result(lambda q: eng.read_obj(q, parts=parts), p)
    assert eng.obj_fallbacks == before + 1
    assert gkind == kind
    if kind == "ok":
        same(got, want)
    else:
        assert got == want


def test_c_abi_refusals_name_path_and_line_and_empty_the_mesh(eng, tmp_path):
    lib = eng.lib
    for case, line, what in [("quad", 5, "only triangle faces are supported, found 4 corners"),
                             ("index_past_v", 4, "face index"), ("underscore", 1, "coordinate"),
                             ("non_ascii_name", 4, "non-ASCII"), ("two_coordinates", 1, "fewer than 3")]:
        p = str(tmp_path / (case + ".obj"))
        with open(p, "wb") as fh:
            fh.write(FALLBACKS[case])
        eng.load_mesh(np.eye(3, dtype=np.float32), np.int32([[0, 1, 2]]))
        nv, nf, np_ = C.c_int64(-1), C.c_int64(-1), C.c_int32(-1)
        rc = lib.disn_obj_read(eng._h, p.encode(), 0, C.byref(nv), C.byref(nf), C.byref(np_))
        msg = lib.disn_last_error().decode()
        assert rc == _lib.DISN_ERR_OBJ_UNSUPPORTED, (case, rc, msg)
        assert msg.startswith("%s:%d: " % (p, line)) and what in msg, (case, msg)
        assert (nv.value, nf.value) == (0, 0)
        assert eng.mesh_counts() == (0, 0)
        v, f = np.empty((0, 3), np.float32), np.empty((0, 3), np.int32)
        _lib.check(lib.disn_mc_fetch(eng._h, v.ctypes.data_as(C.c_void_p), f.ctypes.data_as(C.c_void_p)))
        clean = eng.clean_mesh(fetch=False)
        assert (clean.n_verts, clean.n_faces) == (0, 0)
    rc = lib.disn_obj_read(eng._h, str(tmp_path / "missing.obj").encode(), 0, None, None, None)
    assert rc == _lib.DISN_ERR_OBJ_UNSUPPORTED and "missing.obj" in lib.disn_last_error().decode()


def test_mesh_calls_after_the_device_read_equal_them_after_load_mesh(tmp_path):
    v, f, pid = raw_model()
    model = str(tmp_path / "raw" / "model.obj")
    write_raw_obj(model, v, f, pid)
    outs = []
    for device in (True, False):
        e = Engine(device=0, precision="fp32")
        try:
            def load():
                if device:
                    e.read_obj(model, parts=True)
                else:
                    rv, rf, _, _ = read_obj_parts(model)
                    e.load_mesh(rv, rf)
            _, _, rp, names = read_obj_parts(model)
            load()
            clean = e.clean_mesh(0.5, 0.3, want_labels=True)
            load()
            q = e.part_areas(rp, len(names))
            np.random.seed(3)
            norm = cpsg.normalize_resident(e, rp, len(names), want_samples=True)
            nmesh = e.fetch_mesh()
            load()
            grid, bbox = e.mesh_sdf(128)
            obj = str(tmp_path / ("w%d.obj" % device))
            e.write_mesh_obj(obj)
            with open(obj, "rb") as fh:
                outs.append((clean, q, norm, nmesh, grid, bbox, fh.read()))
        finally:
            e.close()
    a, b = outs
    for x, y in zip(a, b):
        if isinstance(x, bytes):
            assert x == y
        elif isinstance(x, tuple):
            for xx, yy in zip(x, y):
                np.testing.assert_array_equal(bits(np.asarray(xx)), bits(np.asarray(yy)))
        else:
            np.testing.assert_array_equal(bits(np.asarray(x)), bits(np.asarray(y)))


def python_reader(self, path, parts=False, load=False):
    mesh = read_obj_parts(path) if parts else read_obj(path)
    if load:
        self.load_mesh(mesh[0], mesh[1])
    return mesh


def test_drivers_write_the_same_files_through_either_reader(tmp_path, monkeypatch):
    v, f, pid = raw_model()
    cat, obj = "02691156", "obj_a"
    model = str(tmp_path / "mesh" / cat / obj / "model.obj")
    write_raw_obj(model, v, f, pid)
    src = str(tmp_path / "src.obj")
    write_obj(src, v, f)

    def run(tag):
        out = tmp_path / tag
        out.mkdir()
        csp.clean_single_mesh(src, str(out / "clean.obj"), 0.5, 0.3)
        csp.separate_single_mesh(src, str(out / "sep"))
        e = Engine(device=0, precision="fp32")
        try:
            np.random.seed(21)
            cpsg.create_sdf_obj(None, None, str(tmp_path / "mesh" / cat), str(out / "norm" / cat), str(out / "sdf" / cat),
                                obj, 32, 0.003, 1.2, 0, True, True, 2000, 0.1, 16384, cat, 0.0, 1, False, engine=e,
                                keep_dist=True)
            cpsg.create_one_sdf(None, 32, 1.2, str(out / "one.dist"), model, 0, engine=e)
            fallbacks = e.obj_fallbacks
        finally:
            e.close()
        files = {}
        for root, _, names in os.walk(out):
            for n in names:
                full = os.path.join(root, n)
                files[os.path.relpath(full, out)] = (np.load(full) if n.endswith(".npz") else open(full, "rb").read())
        return files, fallbacks

    dev, nfb = run("device")
    assert nfb == 0
    monkeypatch.setattr(Engine, "read_obj", python_reader)
    host, _ = run("python")
    assert sorted(dev) == sorted(host) and len(dev) > 6
    for k in dev:
        if isinstance(dev[k], bytes):
            assert dev[k] == host[k], k
        else:
            for a in dev[k].files:
                np.testing.assert_array_equal(dev[k][a], host[k][a])


def test_eval_drivers_read_through_the_device_reader(eng, tmp_path, monkeypatch):
    from disn_b200 import eval_iou
    from disn_b200.eval_common import read_mesh
    v, f = mesh(eng, "sphere_33")
    p = str(tmp_path / "m.obj")
    write_obj(p, v, f)
    calls = []
    monkeypatch.setattr(eng, "read_obj", lambda path: calls.append(path) or Engine.read_obj(eng, path))
    monkeypatch.setattr(eval_iou, "_engine", lambda: eng)
    before = eng.obj_fallbacks
    same(eval_iou._read_mesh(p), read_obj(p))
    same(read_mesh(eng, p), read_obj(p))
    assert calls == [p, p] and eng.obj_fallbacks == before
    same(read_mesh(object(), p), read_obj(p))       # an engine without a device reader reads with the Python reader
