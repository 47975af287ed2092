"""Generate tests/golden/eval_ref.npz by running the REFERENCE's own evaluation scripts (test/test_cd_emd.py,
test/test_f_score.py, test/test_iou.py) on a small seeded fixture dataset, through make_golden.py-style module stubs.

Run in the build container only (the GPU machine has no reference tree):
    python tests/golden/make_golden_eval.py
Stubs (TF 1.x, the compiled tf_ops and PyMesh do not run here):
  * tensorflow: placeholder / tile / expand_dims / reduce_mean / reduce_min / argmin / sqrt / reshape build a small lazy
    graph, and Session.run evaluates it with numpy -- so the reference's own get_points_loss / get_points_distance run;
  * tf_nndistance.nn_distance, tf_approxmatch.approx_match / match_cost: the CPU twins of oracle/metrics_oracle.py;
  * pymesh.load_mesh: the OBJ's vertices parsed as float64; pymesh.VoxelGrid: the twin's occupied cells as a voxel mesh
    (oracle/eval_oracle.py), so that the reference's own binning line runs on its vertices;
  * joblib: sequential; create_file_lst: the fixture's directories.
os.listdir is sorted while the reference runs (the drivers list in sorted order; see disn_b200/eval_common.py).

The fixture: 2 categories x 3 objects x 4 views (--view_num 4, --num_sample_points 256) of marching-cubes meshes of
analytic fields (oracle/mc_oracle.py); one view is a file of at most 200 bytes and one is empty, so two objects have fewer
usable IoU files than view_num.  Recorded, for batch_size = view_num and batch_size = 1: every np.random.randint draw,
every random.sample choice, the lines the scripts print (fixture root replaced by <root>), the numbers in them, the
saved point files, and the F-score lines of the computed and of the cached path.  Only the data is committed.
"""
import contextlib
import importlib.util
import io
import os
import random
import re
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
from make_golden import _stub  # noqa: E402
from oracle import eval_oracle as eo  # noqa: E402
from oracle import mc_oracle  # noqa: E402
from oracle import metrics_oracle as mo  # noqa: E402

CATS = {"display": "03211117", "rifle": "04090263"}
VIEW_NUM, NPTS, DIM, TRUETHRESHOLD = 4, 256, 110, 2.5
SEEDS = {"cd_emd": 11, "save_pnt": 12, "iou": 13}
# the result lines the three scripts print (their debug prints of shapes and paths are not compared)
LINE_PATTERN = (r"^(1  .* avg cf:|cat_nm:|cat_id \d+, obj_id|[a-z]+, \d+, precision_avg|pre_w_avg|obj_id iou avg:|"
                r"saved gt pnt of)")


# ---------------------------------------------------------------------------------------------------------------- fixture
def _field_mesh(R, centre, radii, twist):
    ax = np.linspace(-1, 1, R)
    z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
    x, y, z = x - centre[0], y - centre[1], z - centre[2]
    f = np.sqrt((x / radii[0]) ** 2 + (y / radii[1]) ** 2 + (z / radii[2]) ** 2) - 1.0 + twist * np.sin(4 * x) * np.cos(3 * y)
    v, fc = mc_oracle.marching_cubes(f.astype(np.float32), [-1, -1, -1, 1, 1, 1], 0.0)
    return v.astype(np.float32), fc.astype(np.int32)


def _obj_text(v, f):
    return "".join("v %.6f %.6f %.6f\n" % tuple(p) for p in v) + "".join("f %d %d %d\n" % tuple(t + 1) for t in f)


def fixture_files():
    """relative path -> file bytes of the fixture tree (gt/, pred/, lst/)."""
    rng = np.random.default_rng(2024)
    files = {}
    for ci, (cat_nm, cat_id) in enumerate(CATS.items()):
        objs = ["%s%02d" % ("abcdef"[ci * 3 + k], 10 + ci * 3 + k) for k in range(3)]
        files["lst/%s_test.lst" % cat_id] = "".join(o + "\n" for o in objs).encode()
        for k, obj in enumerate(objs):
            centre = rng.uniform(-0.1, 0.1, 3)
            radii = rng.uniform(0.3, 0.55, 3)
            twist = rng.uniform(0.0, 0.1)
            v, f = _field_mesh(21, centre, radii, twist)
            files["gt/%s/%s/isosurf.obj" % (cat_id, obj)] = _obj_text(v, f).encode()
            for view in range(VIEW_NUM):
                name = "pred/%s/%s_%s_%02d.obj" % (cat_id, cat_id, obj, view)
                if ci == 0 and k == 1 and view == 2:         # a file of at most 200 bytes: one triangle
                    files[name] = _obj_text(np.array([[0, 0, 0], [0.1, 0, 0], [0, 0.1, 0]], np.float32),
                                            np.array([[0, 1, 2]])).encode()
                    continue
                if ci == 1 and k == 2 and view == 0:         # an empty file
                    files[name] = b""
                    continue
                R = int(rng.integers(11, 20))
                vv, ff = _field_mesh(R, centre + rng.uniform(-0.04, 0.04, 3), radii * rng.uniform(0.9, 1.1, 3),
                                     twist * rng.uniform(0.5, 1.5))
                files[name] = _obj_text(vv, ff).encode()
    return files


def write_tree(root, files):
    for rel, data in files.items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as fh:
            fh.write(data)


# ------------------------------------------------------------------------------------------------------------- TF stub
class _Shape:
    def __init__(self, dims):
        self.dims = dims

    def as_list(self):
        return list(self.dims) if self.dims is not None else None

    def __str__(self):
        return str(tuple(self.dims)) if self.dims is not None else "<unknown>"


class Node:
    def __init__(self, fn, *args, shape=None):
        self.fn, self.args, self.shape = fn, args, shape

    def __getitem__(self, key):
        return Node(lambda x: x[key], self)

    def __add__(self, other):
        return Node(lambda x, y: x + y, self, other)

    def __mul__(self, other):
        return Node(lambda x, y: x * y, self, other)

    __rmul__ = __mul__

    def get_shape(self):
        return _Shape(self.shape)


def _evaluate(node, feed, memo):
    if not isinstance(node, Node):
        return node
    if node in feed:
        return feed[node]
    if id(node) not in memo:
        memo[id(node)] = node.fn(*[_evaluate(a, feed, memo) for a in node.args])
    return memo[id(node)]


class _Session:
    def __init__(self, config=None):
        pass

    def run(self, fetches, feed_dict=None):
        memo = {}
        feed = {k: np.asarray(v, np.float32) for k, v in (feed_dict or {}).items()}
        return [_evaluate(f, feed, memo) for f in fetches]


class _Ctx:
    def __init__(self, *a, **k):
        pass

    def as_default(self):
        return self

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def _multi(fn, n, *args):
    base = Node(fn, *args)
    return tuple(Node(lambda t, i=i: t[i], base) for i in range(n))


def install_stubs():
    tf = _stub("tensorflow", float32=np.float32, Graph=_Ctx, device=_Ctx, Session=_Session,
               ConfigProto=lambda: types.SimpleNamespace(gpu_options=types.SimpleNamespace()),
               placeholder=lambda dtype, shape: Node(None, shape=shape),
               tile=lambda x, reps: Node(lambda a: np.tile(a, reps), x),
               expand_dims=lambda x, axis: Node(lambda a: np.expand_dims(a, axis), x),
               reduce_mean=lambda x, axis=None: Node(lambda a: np.mean(a, axis=axis), x),
               reduce_min=lambda x, axis=None: Node(lambda a: np.min(a, axis=axis), x),
               argmin=lambda x, axis=0: Node(lambda a: np.argmin(a, axis=axis), x),
               sqrt=lambda x: Node(np.sqrt, x),
               reshape=lambda x, shape: Node(lambda a: np.reshape(a, shape), x),
               trainable_variables=lambda: [])
    tf.contrib = types.SimpleNamespace(slim=None)
    fw = _stub("tensorflow.contrib.framework.python.framework", checkpoint_utils=None)
    for name in ("tensorflow.contrib", "tensorflow.contrib.framework", "tensorflow.contrib.framework.python"):
        _stub(name)
    del fw
    nnd = _stub("models.tf_ops.nn_distance.tf_nndistance",
                nn_distance=lambda a, b: _multi(lambda x, y: mo.nn_distance(x, y), 4, a, b))
    am = _stub("models.tf_ops.approxmatch.tf_approxmatch",
               approx_match=lambda a, b: Node(mo.approx_match, a, b),
               match_cost=lambda a, b, m: Node(mo.match_cost, a, b, m))
    models = _stub("models")
    ops = _stub("models.tf_ops")
    models.tf_ops = ops
    ops.nn_distance = _stub("models.tf_ops.nn_distance", tf_nndistance=nnd)
    ops.approxmatch = _stub("models.tf_ops.approxmatch", tf_approxmatch=am)

    def load_mesh(path):
        verts, faces = [], []
        with open(path) as fh:
            for line in fh:
                tok = line.split()
                if tok and tok[0] == "v":
                    verts.append([float(x) for x in tok[1:4]])
                elif tok and tok[0] == "f":
                    faces.append([int(t.split("/")[0]) - 1 for t in tok[1:]])
        return types.SimpleNamespace(vertices=np.array(verts, np.float64).reshape(-1, 3),
                                     faces=np.array(faces, np.int64).reshape(-1, 3))

    class VoxelGrid:
        def __init__(self, cell):
            self.dim = int(round(2.0 / cell))

        def insert_mesh(self, mesh):
            self.src = mesh

        def create_grid(self):
            self.mesh = types.SimpleNamespace(vertices=eo.voxel_mesh_vertices(self.src.vertices, self.src.faces, self.dim))

    _stub("pymesh", load_mesh=load_mesh, VoxelGrid=VoxelGrid)

    class Parallel:
        def __init__(self, n_jobs=1):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

        def __call__(self, calls):
            return [f(*a) for f, a in calls]

    _stub("joblib", Parallel=Parallel, delayed=lambda f: (lambda *a: (f, a)))
    np.int = int     # the reference's astype(np.int); the alias was removed from numpy


def import_script(name, argv, raw_dirs):
    _stub("create_file_lst", get_all_info=lambda: (raw_dirs["lst_dir"], None, None, raw_dirs))
    saved = sys.argv
    sys.argv = [name + ".py"] + argv
    try:
        spec = importlib.util.spec_from_file_location(name, os.path.join(REF, "test", name + ".py"))
        mod = importlib.util.module_from_spec(spec)
        with contextlib.redirect_stdout(io.StringIO()):
            spec.loader.exec_module(mod)
    finally:
        sys.argv = saved
    return mod


# ----------------------------------------------------------------------------------------------------------- recording
class Recorder:
    """Wraps np.random.randint and random.sample: every draw, in call order."""

    def __init__(self):
        self.randint, self.sample = [], []

    @contextlib.contextmanager
    def active(self):
        ri, rs = np.random.randint, random.sample

        def randint(*a, **k):
            r = ri(*a, **k)
            self.randint.append(np.asarray(r, np.int64).reshape(-1))
            return r

        def sample(population, k):
            r = rs(population, k)
            self.sample.append(np.array([population.index(x) for x in r], np.int64))
            return r

        np.random.randint, random.sample = randint, sample
        try:
            yield self
        finally:
            np.random.randint, random.sample = ri, rs

    def arrays(self, prefix):
        cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int64)
        return {prefix + "_randint": cat(self.randint), prefix + "_randint_len": np.array([len(x) for x in self.randint]),
                prefix + "_sample": cat(self.sample), prefix + "_sample_len": np.array([len(x) for x in self.sample])}


def result_lines(text, root):
    return [ln.replace(root, "<root>") for ln in text.splitlines() if re.match(LINE_PATTERN, ln.replace(root, "<root>"))]


CD_RE = re.compile(r"avg cf:([^,]+), min_cf:([^,]+), arg_cf view:(\d+), avg emd:([^,]+), min_emd:([^,]+), arg_em view:(\d+)")
CAT_RE = re.compile(r"cat_nm:[^,]+, cat_id:\d+, avg_cf:([^,]+), avg_emd:(.+)$")


def cd_numbers(lines):
    objs = [[float(x) for x in m.groups()] for m in map(CD_RE.search, lines) if m]
    cats = [[float(x) for x in m.groups()] for m in map(CAT_RE.search, lines) if m]
    return np.array(objs, np.float64), np.array(cats, np.float64)


def run(fn, seed, root):
    np.random.seed(seed)
    random.seed(seed)
    rec = Recorder()
    buf = io.StringIO()
    listdir = os.listdir
    os.listdir = lambda d=".": sorted(listdir(d))
    try:
        with rec.active(), contextlib.redirect_stdout(buf):
            fn()
    finally:
        os.listdir = listdir
    return rec, result_lines(buf.getvalue(), root)


def main():
    install_stubs()
    files = fixture_files()
    out = {"files": np.array(sorted(files)), "line_pattern": np.array(LINE_PATTERN),
           "meta": np.array([VIEW_NUM, NPTS, DIM, SEEDS["cd_emd"], SEEDS["save_pnt"], SEEDS["iou"]], np.int64),
           "truethreshold": np.float64(TRUETHRESHOLD), "cats": np.array([[k, v] for k, v in CATS.items()])}
    for i, rel in enumerate(sorted(files)):
        out["file_%d" % i] = np.frombuffer(files[rel], np.uint8)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as td:
        root = os.path.join(td, "fx")
        write_tree(root, files)
        gt, pred, lst = (os.path.join(root, d) for d in ("gt", "pred", "lst"))
        raw_dirs = {"lst_dir": lst, "norm_mesh_dir_v2": gt, "renderedh5_dir_v2": "", "sdf_dir_v2": ""}
        os.chdir(td)
        try:
            common = ["--view_num", str(VIEW_NUM), "--num_sample_points", str(NPTS), "--log_dir", os.path.join(td, "log")]
            cd = import_script("test_cd_emd", common + ["--batch_size", str(VIEW_NUM)], raw_dirs)
            for bs in (VIEW_NUM, 1):
                cd.FLAGS.batch_size = bs
                rec, lines = run(lambda: cd.cd_emd_all(CATS, pred, gt, lst), SEEDS["cd_emd"], root)
                out.update(rec.arrays("cd_emd_bs%d" % bs))
                out["cd_emd_bs%d_lines" % bs] = np.array(lines)
                out["cd_emd_bs%d_obj" % bs], out["cd_emd_bs%d_cat" % bs] = cd_numbers(lines)
                print("cd_emd batch_size", bs, *lines, sep="\n  ")

            def save():
                cd.save_all_cat_gt_pnt(CATS, gt, lst)
                cd.save_all_cat_pred_pnt(CATS, pred, lst)

            rec, lines = run(save, SEEDS["save_pnt"], root)
            out.update(rec.arrays("save_pnt"))
            out["save_pnt_lines"] = np.array(lines)
            pnt = sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs
                         if f.startswith("pnt_"))
            out["pnt_files"] = np.array(pnt)
            out["pnt_values"] = np.stack([np.loadtxt(os.path.join(root, p), dtype=float, delimiter=",").astype(np.float32)
                                          for p in pnt])

            fs = import_script("test_f_score", common + ["--batch_size", str(VIEW_NUM), "--truethreshold",
                                                         str(TRUETHRESHOLD)], raw_dirs)
            for path in ("computed", "cached"):
                thr = [[0.5], [1], [2], [5], [10], [20]]
                _, lines = run(lambda: fs.cal_f_score_all_cat(CATS, pred, gt, lst, thr, fs.FLAGS.truethreshold), 0, root)
                out["f_score_%s_lines" % path] = np.array(lines)
                print("f_score", path, *lines, sep="\n  ")
            for cat_id in CATS.values():
                shutil.rmtree(os.path.join(pred, "pnt_%d_%s" % (NPTS, cat_id)))

            io_ = import_script("test_iou", common + ["--dim", str(DIM)], raw_dirs)
            rec, lines = run(lambda: io_.iou_all(CATS, pred, gt, lst, dim=DIM), SEEDS["iou"], root)
            out.update(rec.arrays("iou"))
            out["iou_lines"] = np.array(lines)
            print("iou", *lines, sep="\n  ")
        finally:
            os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "eval_ref.npz"), **out)


if __name__ == "__main__":
    main()
