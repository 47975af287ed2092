"""Drop-in mirror of the reference's inference driver ``test/create_sdf.py`` (and ``demo/demo.py``) for the
SDF hot path: same module-level constants, same function names and argument meaning
(``create``, ``test_one_epoch``, ``to_binary``, ``create_obj``, ``create_one_cube_obj``), running on the
DISN library.  ``create`` takes an iterable of ``batch_data`` dicts in the loader's layout
(data/data_sdf_h5_queue.py:291-303); ``python -m disn_b200.create_sdf`` feeds it from the test-set loader
(disn_b200/data_sdf_h5_queue.py) over the view files of create_img_h5, as the reference script does.

    import disn_b200.create_sdf as cs
    cs.configure(FLAGS)                       # the reference does this at import time from argparse
    cs.create(weights, batches)               # -> one .obj per (object, view) under RESULT_OBJ_PATH
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from concurrent.futures import ThreadPoolExecutor
from datetime import datetime
from types import SimpleNamespace

import numpy as np

from . import _lib
from . import model_normalization as model
from .engine import write_dist

# module state, same names as test/create_sdf.py:66-98
FLAGS = None
BATCH_SIZE = RESOLUTION = TOTAL_POINTS = SPLIT_SIZE = NUM_SAMPLE_POINTS = NUM_POINTS = None
SDF_WEIGHT = 10.0
LOG_DIR = RESULT_OBJ_PATH = None
IMG_SIZE = 137
LOG_FOUT = None
_ENGINE = None          # engine used by create_one_cube_obj for the marching-cubes post-pass
_ENGINE_LOCK = threading.Lock()   # a context is not thread-safe; create_obj runs on a 4-worker pool


def default_flags(**kw):
    """argparse defaults of test/create_sdf.py:26-63 / demo/demo.py:27-65."""
    d = dict(gpu="0", img_h=137, img_w=137, batch_size=1, num_classes=1024, num_points=1, sdf_res=64, alpha=False,
             rot=False, tanh=False, multi_view=False, num_sample_points=1, log_dir="checkpoint/SDF_DISN",
             iso=0.0, threedcnn=False, img_feat_onestream=False, img_feat_twostream=True, binary=False,
             cam_est=False, view_num=24, category="all", precision="f16f8")
    d.update(kw)
    return SimpleNamespace(**d)


def configure(flags):
    """Derive the module constants exactly as test/create_sdf.py:66-98 does."""
    global FLAGS, BATCH_SIZE, RESOLUTION, TOTAL_POINTS, SPLIT_SIZE, NUM_SAMPLE_POINTS, NUM_POINTS
    global LOG_DIR, RESULT_OBJ_PATH, IMG_SIZE, LOG_FOUT
    FLAGS = flags
    NUM_POINTS = FLAGS.num_points
    BATCH_SIZE = FLAGS.batch_size
    RESOLUTION = FLAGS.sdf_res + 1
    TOTAL_POINTS = RESOLUTION * RESOLUTION * RESOLUTION
    if FLAGS.img_feat_twostream:
        SPLIT_SIZE = int(np.ceil(TOTAL_POINTS / 214669.0))
    elif FLAGS.threedcnn:
        SPLIT_SIZE = 1
    else:
        SPLIT_SIZE = int(np.ceil(TOTAL_POINTS / 274625.0))
    NUM_SAMPLE_POINTS = int(np.ceil(TOTAL_POINTS / SPLIT_SIZE))
    LOG_DIR = FLAGS.log_dir
    os.makedirs(LOG_DIR, exist_ok=True)
    tag = ("camest_" if FLAGS.cam_est else "") + str(RESOLUTION) + "_" + str(FLAGS.iso)
    RESULT_OBJ_PATH = os.path.join(LOG_DIR, "test_objs", tag)
    os.makedirs(RESULT_OBJ_PATH, exist_ok=True)
    IMG_SIZE = FLAGS.img_h
    LOG_FOUT = open(os.path.join(LOG_DIR, "log_test.txt"), "w")
    LOG_FOUT.write(str(FLAGS) + "\n")


def log_string(out_str):
    LOG_FOUT.write(out_str + "\n")
    LOG_FOUT.flush()
    print(out_str)


def create(weights, batches, device=0):
    """test/create_sdf.py:152-208.  ``weights``: TF-variable-name -> array, or None to mirror the reference's
    behaviour when no checkpoint restores (it then runs on its random initialisation; here that must be
    supplied explicitly -- the encoder refuses to run on absent weights).  ``batches``: iterable of
    batch_data dicts (img [B,137,137,3], trans_mat [B,4,3], sdf_params [B,6], cat_id, obj_nm, view_id)."""
    global _ENGINE
    log_string(LOG_DIR)
    input_pls = model.placeholder_inputs(BATCH_SIZE, NUM_POINTS, (IMG_SIZE, IMG_SIZE),
                                         num_sample_pc=NUM_SAMPLE_POINTS, scope="inputs_pl", FLAGS=FLAGS)
    is_training_pl = model.Placeholder("is_training", ())
    end_points = model.get_model(input_pls, NUM_POINTS, is_training_pl, bn=False, FLAGS=FLAGS)
    loss, end_points = model.get_loss(end_points, sdf_weight=SDF_WEIGHT, num_sample_points=NUM_SAMPLE_POINTS, FLAGS=FLAGS)
    sess = model.Session(device=device, precision=getattr(FLAGS, "precision", "f16f8"), max_batch=max(1, BATCH_SIZE))
    if weights is None:
        print("Fail to load overall modelfile: %s" % LOG_DIR)       # create_sdf.py:192
        raise RuntimeError("no weights supplied: pass the checkpoint variables (or a random init) explicitly")
    sess.load_weights(weights)
    print("Model loaded in file: %s" % LOG_DIR)
    _ENGINE = sess.engine
    ops = {"input_pls": input_pls, "is_training_pl": is_training_pl, "loss": loss, "step": 0,
           "end_points": end_points}
    try:
        return test_one_epoch(sess, ops, batches)
    finally:
        _ENGINE = None
        sess.close()


# FLAGS.adaptive without keep_dist meshes through Engine.mesh_grid_adaptive from this sdf_res on: the first resolution the
# dense adaptive grid plus marching cubes cannot run (marching cubes needs 3 (sdf_res+1)^3 < 2^32, so sdf_res <= 1126).
# Wherever that path runs it is faster (H100 80GB HBM3, 700 W, tools/adaptive_mesh_bench.py, BASELINE.md §8: 2.4 s
# against 8.3 s at 1025^3 on the median iso, 0.48 s against 2.9 s on the 0.95 quantile).
SURFACE_MESH_MIN_RES = 1127


def build_grid_points(sdf_params_b):
    """test/create_sdf.py:246-255 -- host float64 linspace grid, (x,y,z) float32, x fastest."""
    x_ = np.linspace(sdf_params_b[0], sdf_params_b[3], num=RESOLUTION)
    y_ = np.linspace(sdf_params_b[1], sdf_params_b[4], num=RESOLUTION)
    z_ = np.linspace(sdf_params_b[2], sdf_params_b[5], num=RESOLUTION)
    z, y, x = np.meshgrid(z_, y_, x_, indexing="ij")
    return np.stack([x, y, z], axis=3).astype(np.float32).reshape(1, -1, 3)


def obj_path(dir, cat_id, obj_nm, view_id):
    """file naming of create_obj (test/create_sdf.py:305-312)"""
    if not isinstance(view_id, str):
        view_id = "%02d" % view_id
    dir = os.path.join(dir, cat_id)
    os.makedirs(dir, exist_ok=True)
    return os.path.join(dir, cat_id + "_" + obj_nm + "_" + view_id + ".obj")


def test_one_epoch(sess, ops, batches):
    """test/create_sdf.py:224-289 on the device: per batch one encode + one dense-grid evaluation that STAYS in HBM
    (disn_eval_grid_resident), then per image the CUDA marching-cubes post-pass straight on that buffer and the OBJ writer
    (formatted on a worker thread, like the reference's 4-worker pool for its mesher, create_sdf.py:238,288).
    No .dist round trip through the file system; FLAGS.keep_dist=True also writes the reference's .dist artefact.
    FLAGS.clean_smallparts=True runs the reference's postprocessing/clean_smallparts.py step on each mesh while it is
    still in HBM (thresholds FLAGS.clean_dist_thresh / clean_num_thresh, default 0.5 / 0.3).
    FLAGS.adaptive=True (default False) replaces the batch's dense grid with coarse-to-fine evaluation per image (band
    FLAGS.adaptive_band, default 1.0): the network runs only near the surface.  From sdf_res SURFACE_MESH_MIN_RES on and
    without keep_dist no grid is built: Engine.mesh_grid_adaptive meshes from the surface blocks alone (DESIGN.md §4.10,
    the same mesh bit for bit); otherwise Engine.eval_grid_adaptive builds the grid.  Output names, cleaning and the OBJ
    writer are unchanged.
    The reference's literal loop (host grid, SPLIT_SIZE chunks through sess.run, reassembly, /SDF_WEIGHT) is kept as a
    verification aid in tests/reference_loop.py."""
    log_string(str(datetime.now()))
    written = []
    R = RESOLUTION
    with ThreadPoolExecutor(max_workers=4) as executor:
        futures = []
        for batch_idx, batch_data in enumerate(batches):
            with _ENGINE_LOCK:
                sess.engine.encode(batch_data["img"])
                sess._img_key = None
                adaptive = getattr(FLAGS, "adaptive", False)
                if not adaptive:
                    grid_ptr = sess.engine.eval_grid_resident(batch_data["sdf_params"], batch_data["trans_mat"], FLAGS.sdf_res)
                for b in range(BATCH_SIZE):
                    print("{}/{}, submit create_obj {}, {}, {}".format(batch_idx, "?", batch_data["cat_id"][b],
                                                                       batch_data["obj_nm"][b], batch_data["view_id"][b]))
                    path = obj_path(RESULT_OBJ_PATH, batch_data["cat_id"][b], batch_data["obj_nm"][b], batch_data["view_id"][b])
                    keep_dist = getattr(FLAGS, "keep_dist", False)
                    band = float(getattr(FLAGS, "adaptive_band", 1.0))
                    if adaptive and not keep_dist and FLAGS.sdf_res >= SURFACE_MESH_MIN_RES:
                        # no grid needed: mesh from the surface blocks (DESIGN.md §4.10)
                        sess.engine.mesh_grid_adaptive(
                            np.asarray(batch_data["sdf_params"], np.float64)[b], np.asarray(batch_data["trans_mat"])[b],
                            FLAGS.sdf_res, iso=float(FLAGS.iso), band=band, image=b, fetch=False)
                        dev = None
                    elif adaptive:      # coarse-to-fine grid of this image (DESIGN.md §4.9), meshed before the next one
                        dev, _ = sess.engine.eval_grid_adaptive(
                            np.asarray(batch_data["sdf_params"], np.float64)[b], np.asarray(batch_data["trans_mat"])[b],
                            FLAGS.sdf_res, iso=float(FLAGS.iso), band=band, image=b)
                    else:
                        dev = grid_ptr + b * R * R * R * 4
                    if dev is None:
                        if getattr(FLAGS, "clean_smallparts", False):
                            verts, faces = sess.engine.clean_mesh(getattr(FLAGS, "clean_dist_thresh", 0.5),
                                                                  getattr(FLAGS, "clean_num_thresh", 0.3))
                        else:
                            verts, faces = sess.engine.fetch_mesh()
                    elif getattr(FLAGS, "clean_smallparts", False):
                        # postprocessing/clean_smallparts.py on the resident mesh before it leaves HBM
                        sess.engine.marching_cubes(None, batch_data["sdf_params"][b], float(FLAGS.iso), device_ptr=dev,
                                                   R=R, fetch=False)
                        verts, faces = sess.engine.clean_mesh(getattr(FLAGS, "clean_dist_thresh", 0.5),
                                                              getattr(FLAGS, "clean_num_thresh", 0.3))
                    else:
                        verts, faces = sess.engine.marching_cubes(None, batch_data["sdf_params"][b], float(FLAGS.iso),
                                                                  device_ptr=dev, R=R)
                    if keep_dist:
                        to_binary(R - 1, batch_data["sdf_params"][b], sess.engine.fetch(dev, (R, R, R)), path[:-4] + ".dist")
                    futures.append(executor.submit(_write_and_return, path, verts, faces))
        for f in futures:
            written.append(f.result())
    return written


def _write_and_return(path, verts, faces):
    write_obj(path, verts, faces)
    return path


def to_binary(res, pos, pred_sdf_val_all, sdf_file):
    """test/create_sdf.py:292-303 -- .dist: int32 -res,res,res; 6 float64; (res+1)^3 float32.  Written by the
    C-ABI writer (the reference struct.packs R^3 Python floats)."""
    write_dist(sdf_file, res, pos, np.asarray(pred_sdf_val_all, dtype=np.float32).reshape(-1))


def create_obj(pred_sdf_val, sdf_params, dir, cat_id, obj_nm, view_id, i):
    """test/create_sdf.py:305-317."""
    cube_obj_file = obj_path(dir, cat_id, obj_nm, view_id)
    sdf_file = cube_obj_file[:-4] + ".dist"
    to_binary((RESOLUTION - 1), sdf_params, pred_sdf_val, sdf_file)
    create_one_cube_obj("./isosurface/computeMarchingCubes", i, sdf_file, cube_obj_file)
    if os.path.exists(sdf_file):
        os.remove(sdf_file)                   # the reference shells out to `rm -rf`
    return cube_obj_file


def read_dist(sdf_file):
    """Parse a .dist (layout pinned by preprocessing/create_point_sdf_grid.py:29-51)."""
    with open(sdf_file, "rb") as f:
        hdr = np.frombuffer(f.read(12), dtype=np.int32)
        if not (hdr[0] < 0 and hdr[1] == -hdr[0] and hdr[2] == -hdr[0]):
            raise ValueError("%s: not a float32 cubic .dist file" % sdf_file)
        res = int(-hdr[0])
        bbox = np.frombuffer(f.read(48), dtype=np.float64)
        vals = np.frombuffer(f.read(), dtype=np.float32)
    R = res + 1
    if vals.size != R ** 3:
        raise ValueError("%s: expected %d samples, found %d" % (sdf_file, R ** 3, vals.size))
    return res, bbox, vals.reshape(R, R, R)


def write_obj(path, verts, faces):
    """OBJ with the reference output's conventions (demo/result.obj: `v %g %g %g`, 1-based `f`), via the C ABI."""
    v = np.ascontiguousarray(verts, np.float32)
    f = np.ascontiguousarray(faces, np.int32)
    _lib.check(_lib.load().disn_write_obj(path.encode(), v.ctypes.data_as(C.c_void_p), len(v),
                                          f.ctypes.data_as(C.c_void_p), len(f)))


def read_obj(path):
    """Triangle mesh of an OBJ file: `v x y z` records and `f` records of `i`, `i/j` or `i/j/k` tokens (1-based) ->
    (verts [V,3] float32, faces [F,3] int32 0-based).  Other record types are ignored; a face that is not a triangle
    raises ValueError."""
    verts, faces = [], []
    with open(path) as fh:
        for n, line in enumerate(fh, 1):
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                verts.append([float(x) for x in tok[1:4]])
            elif tok[0] == "f":
                if len(tok) != 4:
                    raise ValueError("%s:%d: only triangle faces are supported, found %d corners" % (path, n, len(tok) - 1))
                faces.append([int(t.split("/")[0]) - 1 for t in tok[1:]])
    return (np.array(verts, np.float64).astype(np.float32).reshape(-1, 3),
            np.array(faces, np.int64).astype(np.int32).reshape(-1, 3))


def read_obj_parts(path):
    """read_obj plus the parts trimesh.load_mesh(process=False) splits an OBJ into (restated, unpinned: one part per
    `usemtl` material name, in order of first appearance; faces before the first `usemtl`, or every face of a file
    without one, form their own part) -> (verts [V,3] float32, faces [F,3] int32 0-based, part_ids [F] int32,
    names: one material name, or None, per part).  The vertex array is shared by all parts."""
    verts, faces, pids, names, index = [], [], [], [], {}
    cur = None
    with open(path) as fh:
        for n, line in enumerate(fh, 1):
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                verts.append([float(x) for x in tok[1:4]])
            elif tok[0] == "usemtl":
                cur = tok[1] if len(tok) > 1 else ""
            elif tok[0] == "f":
                if len(tok) != 4:
                    raise ValueError("%s:%d: only triangle faces are supported, found %d corners" % (path, n, len(tok) - 1))
                if cur not in index:
                    index[cur] = len(names)
                    names.append(cur)
                faces.append([int(t.split("/")[0]) - 1 for t in tok[1:]])
                pids.append(index[cur])
    return (np.array(verts, np.float64).astype(np.float32).reshape(-1, 3),
            np.array(faces, np.int64).astype(np.int32).reshape(-1, 3), np.array(pids, np.int32), names)


def create_one_cube_obj(marching_cube_command, i, sdf_file, cube_obj_file):
    """test/create_sdf.py:319-323.  The reference runs `<marching_cube_command> <dist> <obj> -i <iso>` (a
    closed-source CPU binary); here the .dist is meshed by the CUDA marching-cubes post-pass.
    ``marching_cube_command`` is accepted for signature compatibility and ignored."""
    from .engine import Engine
    res, bbox, sdf = read_dist(sdf_file)
    eng = _ENGINE
    own = eng is None
    if own:
        eng = Engine(device=0, precision="fp32")
    try:
        with _ENGINE_LOCK:
            verts, faces = eng.marching_cubes(sdf, bbox, float(i))
    finally:
        if own:
            eng.close()
    write_obj(cube_obj_file, verts, faces)
    return cube_obj_file


def main(argv=None, weights=None):
    """`python -m disn_b200.create_sdf`: test/create_sdf.py as a script -- the test lists (test/create_sdf.py:106-149:
    random.sample(range(24), view_num) views per object), the test-set loader without shuffling, and create().  weights
    (TF variable name -> array) replaces the checkpoint of --log_dir."""
    import argparse
    import random
    from . import data_sdf_h5_queue
    from .test_sdf_acc import CATS, build_listinfo, checkpoint_prefix
    ap = argparse.ArgumentParser()
    d = default_flags()
    for k in ("gpu", "log_dir", "category", "precision"):
        ap.add_argument("--" + k, default=d.__dict__[k])
    for k in ("max_epoch", "img_h", "img_w", "batch_size", "num_classes", "num_points", "sdf_res", "cat_limit",
              "num_sample_points", "view_num"):
        ap.add_argument("--" + k, type=int, default=dict(max_epoch=1, cat_limit=168000).get(k, d.__dict__.get(k)))
    ap.add_argument("--iso", type=float, default=0.0)
    for k in ("alpha", "rot", "tanh", "multi_view", "threedcnn", "img_feat_onestream", "binary", "create_obj", "store",
              "cam_est", "augcolorfore", "augcolorback", "backcolorwhite", "adaptive", "clean_smallparts", "keep_dist"):
        ap.add_argument("--" + k, action="store_true")
    ap.add_argument("--img_feat_twostream", action="store_true", default=True)
    ap.add_argument("--test_lst_dir", required=True, help="<cat_id>_test.lst")
    ap.add_argument("--view_dir", required=True, help="view files of create_img_h5: <view_dir>/<cat>/<obj>/%%02d.npz")
    ap.add_argument("--sdf_dir", required=True, help="<sdf_dir>/<cat>/<obj>/ori_sample.npz")
    flags = ap.parse_args(argv)
    print(flags)
    data_sdf_h5_queue.check_flags(flags)
    listinfo, cats_limit = build_listinfo(flags, CATS, view_lists=lambda: random.sample(range(24), flags.view_num))
    dataset = data_sdf_h5_queue.Pt_sdf_img(flags, listinfo=listinfo, cats_limit=cats_limit, shuffle=False,
                                           info={"rendered_dir": flags.view_dir, "sdf_dir": flags.sdf_dir})
    configure(flags)
    if weights is None:
        from .tf_checkpoint import load_checkpoint
        prefix = checkpoint_prefix(flags.log_dir)
        weights = None if prefix is None else load_checkpoint(prefix, prefixes=("vgg_16/", "sdfprediction"))
    num_batches = int(len(dataset) / BATCH_SIZE)
    dataset.start()
    try:
        return create(weights, (dataset.fetch() for _ in range(num_batches)))
    finally:
        dataset.shutdown()
        LOG_FOUT.close()


if __name__ == "__main__":
    main()
