"""Ground-truth signed distance grids and their point samples: the GPU counterpart of the reference's
preprocessing/create_point_sdf_grid.py, raw OBJ -> normalised mesh -> field -> isosurface -> samples.

  get_normalize_mesh  <-> get_normalize_mesh (:169-198): surface-sample normalisation on the device (DESIGN.md §4.8);
                          writes pc_norm.obj, returns (obj_file, centroid, m)
  create_one_sdf      <-> create_one_sdf (:200-210): the closed computeDistanceField binary is replaced by the CUDA field
                          of disn_mesh_sdf (DESIGN.md §4.7); `sdfcommand` is accepted for signature compatibility and ignored
  create_one_cube_obj <-> create_one_cube_obj (:248-252): CUDA marching cubes of the .dist, written as an OBJ
  get_sdf             <-> get_sdf (:29-51), on the shared .dist reader
  sample_sdf          <-> sample_sdf (:74-113), host numpy, the reference's np.random call sequence
  check_insideout     <-> check_insideout (:115-137)
  create_h5_sdf_pt    <-> create_h5_sdf_pt (:139-166): band samples on the device; h5py is absent, so the datasets go to
                          an .npz with the reference's names; pc_norm.obj and the .dist are kept
  create_sdf_obj      <-> create_sdf_obj (:213-246): the per-object chain on one resident mesh and one resident field
  create_sdf          <-> create_sdf (:254-317): the batch driver over <lst_dir>/<cat>_{test,train}.lst

CLI: python -m disn_b200.create_point_sdf_grid --obj IN.obj --res 256 --out OUT.dist [--expand 1.2 --g 0.0
     --samples N --sample_out S.npz --seed K]
     python -m disn_b200.create_point_sdf_grid --mesh_dir M --lst_dir L --sdf_dir S --norm_mesh_dir N --cats ID [ID ...]
     [--res 256 --num_sample 32768 --bandwidth 0.1 --iso 0.003 --g 0.0 --version 1 --skip_all_exist --keep_dist --seed K]
"""
from __future__ import annotations

import argparse
import os

import numpy as np

from .create_sdf import read_dist
from .engine import write_dist

TOTAL_SURFACE_SAMPLES = 16384     # get_normalize_mesh's `total` (:170)
INSIDEOUT_CATS = ["02958343", "02691156", "04530566"]


def create_one_sdf(sdfcommand, res, expand_rate, sdf_file, obj_file, indx, g=0.0, engine=None):
    """Signed distance field of the OBJ mesh on a (res+1)^3 grid over the cube around its AABB scaled by expand_rate,
    wall threshold g, written as a .dist (the box goes in the header).  Returns (grid, bbox)."""
    from .engine import Engine
    eng = engine if engine is not None else Engine(device=0, precision="fp32")
    try:
        eng.read_obj(obj_file, load=True)
        grid, bbox = eng.mesh_sdf(int(res), expand_rate=float(expand_rate), sigma=float(g))
    finally:
        if engine is None:
            eng.close()
    write_dist(sdf_file, int(res), bbox, grid)
    return grid, bbox


def get_sdf(sdf_file, sdf_res):
    """{'param': float32 [6] box, 'value': float32 [R,R,R]}; the resolution must equal sdf_res."""
    res, bbox, vals = read_dist(sdf_file)
    if res != sdf_res:
        raise ValueError("%s: res %d not consistent with %d" % (sdf_file, res, sdf_res))
    return {"param": np.float32(bbox), "value": vals}


def sample_sdf(cat_id, num_sample, bandwidth, iso_val, sdf_dict, sdf_res):
    """Samples [n,4] (x, y, z, sdf) in four bands of sdf - iso_val (a quarter of num_sample each, a shortfall carried
    to the next band), drawn with np.random.randint, and check_insideout of the field."""
    percentages = [[-1. * bandwidth, -1. * bandwidth * 0.30, int(num_sample * 0.25)],
                   [-1. * bandwidth * 0.30, 0, int(num_sample * 0.25)],
                   [0, bandwidth * 0.30, int(num_sample * 0.25)],
                   [bandwidth * 0.30, bandwidth, int(num_sample * 0.25)]]
    params = sdf_dict["param"]
    sdf_values = sdf_dict["value"].flatten()
    x = np.linspace(params[0], params[3], num=sdf_res + 1).astype(np.float32)
    y = np.linspace(params[1], params[4], num=sdf_res + 1).astype(np.float32)
    z = np.linspace(params[2], params[5], num=sdf_res + 1).astype(np.float32)
    dis = sdf_values - iso_val
    sdf_pt_val = np.zeros((0, 4), dtype=np.float32)
    for i in range(len(percentages)):
        ind = np.argwhere((dis >= percentages[i][0]) & (dis < percentages[i][1]))
        if len(ind) < percentages[i][2]:
            if i < len(percentages) - 1:
                percentages[i + 1][2] += percentages[i][2] - len(ind)
            percentages[i][2] = len(ind)
        if len(ind) == 0:
            continue
        choice = np.random.randint(len(ind), size=percentages[i][2])
        chosen = ind[choice]
        x_ind = chosen % (sdf_res + 1)
        y_ind = (chosen // (sdf_res + 1)) % (sdf_res + 1)
        z_ind = chosen // (sdf_res + 1) ** 2
        rows = np.concatenate((x[x_ind], y[y_ind], z[z_ind], sdf_values[chosen]), axis=-1)
        sdf_pt_val = np.concatenate((sdf_pt_val, rows), axis=0)
    return sdf_pt_val, check_insideout(cat_id, sdf_values, sdf_res, x, y, z)


def check_insideout(cat_id, sdf_val, sdf_res, x, y, z):
    """For cars, airplanes and watercraft: True when the grid point nearest the origin is outside (sdf > 0), the sign
    of an inside-out field; the reference then regenerates it with a larger g.  False for every other category."""
    if cat_id in ["02958343", "02691156", "04530566"]:
        x_ind = np.argmin(np.absolute(x))
        y_ind = np.argmin(np.absolute(y))
        z_ind = np.argmin(np.absolute(z))
        all_val = sdf_val.flatten()
        num_val = all_val[x_ind + y_ind * (sdf_res + 1) + z_ind * (sdf_res + 1) ** 2]
        return num_val > 0.0
    return False


# ---- per-object chain ----------------------------------------------------------------------------------------------
def _engine(engine):
    from .engine import Engine
    return (engine, False) if engine is not None else (Engine(device=0, precision="fp32"), True)


def surface_draws(amounts):
    """The np.random draws of trimesh.sample.sample_surface for each part in turn: np.random.random(n) for the face
    pick, then np.random.random((n, 2, 1)) for the barycentric lengths -> [sum n, 3] rows (pick, r1, r2)."""
    rows = [np.zeros((0, 3))]
    for n in amounts:
        u = np.random.random(int(n))
        r = np.random.random((int(n), 2, 1))
        rows.append(np.stack([u, r[:, 0, 0], r[:, 1, 0]], axis=1))
    return np.concatenate(rows)


def surface_amounts(part_q, total=TOTAL_SURFACE_SAMPLES):
    """n_p = floor(Q_p * total / sum Q) in exact integers (the reference's int32(area_p * total / area_sum))."""
    qs = sum(int(q) for q in part_q)
    return [int(q) * total // qs if qs else 0 for q in part_q]


def normalize_resident(engine, part_ids=None, n_parts=1, want_samples=False):
    """Surface-sample normalisation of the engine's resident mesh -> (centroid, m[, samples])."""
    q, _ = engine.part_areas(part_ids, n_parts)
    amts = surface_amounts(q)
    return engine.normalize_mesh(part_ids, n_parts, amts, surface_draws(amts), want_samples=want_samples)


def write_obj_exact(path, verts, faces):
    """OBJ whose vertices read back to the same float32 values (%.9g), 1-based faces: the normalised mesh file, so the
    field of pc_norm.obj equals the field of the resident mesh it was written from."""
    v = np.asarray(verts, np.float32).astype(np.float64).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3) + 1
    with open(path, "w") as fh:
        fh.write("# Number of vertices: %d\n# Number of faces: %d\n" % (len(v), len(f)))
        if len(v):
            np.savetxt(fh, v, fmt="v %.9g %.9g %.9g")
        if len(f):
            np.savetxt(fh, f, fmt="f %d %d %d")


def get_normalize_mesh(model_file, norm_mesh_sub_dir, engine=None, mesh=None):
    """get_normalize_mesh (:169-198) on the device: reads the OBJ into the engine (or takes mesh = read_obj_parts' tuple),
    leaves the normalised mesh resident in the engine, writes <norm_mesh_sub_dir>/pc_norm.obj -> (obj_file, centroid, m)."""
    eng, own = _engine(engine)
    try:
        if mesh is None:
            verts, faces, pid, names = eng.read_obj(model_file, parts=True, load=True)
        else:
            verts, faces, pid, names = mesh
            eng.load_mesh(verts, faces)
        centroid, m = normalize_resident(eng, pid, max(len(names), 1))
        obj_file = os.path.join(norm_mesh_sub_dir, "pc_norm.obj")
        write_obj_exact(obj_file, *eng.fetch_mesh())
    finally:
        if own:
            eng.close()
    return obj_file, centroid, m


def create_one_cube_obj(marching_cube_command, i, sdf_file, cube_obj_file, engine=None):
    """create_one_cube_obj (:248-252): the reference runs `<marching_cube_command> <sdf_file> <obj> -i <iso>`; here CUDA
    marching cubes of the .dist at iso i, written in disn_write_obj's format.  The command is ignored."""
    res, bbox, sdf = read_dist(sdf_file)
    eng, own = _engine(engine)
    try:
        eng.marching_cubes(sdf, bbox, float(i), fetch=False)
        eng.write_mesh_obj(cube_obj_file)
    finally:
        if own:
            eng.close()
    return cube_obj_file


def insideout_index(sdf_res, params):
    """Flat index of the grid point check_insideout reads (the point nearest the origin on each axis)."""
    R = sdf_res + 1
    x, y, z = (np.linspace(params[a], params[3 + a], num=R).astype(np.float32) for a in range(3))
    return int(np.argmin(np.absolute(x)) + np.argmin(np.absolute(y)) * R + np.argmin(np.absolute(z)) * R * R)


def write_sample_file(h5_file, flag_file, samples, insideout, centroid, m, sdf_params):
    """The datasets of create_h5_sdf_pt (:145-159) in an .npz (h5py is absent) and the isinsideout.txt flag rule."""
    if insideout:
        with open(flag_file, "w") as f:
            f.write("mid point sdf val > 0")
    elif os.path.exists(flag_file):
        os.remove(flag_file)
    norm_params = np.concatenate((np.asarray(centroid), np.asarray([m]).astype(np.float32)))
    np.savez(h5_file, pc_sdf_original=np.zeros((1, 3), np.float32), pc_sdf_sample=np.asarray(samples, np.float32),
             norm_params=norm_params, sdf_params=np.float32(sdf_params))


def create_h5_sdf_pt(cat_id, h5_file, sdf_file, flag_file, cube_obj_file, norm_obj_file, centroid, m, sdf_res,
                     num_sample, bandwidth, iso_val, max_verts, normalize, engine=None):
    """create_h5_sdf_pt (:139-166) with the band samples drawn on the device (Engine.band_samples, bit for bit the host
    sample_sdf for the same np.random state).  h5_file gets the .npz layout of write_sample_file; unlike the reference
    it leaves norm_obj_file and sdf_file in place."""
    sdf_dict = get_sdf(sdf_file, sdf_res)
    eng, own = _engine(engine)
    try:
        samples = eng.band_samples(num_sample, bandwidth, iso_val, sdf_dict["param"], sdf_res, sdf=sdf_dict["value"])
    finally:
        if own:
            eng.close()
    params = sdf_dict["param"]
    R = sdf_res + 1
    x, y, z = (np.linspace(params[a], params[3 + a], num=R).astype(np.float32) for a in range(3))
    insideout = check_insideout(cat_id, sdf_dict["value"], sdf_res, x, y, z)
    write_sample_file(h5_file, flag_file, samples, insideout, centroid, m, params)
    return samples, insideout


def create_sdf_obj(sdfcommand, marching_cube_command, cat_mesh_dir, cat_norm_mesh_dir, cat_sdf_dir, obj, res, iso_val,
                   expand_rate, indx, ish5, normalize, num_sample, bandwidth, max_verts, cat_id, g, version,
                   skip_all_exist, engine=None, keep_dist=False):
    """create_sdf_obj (:213-246) as one device chain: the raw OBJ is read once, normalised in HBM and written as
    pc_norm.obj; its field goes to the context's resident field buffer, marching cubes at iso_val writes isosurf.obj and
    the band sampler draws ori_sample.npz from the same buffer.  The field leaves HBM only as samples, one value for
    check_insideout and, with keep_dist, isosurf.sdf.  Same skip rule and version 1 / 2 model paths as the reference.
    Returns the .npz path, or None when skipped."""
    obj = obj.rstrip("\r\n")
    sdf_sub_dir = os.path.join(cat_sdf_dir, obj)
    norm_mesh_sub_dir = os.path.join(cat_norm_mesh_dir, obj)
    os.makedirs(sdf_sub_dir, exist_ok=True)
    os.makedirs(norm_mesh_sub_dir, exist_ok=True)
    sdf_file = os.path.join(sdf_sub_dir, "isosurf.sdf")
    flag_file = os.path.join(sdf_sub_dir, "isinsideout.txt")
    cube_obj_file = os.path.join(norm_mesh_sub_dir, "isosurf.obj")
    h5_file = os.path.join(sdf_sub_dir, "ori_sample.npz")
    if ish5 and os.path.exists(h5_file) and (skip_all_exist or not os.path.exists(flag_file)):
        print("skip existed: ", h5_file)
        return None
    if not ish5 and os.path.exists(sdf_file):
        print("skip existed: ", sdf_file)
        return None
    if version == 1:
        model_file = os.path.join(cat_mesh_dir, obj, "model.obj")
    else:
        model_file = os.path.join(cat_mesh_dir, obj, "models", "model_normalized.obj")
    eng, own = _engine(engine)
    try:
        if normalize:
            _, centroid, m = get_normalize_mesh(model_file, norm_mesh_sub_dir, eng)
        else:
            eng.read_obj(model_file, parts=True, load=True)
            centroid, m = np.zeros(3), 1.0
        R = res + 1
        ptr = eng.field_buffer(R)
        _, bbox = eng.mesh_sdf(int(res), expand_rate=float(expand_rate), sigma=float(g), device_ptr=ptr)
        if keep_dist or not ish5:
            write_dist(sdf_file, int(res), bbox, eng.fetch(ptr, (R, R, R)))
        eng.marching_cubes(None, bbox, float(iso_val), device_ptr=ptr, R=R, fetch=False)
        eng.write_mesh_obj(cube_obj_file)
        if not ish5:
            return sdf_file
        params = np.float32(bbox)
        samples = eng.band_samples(num_sample, bandwidth, iso_val, params, int(res), device_ptr=ptr)
        insideout = False
        if cat_id in INSIDEOUT_CATS:
            insideout = bool(eng.fetch(ptr + 4 * insideout_index(int(res), params), (1,))[0] > 0.0)
        write_sample_file(h5_file, flag_file, samples, insideout, centroid, m, params)
    finally:
        if own:
            eng.close()
    return h5_file


def create_sdf(sdfcommand, marching_cube_command, LIB_command, num_sample, bandwidth, res, expand_rate, cats, raw_dirs,
               lst_dir, iso_val, max_verts, ish5=True, normalize=True, g=0.00, version=2, skip_all_exist=False,
               engine=None, keep_dist=False):
    """create_sdf (:254-317): every object of <lst_dir>/<cat_id>_test.lst then _train.lst of each category in `cats`
    (name -> id) through create_sdf_obj, under raw_dirs['sdf_dir'|'mesh_dir'|'norm_mesh_dir']/<cat_id>/<obj>.  One
    engine serves every object in turn (the reference's joblib pool ran the closed binaries in parallel processes).
    The commands are ignored.  Returns the paths written."""
    os.makedirs(raw_dirs["sdf_dir"], exist_ok=True)
    eng, own = _engine(engine)
    done = []
    try:
        indx = 0
        for catnm in cats.keys():
            cat_id = cats[catnm]
            cat_sdf_dir = os.path.join(raw_dirs["sdf_dir"], cat_id)
            os.makedirs(cat_sdf_dir, exist_ok=True)
            cat_mesh_dir = os.path.join(raw_dirs["mesh_dir"], cat_id)
            cat_norm_mesh_dir = os.path.join(raw_dirs["norm_mesh_dir"], cat_id)
            list_obj = []
            for split in ("test", "train"):
                with open(os.path.join(lst_dir, str(cat_id) + "_" + split + ".lst")) as f:
                    list_obj += f.readlines()
            for obj in list_obj:
                if not obj.strip():
                    continue
                out = create_sdf_obj(sdfcommand, marching_cube_command, cat_mesh_dir, cat_norm_mesh_dir, cat_sdf_dir, obj,
                                     res, iso_val, expand_rate, indx, ish5, normalize, num_sample, bandwidth, max_verts,
                                     cat_id, g, version, skip_all_exist, engine=eng, keep_dist=keep_dist)
                indx += 1
                if out:
                    done.append(out)
    finally:
        if own:
            eng.close()
    return done


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--obj", help="single-mesh mode: OBJ input (with --out)")
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--out", help="single-mesh mode: .dist output")
    ap.add_argument("--expand", type=float, default=1.2)
    ap.add_argument("--g", type=float, default=0.0, help="wall threshold sigma (closes gaps narrower than about 2g)")
    ap.add_argument("--samples", type=int, default=0, help="points to sample with sample_sdf (0: none)")
    ap.add_argument("--bandwidth", type=float, default=0.1)
    ap.add_argument("--iso", type=float, default=None, help="iso value (default 0.0; batch mode 0.003)")
    ap.add_argument("--cat_id", default="")
    ap.add_argument("--sample_out", default=None)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--mesh_dir", help="batch mode: <mesh_dir>/<cat>/<obj>/model.obj (version 1) or "
                                       "models/model_normalized.obj (version 2)")
    ap.add_argument("--lst_dir", help="batch mode: <lst_dir>/<cat>_test.lst and <cat>_train.lst")
    ap.add_argument("--sdf_dir", help="batch mode: output <sdf_dir>/<cat>/<obj>/ori_sample.npz")
    ap.add_argument("--norm_mesh_dir", help="batch mode: output <norm_mesh_dir>/<cat>/<obj>/{pc_norm,isosurf}.obj")
    ap.add_argument("--cats", nargs="+", default=[], help="batch mode: category ids")
    ap.add_argument("--num_sample", type=int, default=32768)
    ap.add_argument("--version", type=int, default=1, choices=(1, 2))
    ap.add_argument("--skip_all_exist", action="store_true")
    ap.add_argument("--keep_dist", action="store_true", help="batch mode: also write isosurf.sdf")
    a = ap.parse_args(argv)
    if a.mesh_dir is not None:
        if not (a.lst_dir and a.sdf_dir and a.norm_mesh_dir and a.cats):
            ap.error("batch mode needs --mesh_dir, --lst_dir, --sdf_dir, --norm_mesh_dir and --cats")
        np.random.seed(a.seed)
        raw_dirs = {"mesh_dir": a.mesh_dir, "sdf_dir": a.sdf_dir, "norm_mesh_dir": a.norm_mesh_dir}
        done = create_sdf(None, None, None, a.num_sample, a.bandwidth, a.res, a.expand, {c: c for c in a.cats}, raw_dirs,
                          a.lst_dir, 0.003 if a.iso is None else a.iso, 16384, g=a.g, version=a.version,
                          skip_all_exist=a.skip_all_exist, keep_dist=a.keep_dist)
        print("%d objects written" % len(done))
        return
    if not (a.obj and a.out):
        ap.error("the following arguments are required: --obj, --out (or the batch-mode flags)")
    a.iso = 0.0 if a.iso is None else a.iso
    grid, bbox = create_one_sdf(None, a.res, a.expand, a.out, a.obj, 0, a.g)
    print("%s: %d^3 points, box %s, %d negative" % (a.out, a.res + 1, np.round(bbox, 6).tolist(), int((grid < 0).sum())))
    if a.samples:
        np.random.seed(a.seed)
        pts, insideout = sample_sdf(a.cat_id, a.samples, a.bandwidth, a.iso, get_sdf(a.out, a.res), a.res)
        out = a.sample_out or (a.out[:-5] if a.out.endswith(".dist") else a.out) + "_samples.npz"
        np.savez(out, sdf_pt_val=pts, insideout=insideout)
        print("%s: %d samples, check_insideout=%s" % (out, len(pts), bool(insideout)))


if __name__ == "__main__":
    main()
