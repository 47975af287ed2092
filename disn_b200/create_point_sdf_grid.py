"""Ground-truth signed distance grids and their point samples: the GPU counterpart of the reference's
preprocessing/create_point_sdf_grid.py on the path mesh -> .dist -> samples.

  create_one_sdf   <-> create_one_sdf (:200-210): the closed computeDistanceField binary is replaced by the CUDA field
                       of disn_mesh_sdf (DESIGN.md §4.7); `sdfcommand` is accepted for signature compatibility and ignored
  get_sdf          <-> get_sdf (:29-51), on the shared .dist reader
  sample_sdf       <-> sample_sdf (:74-113), host numpy, the reference's np.random call sequence
  check_insideout  <-> check_insideout (:115-137)

CLI: python -m disn_b200.create_point_sdf_grid --obj IN.obj --res 256 --out OUT.dist [--expand 1.2 --g 0.0
     --samples N --sample_out S.npz --seed K]
"""
from __future__ import annotations

import argparse

import numpy as np

from .create_sdf import read_dist, read_obj
from .engine import write_dist


def create_one_sdf(sdfcommand, res, expand_rate, sdf_file, obj_file, indx, g=0.0, engine=None):
    """Signed distance field of the OBJ mesh on a (res+1)^3 grid over the cube around its AABB scaled by expand_rate,
    wall threshold g, written as a .dist (the box goes in the header).  Returns (grid, bbox)."""
    from .engine import Engine
    verts, faces = read_obj(obj_file)
    eng = engine if engine is not None else Engine(device=0, precision="fp32")
    try:
        grid, bbox = eng.mesh_sdf(int(res), expand_rate=float(expand_rate), sigma=float(g), verts=verts, faces=faces)
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


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--obj", required=True)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--out", required=True, help=".dist output")
    ap.add_argument("--expand", type=float, default=1.2)
    ap.add_argument("--g", type=float, default=0.0, help="wall threshold sigma (closes gaps narrower than about 2g)")
    ap.add_argument("--samples", type=int, default=0, help="points to sample with sample_sdf (0: none)")
    ap.add_argument("--bandwidth", type=float, default=0.1)
    ap.add_argument("--iso", type=float, default=0.0)
    ap.add_argument("--cat_id", default="")
    ap.add_argument("--sample_out", default=None)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
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
