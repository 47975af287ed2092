"""The strided full-grid samples of the reference's preprocessing/create_point_sdf_fullgrid.py on the device.

  sample_sdf          <-> sample_sdf (:70-96): every `reduce`-th field value on each axis (disn_sdf_strided), with the
                          grid point nearest the origin read for check_insideout
  get_param_from_h5   <-> get_param_from_h5 (:152-161), on the .npz that create_point_sdf_grid writes
  get_normalize_mesh  <-> get_normalize_mesh (:163-183): the largest part by area (ties: the lowest part, the reference's
                          strict <) transformed with the grid run's norm_params (disn_mesh_normalize with given (c, m))
"""
from __future__ import annotations

import os

import numpy as np

from .create_point_sdf_grid import _engine, check_insideout, write_obj_exact
from .create_sdf import read_obj_parts


def sample_sdf(cat_id, num_sample, bandwidth, iso_val, sdf_dict, sdf_res, reduce, engine=None, device_ptr=None):
    """-> (values [M^3, 1] float32 in (z, y, x) order, M = sdf_res // reduce + 1, check_insideout of the full field).
    sdf_dict: get_sdf's {'param', 'value'}; with device_ptr the field is read from HBM instead of sdf_dict['value']."""
    params = sdf_dict["param"]
    R = sdf_res + 1
    eng, own = _engine(engine)
    try:
        vals = eng.sdf_strided(R, int(reduce), sdf=None if device_ptr is not None else sdf_dict["value"],
                               device_ptr=device_ptr)
    finally:
        if own:
            eng.close()
    x, y, z = (np.linspace(params[a], params[3 + a], num=R).astype(np.float32) for a in range(3))
    return vals.reshape(-1, 1), check_insideout(cat_id, sdf_dict["value"], sdf_res, x, y, z)


def get_param_from_h5(sdf_h5_file, cat_id, obj):
    """(centroid [3], m) from the norm_params of an ori_sample.npz."""
    with np.load(sdf_h5_file) as z:
        if "norm_params" not in z.files:
            raise Exception(cat_id, obj, "no sdf and sample")
        norm_params = z["norm_params"]
    return norm_params[:3], norm_params[3]


def largest_part(engine, part_ids, n_parts):
    """Index of the part with the largest quantised area; ties go to the lowest index."""
    q, _ = engine.part_areas(part_ids, n_parts)
    best, best_q = 0, 0
    for p, v in enumerate(q):
        if best_q < int(v):
            best, best_q = p, int(v)
    return best


def get_normalize_mesh(model_file, norm_sdf_file, cat_id, obj, sdf_sub_dir, engine=None):
    """The largest part of the raw OBJ, transformed with the (c, m) of norm_sdf_file and written as
    <sdf_sub_dir>/pc_norm.obj -> (obj_file, centroid, m).  The part's vertices are the ones its faces reference, in their
    original order."""
    verts, faces, pid, names = read_obj_parts(model_file)
    centroid, m = get_param_from_h5(norm_sdf_file, cat_id, obj)
    eng, own = _engine(engine)
    try:
        eng.load_mesh(verts, faces)
        keep = pid == largest_part(eng, pid, max(len(names), 1))
        used = np.zeros(len(verts), bool)
        used[faces[keep].reshape(-1)] = True
        remap = np.cumsum(used) - 1
        eng.load_mesh(verts[used], remap[faces[keep]].astype(np.int32))
        eng.normalize_mesh(given=[centroid[0], centroid[1], centroid[2], float(m)])
        obj_file = os.path.join(sdf_sub_dir, "pc_norm.obj")
        write_obj_exact(obj_file, *eng.fetch_mesh())
    finally:
        if own:
            eng.close()
    return obj_file, centroid, m
