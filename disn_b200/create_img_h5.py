"""Per-view camera files, the reference's ``preprocessing/create_img_h5.py`` (gen_obj_img_h5 / convert_img2h5, :14-201).

For every object of ``<lst_dir>/<cat>_train.lst`` and ``_test.lst``, each rendering listed in
``<source_dir>/<cat>/<obj>/rendering/renderings.txt`` becomes ``<view_dir>/<cat>/<obj>/%02d.npz`` with the reference's
dataset names: ``img_arr`` (the PNG as cv2.IMREAD_UNCHANGED reads it, uint8), ``trans_mat`` = (K·RT·rot·norm)ᵀ [4,3],
``K``, ``RT``, ``obj_rot_mat`` and ``regress_mat`` = (RT·rot·norm)ᵀ, all float32.  norm comes from the object's
``<sdf_dir>/<cat>/<obj>/ori_sample.npz`` (create_point_sdf_grid); h5py is absent, so the files are .npz, as that one is.
The camera arithmetic is synth's (getBlenderProj, get_rotate_matrix, get_norm_matrix), fed the float32 values of
rendering_metadata.txt as the reference feeds them.  A file that exists and holds a trans_mat is skipped.

    python -m disn_b200.create_img_h5 --source_dir ShapeNetRendering --view_dir V --sdf_dir S --lst_dir L --cats ID [ID ...]
"""
from __future__ import annotations

import argparse
import os

import numpy as np

from . import synth

rot90y = np.array([[0, 0, -1],
                   [0, 1, 0],
                   [1, 0, 0]], dtype=np.float32)


def getBlenderProj(az, el, distance_ratio, img_w=137, img_h=137):
    """:14-63 -> (K [3,3], RT [3,4]) float64."""
    if (img_w, img_h) != (synth.IMG_W, synth.IMG_H):
        raise ValueError("the renderings are 137x137")
    return synth.intrinsics(), synth.blender_extrinsics(az, el, distance_ratio)


def get_rotate_matrix(rotation_angle1):
    """:65-103 (called with -pi/2)."""
    return synth.axis_rotation_matrix(rotation_angle1)


def get_norm_matrix(sdf_file):
    """:106-123: T(centre)·S(m) from the norm_params of ori_sample.npz."""
    norm_params = np.load(sdf_file)["norm_params"]
    return synth.norm_matrix(norm_params[:3], norm_params[3])


def _axis_mats(param):
    """get_az / get_el / get_inl (:222-249) of degree2rad(param) (:203-208), float32 as in the reference."""
    az, el, inl = (np.float32(np.deg2rad(param[0] + np.float32(180.0))), np.float32(np.deg2rad(param[1])),
                   np.float32(np.deg2rad(param[2])))
    mat = lambda v: np.asarray(v, dtype=np.float32).reshape(3, 3)
    return (mat([np.cos(az), 0.0, np.sin(az), 0.0, 1.0, 0.0, -1.0 * np.sin(az), 0.0, np.cos(az)]),
            mat([1.0, 0.0, 0.0, 0.0, np.cos(el), -1.0 * np.sin(el), 0.0, np.sin(el), np.cos(el)]),
            mat([np.cos(inl), -1.0 * np.sin(inl), 0.0, np.sin(inl), np.cos(inl), 0.0, 0.0, 0.0, 1.0]))


def get_img_cam(param):
    """:199-201 / :210-220 camera_info: the camera rotation (inl·el·az)ᵀ, float32 (the position is unused)."""
    az_mat, el_mat, inl_mat = _axis_mats(param)
    return np.transpose(np.matmul(np.matmul(inl_mat, el_mat), az_mat))


def view_datasets(img_file, param, norm_mat, rot_mat):
    """The six datasets of one view file (:170-195)."""
    import cv2
    obj_rot_mat = np.dot(rot90y, get_img_cam(param))
    img = cv2.imread(img_file, cv2.IMREAD_UNCHANGED)
    if img is None:
        raise FileNotFoundError(img_file)
    az, el, distance_ratio = param[0], param[1], param[3]
    K, RT = getBlenderProj(az, el, distance_ratio, img_w=137, img_h=137)
    trans_mat = np.linalg.multi_dot([K, RT, rot_mat, norm_mat])
    regress_mat = np.transpose(np.linalg.multi_dot([RT, rot_mat, norm_mat]))
    return {"img_arr": img.astype(np.uint8), "trans_mat": np.transpose(trans_mat).astype(np.float32),
            "K": K.astype(np.float32), "RT": RT.astype(np.float32), "obj_rot_mat": obj_rot_mat.astype(np.float32),
            "regress_mat": regress_mat.astype(np.float32)}


def gen_obj_img_h5(source_dir, cat_target_dir, sdf_dir, vals, obj):
    """:156-197: the view files of one object; returns the paths written."""
    img_dir = os.path.join(source_dir, vals, obj, "rendering")
    tar_obj_dir = os.path.join(cat_target_dir, obj)
    os.makedirs(tar_obj_dir, exist_ok=True)
    norm_mat = get_norm_matrix(os.path.join(sdf_dir, vals, obj, "ori_sample.npz"))
    rot_mat = get_rotate_matrix(-np.pi / 2)
    with open(img_dir + "/renderings.txt", "r") as f:
        file_lst = [line.strip() for line in f.read().splitlines()]
    params = np.loadtxt(img_dir + "/rendering_metadata.txt")
    written = []
    for i in range(len(file_lst)):
        view_file = os.path.join(tar_obj_dir, file_lst[i][:2] + ".npz")
        if os.path.exists(view_file):
            try:
                with np.load(view_file) as fh:
                    print("{} exist! trans first shape is {}".format(view_file, fh["trans_mat"].shape[0]))
                continue
            except Exception:
                print("{} exist! but file error".format(view_file))
        d = view_datasets(os.path.join(img_dir, file_lst[i]), params[i, ...].astype(np.float32), norm_mat, rot_mat)
        np.savez(view_file, **d)
        print("write:", view_file)
        written.append(view_file)
    return written


def convert_img2h5(source_dir, target_dir, file_lst_dir, cats, sdf_dir):
    """:126-153: every object of each category's train and test lists (sequentially; the reference uses 10 jobs)."""
    os.makedirs(target_dir, exist_ok=True)
    for vals in cats.values():
        cat_target_dir = os.path.join(target_dir, vals)
        os.makedirs(cat_target_dir, exist_ok=True)
        fs = []
        for split in ("train", "test"):
            with open(os.path.join(file_lst_dir, vals + "_%s.lst" % split), "r") as f:
                fs += [obj.rstrip("\r\n") for obj in f.readlines()]
        for obj in fs:
            gen_obj_img_h5(source_dir, cat_target_dir, sdf_dir, vals, obj)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--source_dir", required=True, help="ShapeNetRendering: <cat>/<obj>/rendering/")
    ap.add_argument("--view_dir", required=True, help="output: <view_dir>/<cat>/<obj>/%%02d.npz")
    ap.add_argument("--sdf_dir", required=True, help="<sdf_dir>/<cat>/<obj>/ori_sample.npz")
    ap.add_argument("--lst_dir", required=True, help="<cat>_train.lst and <cat>_test.lst")
    ap.add_argument("--cats", nargs="+", required=True, help="category ids")
    a = ap.parse_args(argv)
    convert_img2h5(a.source_dir, a.view_dir, a.lst_dir, {c: c for c in a.cats}, a.sdf_dir)


if __name__ == "__main__":
    main()
