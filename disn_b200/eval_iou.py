"""Mirror of the reference's ``test/test_iou.py``: volumetric IoU of every reconstructed view against the ground-truth
isosurface at dim^3 voxels.  Same functions, draws and printed lines; the voxelisation runs on the GPU (iou.cu) instead
of PyMesh's VoxelGrid, and an object's views are scored in one Engine.iou_views call, which voxelises the ground truth
once, instead of one iou_pymesh call per view in a joblib pool.

    python -m disn_b200.eval_iou --cal_dir <test_objs/65_0.0> --gt_dir <norm_mesh_dir> --test_lst_dir <filelists> \\
        [--category all] [--view_num 24] [--dim 110]

Only view files larger than 200 bytes count.  An object with fewer of them than --view_num is scored on
np.random.randint draws with replacement, the others on random.sample, as in the reference.  A mesh without faces
raises ValueError naming its file.  The reference's __main__ passes dim=110 whatever --dim says; here --dim (default
110) is used.
"""
from __future__ import annotations

import argparse
import os
import random

import numpy as np

from .eval_common import CATS_CLEAN_IOU, listdir, read_lst, read_mesh, select_cats

_ENGINE = None
_DEVICE = 0


def _engine():
    global _ENGINE
    if _ENGINE is None:
        from .engine import Engine
        _ENGINE = Engine(device=_DEVICE, precision="fp32")
    return _ENGINE


def _read_mesh(path):
    verts, faces = read_mesh(_engine(), path)
    if len(faces) == 0:
        raise ValueError("%s: mesh has no faces, its IoU is undefined" % path)
    return verts, faces


def build_file_dict(dir, view_num=24):
    """test_iou.py:123-145: files of dir larger than 200 bytes grouped by object id, then view_num of them per object
    (np.random.randint with replacement when there are fewer, random.sample otherwise)."""
    file_dict = {}
    for file in listdir(dir):
        full_path = os.path.join(dir, file)
        if os.path.isfile(full_path) and os.stat(full_path)[6] > 200:
            file_dict.setdefault(file.split("_")[1], []).append(full_path)
    for obj_id in file_dict.keys():
        paths = file_dict[obj_id]
        if len(paths) < view_num:
            choice = np.random.randint(len(paths), size=view_num)
            file_dict[obj_id] = [paths[ind] for ind in choice]
        else:
            file_dict[obj_id] = random.sample(paths, view_num)
    return file_dict


def iou_all(cats, pred_dir, gt_dir, test_lst_dir, dim=110, view_num=24):
    """test_iou.py:165-172 -> {cat_nm: (iou_avg, best_iou_pred_lst)}."""
    out = {}
    for cat_nm, cat_id in cats.items():
        pred_dir_cat = os.path.join(pred_dir, cat_id)
        gt_dir_cat = os.path.join(gt_dir, cat_id)
        test_lst_f = os.path.join(test_lst_dir, cat_id + "_test.lst")
        iou_avg, best_iou_pred_lst = iou_cat(pred_dir_cat, gt_dir_cat, test_lst_f, dim=dim, view_num=view_num)
        print("cat_nm: {}, cat_id: {}, iou_avg: {}".format(cat_nm, cat_id, iou_avg))
        out[cat_nm] = (iou_avg, best_iou_pred_lst)
    print("done!")
    return out


def iou_cat(pred_dir, gt_dir, test_lst_f, dim=110, view_num=24):
    """test_iou.py:174-206 with one Engine.iou_views call per object -> (mean IoU over every scored view,
    [[best iou, best view's path] per object])."""
    pred_dict = build_file_dict(pred_dir, view_num=view_num)
    iou_sum = 0.0
    count = 0.0
    best_iou_pred_lst = []
    for obj_id in read_lst(test_lst_f):
        src_path = os.path.join(gt_dir, obj_id, "isosurf.obj")
        pred_path_lst = pred_dict[obj_id]
        result_lst = iou_views(src_path, pred_path_lst, dim)
        iou_vals = np.asarray([result[0] for result in result_lst], dtype=np.float32)
        sum_iou = np.sum(iou_vals)
        iou_sum += sum_iou
        count += len(iou_vals)
        avg_iou = np.mean(iou_vals)
        ind = np.argmax(iou_vals)
        best_iou_pred_lst.append(result_lst[ind])
        print("obj_id iou avg: ", avg_iou, " best pred: ", result_lst[ind])
    return iou_sum / count, best_iou_pred_lst


def iou_views(mesh_src, mesh_preds, dim=110):
    """iou_pymesh of mesh_src against every file of mesh_preds in one Engine.iou_views call (files named more than
    once are read once) -> [[iou, path] per file]."""
    src_v, src_f = _read_mesh(mesh_src)
    meshes = {p: _read_mesh(p) for p in dict.fromkeys(mesh_preds)}
    _, inter, uni = _engine().iou_views(src_v, src_f, [meshes[p] for p in mesh_preds], dim=dim)
    return [[float(i) / u, p] for i, u, p in zip(inter, uni, mesh_preds)]


def iou_pymesh(mesh_src, mesh_pred, dim=110):
    """test_iou.py:208-233 for one pair (Engine.iou) -> [iou, mesh_pred]."""
    v1, f1 = _read_mesh(mesh_src)
    v2, f2 = _read_mesh(mesh_pred)
    _, inter, uni, _, _ = _engine().iou(v1, f1, v2, f2, dim=dim, want_grids=True)
    return [float(inter) / np.int64(uni), mesh_pred]


def main(argv=None):
    global _DEVICE
    parser = argparse.ArgumentParser()
    parser.add_argument("--cal_dir", type=str, default="", help="target obj directory that needs to be tested")
    parser.add_argument("--gt_dir", type=str, required=True,
                        help="ground-truth isosurfaces <cat_id>/<obj_id>/isosurf.obj (create_point_sdf_grid's norm_mesh_dir)")
    parser.add_argument("--test_lst_dir", type=str, required=True, help="test mesh data list")
    parser.add_argument("--category", default="all", help="all, clean or one category name")
    parser.add_argument("--view_num", type=int, default=24, help="how many views do you want to create for each obj")
    parser.add_argument("--dim", type=int, default=110, help="voxels per axis")
    parser.add_argument("--gpu", type=int, default=0, help="CUDA device index")
    flags = parser.parse_args(argv)
    print(flags)
    _DEVICE = flags.gpu
    return iou_all(select_cats(flags.category, CATS_CLEAN_IOU), flags.cal_dir, flags.gt_dir, flags.test_lst_dir,
                   dim=flags.dim, view_num=flags.view_num)


if __name__ == "__main__":
    main()
