"""Mirror of the reference's ``test/test_cd_emd.py``: Chamfer distance and approximate EMD of every reconstructed view
against the ground-truth isosurface, per object and per category.  Same functions and draws; the metric runs on the
GPU (Engine.points_loss: chamfer.cu + emd.cu) instead of TF's tf_nndistance / tf_approxmatch ops.

    python -m disn_b200.eval_cd_emd --cal_dir <test_objs/65_0.0> --gt_dir <norm_mesh_dir> --test_lst_dir <filelists> \\
        [--category all] [--view_num 24] [--num_sample_points 2048] [--batch_size 24] [--save_pnt]

``--gt_dir`` is the directory ``create_point_sdf_grid --norm_mesh_dir`` writes (``<cat_id>/<obj_id>/isosurf.obj``),
the reference's ``info.json`` norm_mesh_dir.  ``--save_pnt`` also writes the sampled point files that
``eval_f_score`` reads (the reference's sample_save_gt_pnt / sample_save_pred_pnt, reachable there only by editing
``__main__``).  They hold the float32 vertices read_obj returns where the reference saves PyMesh's float64 copy;
eval_f_score reads either into float32, so its results do not change.

Only ``--batch_size`` equal to ``--view_num`` (the README's command) compares every view in one metric call.
``--batch_size 1`` reproduces the reference's per-view loop exactly, which pairs the ground truth with
``verts_batch[b]`` for b in range(view_num): b = 0 is the ground truth itself and the last view is never read.
Any other batch size raises ValueError (the reference fails on its placeholder's shape).
"""
from __future__ import annotations

import argparse
import os
import random

import numpy as np

from .create_sdf import read_obj
from .eval_common import listdir, read_lst, select_cats

_ENGINE = None
_DEVICE = 0


def _engine():
    global _ENGINE
    if _ENGINE is None:
        from .engine import Engine
        _ENGINE = Engine(device=_DEVICE, precision="fp32")
    return _ENGINE


def build_file_dict(dir):
    """test_cd_emd.py:126-136: files of dir grouped by object id (second `_` field of <cat_id>_<obj_id>_<view>.obj)."""
    file_dict = {}
    for file in listdir(dir):
        full_path = os.path.join(dir, file)
        if os.path.isfile(full_path):
            file_dict.setdefault(file.split("_")[1], []).append(full_path)
    return file_dict


def cd_emd_all(cats, pred_dir, gt_dir, test_lst_dir, view_num=24, num_sample_points=2048, batch_size=24):
    """test_cd_emd.py:155-161 -> {cat_nm: cd_emd_cat(...)}."""
    out = {}
    for cat_nm, cat_id in cats.items():
        pred_dir_cat = os.path.join(pred_dir, cat_id)
        gt_dir_cat = os.path.join(gt_dir, cat_id)
        test_lst_f = os.path.join(test_lst_dir, cat_id + "_test.lst")
        out[cat_nm] = cd_emd_cat(cat_id, cat_nm, pred_dir_cat, gt_dir_cat, test_lst_f, view_num=view_num,
                                 num_sample_points=num_sample_points, batch_size=batch_size)
    print("done!")
    return out


def _sample(verts, num_sample_points):
    """One draw of num_sample_points vertices (np.random.randint), or zeros for a mesh without vertices (no draw)."""
    if verts.shape[0] > 0:
        return verts[np.random.randint(verts.shape[0], size=num_sample_points), ...]
    return np.zeros((num_sample_points, 3), np.float32)


def cd_emd_cat(cat_id, cat_nm, pred_dir, gt_dir, test_lst_f, view_num=24, num_sample_points=2048, batch_size=24):
    """test_cd_emd.py:220-288.  Returns (rows, avg_cf, avg_emd): one row (src_path, avg_cf, min_cf, arg_cf, avg_emd,
    min_emd, arg_emd) per object of the list, then the category means it prints."""
    if batch_size not in (view_num, 1):
        raise ValueError("batch_size must be view_num (%d) or 1, got %d" % (view_num, batch_size))
    pred_dict = build_file_dict(pred_dir)
    sum_cf_loss = 0.
    sum_em_loss = 0.
    count = 1
    rows = []
    test_objs = read_lst(test_lst_f)
    for obj_id in test_objs:
        src_path = os.path.join(gt_dir, obj_id, "isosurf.obj")
        pred_path_lst = pred_dict[obj_id]
        verts_batch = np.zeros((view_num + 1, num_sample_points, 3), dtype=np.float32)
        verts_batch[0, ...] = _sample(read_obj(src_path)[0], num_sample_points)
        pred_path_lst = random.sample(pred_path_lst, view_num)
        for i in range(len(pred_path_lst)):
            verts = read_obj(pred_path_lst[i])[0]
            if verts.shape[0] > 0:
                verts_batch[i + 1, ...] = _sample(verts, num_sample_points)
        if batch_size == view_num:
            avg_cf_loss_val, min_cf_loss_val, arg_min_cf_val, avg_em_loss_val, min_em_loss_val, arg_min_em_val \
                = _engine().points_loss(verts_batch)
        else:
            sum_avg_cf_loss_val = 0.
            min_cf_loss_val = 9999.
            arg_min_cf_val = 0
            sum_avg_em_loss_val = 0.
            min_em_loss_val = 9999.
            arg_min_em_val = 0
            for b in range(view_num // batch_size):
                verts_batch_b = np.stack([verts_batch[0, ...], verts_batch[b, ...]])
                avg_cf_loss_val, _, _, avg_em_loss_val, _, _ = _engine().points_loss(verts_batch_b)
                sum_avg_cf_loss_val += avg_cf_loss_val
                sum_avg_em_loss_val += avg_em_loss_val
                if min_cf_loss_val > avg_cf_loss_val:
                    min_cf_loss_val = avg_cf_loss_val
                    arg_min_cf_val = b
                if min_em_loss_val > avg_em_loss_val:
                    min_em_loss_val = avg_em_loss_val
                    arg_min_em_val = b
            avg_cf_loss_val = sum_avg_cf_loss_val / (view_num // batch_size)
            avg_em_loss_val = sum_avg_em_loss_val / (view_num // batch_size)
        sum_cf_loss += avg_cf_loss_val
        sum_em_loss += avg_em_loss_val
        print(str(count) + " ", src_path, "avg cf:{}, min_cf:{}, arg_cf view:{}, avg emd:{}, min_emd:{}, arg_em view:{}".
              format(str(avg_cf_loss_val), str(min_cf_loss_val), str(arg_min_cf_val),
                     str(avg_em_loss_val), str(min_em_loss_val), str(arg_min_em_val)))
        rows.append((src_path, avg_cf_loss_val, min_cf_loss_val, arg_min_cf_val, avg_em_loss_val, min_em_loss_val,
                     arg_min_em_val))
    avg_cf, avg_emd = sum_cf_loss / len(test_objs), sum_em_loss / len(test_objs)
    print("cat_nm:{}, cat_id:{}, avg_cf:{}, avg_emd:{}".format(cat_nm, cat_id, avg_cf, avg_emd))
    return rows, avg_cf, avg_emd


def save_all_cat_gt_pnt(cats, gt_dir, test_lst_dir, num_sample_points=2048):
    """test_cd_emd.py:163-168."""
    for cat_nm, cat_id in cats.items():
        gt_dir_cat = os.path.join(gt_dir, cat_id)
        test_lst_f = os.path.join(test_lst_dir, cat_id + "_test.lst")
        sample_save_gt_pnt(cat_id, cat_nm, gt_dir_cat, test_lst_f, num_sample_points=num_sample_points)
    print("done!")


def sample_save_gt_pnt(cat_id, cat_nm, gt_dir_cat, test_lst_f, num_sample_points=2048):
    """test_cd_emd.py:170-186: num_sample_points vertices of <obj>/isosurf.obj -> <obj>/pnt_<N>.txt (comma separated).
    Returns the list of files written."""
    saved = []
    for obj_id in read_lst(test_lst_f):
        obj_path = os.path.join(gt_dir_cat, obj_id, "isosurf.obj")
        verts_batch = _sample(read_obj(obj_path)[0], num_sample_points)
        savefn = os.path.join(gt_dir_cat, obj_id, "pnt_{}.txt".format(num_sample_points))
        np.savetxt(savefn, verts_batch, delimiter=',')
        print("saved gt pnt of {} at {}".format(obj_id, savefn))
        saved.append(savefn)
    return saved


def save_all_cat_pred_pnt(cats, pred_dir, test_lst_dir, view_num=24, num_sample_points=2048):
    """test_cd_emd.py:189-194."""
    for cat_nm, cat_id in cats.items():
        pred_dir_cat = os.path.join(pred_dir, cat_id)
        test_lst_f = os.path.join(test_lst_dir, cat_id + "_test.lst")
        sample_save_pred_pnt(cat_id, cat_nm, pred_dir_cat, test_lst_f, view_num=view_num,
                             num_sample_points=num_sample_points)
    print("done!")


def sample_save_pred_pnt(cat_id, cat_nm, pred_dir, test_lst_f, view_num=24, num_sample_points=2048):
    """test_cd_emd.py:196-216: num_sample_points vertices of every view file -> <pred_dir>/../pnt_<N>_<cat_id>/
    pnt_<obj>_<view>.txt, <view> being the two characters before ".obj".  Returns the list of files written."""
    pred_dict = build_file_dict(pred_dir)
    saved = []
    for obj_id in read_lst(test_lst_f):
        pred_path_lst = pred_dict[obj_id]
        verts_batch = np.zeros((view_num, num_sample_points, 3), dtype=np.float32)
        for i in range(len(pred_path_lst)):
            pred_mesh_fl = pred_path_lst[i]
            verts = read_obj(pred_mesh_fl)[0]
            if verts.shape[0] > 0:
                verts_batch[i, ...] = _sample(verts, num_sample_points)
            savedir = os.path.join(os.path.dirname(pred_dir), "pnt_{}_{}".format(num_sample_points, cat_id))
            os.makedirs(savedir, exist_ok=True)
            view_id = pred_mesh_fl[-6:-4]
            savefn = os.path.join(savedir, "pnt_{}_{}.txt".format(obj_id, view_id))
            print(savefn)
            np.savetxt(savefn, verts_batch[i, ...], delimiter=',')
            print("saved gt pnt of {} at {}".format(obj_id, savefn))
            saved.append(savefn)
    return saved


def main(argv=None):
    global _DEVICE
    parser = argparse.ArgumentParser()
    parser.add_argument("--cal_dir", type=str, default="", help="target obj directory that needs to be tested")
    parser.add_argument("--gt_dir", type=str, required=True,
                        help="ground-truth isosurfaces <cat_id>/<obj_id>/isosurf.obj (create_point_sdf_grid's norm_mesh_dir)")
    parser.add_argument("--test_lst_dir", type=str, required=True, help="test mesh data list")
    parser.add_argument("--category", default="all", help="all, clean or one category name")
    parser.add_argument("--view_num", type=int, default=24, help="how many views do you want to create for each obj")
    parser.add_argument("--num_sample_points", type=int, default=2048, help="Sample Point Number for each obj to test")
    parser.add_argument("--batch_size", type=int, default=24, help="view_num (every view in one call) or 1")
    parser.add_argument("--gpu", type=int, default=0, help="CUDA device index")
    parser.add_argument("--save_pnt", action="store_true", help="also write the point files eval_f_score reads")
    flags = parser.parse_args(argv)
    print(flags)
    _DEVICE = flags.gpu
    cats = select_cats(flags.category)
    out = cd_emd_all(cats, flags.cal_dir, flags.gt_dir, flags.test_lst_dir, view_num=flags.view_num,
                     num_sample_points=flags.num_sample_points, batch_size=flags.batch_size)
    if flags.save_pnt:
        save_all_cat_gt_pnt(cats, flags.gt_dir, flags.test_lst_dir, num_sample_points=flags.num_sample_points)
        save_all_cat_pred_pnt(cats, flags.cal_dir, flags.test_lst_dir, view_num=flags.view_num,
                              num_sample_points=flags.num_sample_points)
    return out


if __name__ == "__main__":
    main()
