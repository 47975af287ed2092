"""Mirror of the reference's ``test/test_f_score.py``: precision, recall and F-score of the reconstructed views at six
distance thresholds, from the point files ``eval_cd_emd --save_pnt`` writes.  Same functions, caches and arithmetic;
the nearest-neighbour distances come from the GPU (Engine.nn_distance: chamfer.cu) instead of TF's tf_nndistance op.

    python -m disn_b200.eval_f_score --cal_dir <test_objs/65_0.0> --gt_dir <norm_mesh_dir> --test_lst_dir <filelists> \\
        [--category all] [--view_num 24] [--num_sample_points 2048] [--batch_size 24] [--truethreshold 2.5]

The distances of an object are cached in ``<cal_dir>/pnt_<N>_<cat_id>/for_dist_<obj>.txt`` / ``bac_dist_<obj>.txt``:
written on the first run and read back (float64) on later runs.  Computing them needs ``--batch_size`` equal to
``--view_num``; any other value raises NotImplementedError, as in the reference.
"""
from __future__ import annotations

import argparse
import os

import numpy as np

from .eval_common import listdir, read_lst, select_cats

_ENGINE = None
_DEVICE = 0
THRESHOLDS = [[0.5], [1], [2], [5], [10], [20]]     # test_f_score.py:291, in percent of truethreshold


def _engine():
    global _ENGINE
    if _ENGINE is None:
        from .engine import Engine
        _ENGINE = Engine(device=_DEVICE, precision="fp32")
    return _ENGINE


def build_file_dict(dir):
    """test_f_score.py:129-139: files of dir grouped by object id."""
    file_dict = {}
    for file in listdir(dir):
        full_path = os.path.join(dir, file)
        if os.path.isfile(full_path):
            file_dict.setdefault(file.split("_")[1], []).append(full_path)
    return file_dict


def cal_f_score_all_cat(cats, pred_dir, gt_dir, test_lst_dir, threshold_lst, side_len, view_num=24,
                        num_sample_points=2048, batch_size=24):
    """test_f_score.py:159-181: per-category precision / recall averaged over the categories with their object counts as
    weights; F from the averaged P and R.  Returns (per_cat {cat_nm: (precision_avg, recall_avg, cnt)}, pre_w_avg,
    rec_w_avg, f_score)."""
    precision_lst = []
    recall_lst = []
    cnt_lst = []
    per_cat = {}
    for cat_nm, cat_id in cats.items():
        pred_dir_cat = os.path.join(pred_dir, cat_id)
        gt_dir_cat = os.path.join(gt_dir, cat_id)
        test_lst_f = os.path.join(test_lst_dir, cat_id + "_test.lst")
        thresholds = np.asarray(threshold_lst, dtype=np.float32) * 0.01 * side_len
        precision_avg, recall_avg, cnt = f_score_cat(cat_id, cat_nm, pred_dir_cat, gt_dir_cat, test_lst_f, thresholds,
                                                     view_num=view_num, num_sample_points=num_sample_points,
                                                     batch_size=batch_size)
        precision_lst.append(precision_avg)
        recall_lst.append(recall_avg)
        cnt_lst.append(cnt)
        per_cat[cat_nm] = (precision_avg, recall_avg, cnt)
        print("{}, {}, precision_avg {}, recal_avg{}, count {}".format(cat_nm, cat_id, precision_avg, recall_avg, cnt))
    print("done!")
    precision = np.asarray(precision_lst)
    recall = np.asarray(recall_lst)
    pre_w_avg = np.average(precision, axis=0, weights=cnt_lst)
    rec_w_avg = np.average(recall, axis=0, weights=cnt_lst)
    f_score = 2 * (pre_w_avg * rec_w_avg) / (pre_w_avg + rec_w_avg)
    print("pre_w_avg {}, rec_w_avg {}, f_score {}".format(pre_w_avg, rec_w_avg, f_score))
    return per_cat, pre_w_avg, rec_w_avg, f_score


def f_score_cat(cat_id, cat_nm, pred_dir, gt_dir, test_lst_f, thresholds, view_num=24, num_sample_points=2048,
                batch_size=24):
    """test_f_score.py:183-243 -> (precision_sum / count, recall_sum / count, count), one value per threshold."""
    pred_dict = build_file_dict(pred_dir)
    count = 0
    precision_sum = 0
    recall_sum = 0
    for obj_id in read_lst(test_lst_f):
        pred_pnt_dir = os.path.join(os.path.dirname(pred_dir), "pnt_{}_{}".format(num_sample_points, cat_id))
        forfl = os.path.join(pred_pnt_dir, "for_dist_{}.txt".format(obj_id))
        backfl = os.path.join(pred_pnt_dir, "bac_dist_{}.txt".format(obj_id))
        if not os.path.exists(forfl):
            gt_pnt_path = os.path.join(gt_dir, obj_id, "pnt_{}.txt".format(num_sample_points))
            gt_pnts = np.loadtxt(gt_pnt_path, dtype=float, delimiter=',')
            pred_path_lst = pred_dict[obj_id]
            verts_batch = np.zeros((view_num + 1, num_sample_points, 3), dtype=np.float32)
            verts_batch[0, ...] = gt_pnts
            for i in range(len(pred_path_lst)):
                view_id = pred_path_lst[i][-6:-4]
                pred_pnt_path = os.path.join(pred_pnt_dir, "pnt_{}_{}.txt".format(obj_id, view_id))
                verts_batch[i + 1, ...] = np.loadtxt(pred_pnt_path, dtype=float, delimiter=',')
            if batch_size == view_num:
                dists_forward_sqrt_val, dists_backward_sqrt_val = get_points_distance(verts_batch)
            else:
                raise NotImplementedError("computing the distances needs batch_size == view_num")
            np.savetxt(forfl, dists_forward_sqrt_val)
            np.savetxt(backfl, dists_backward_sqrt_val)
        else:
            dists_forward_sqrt_val = np.loadtxt(forfl)
            dists_backward_sqrt_val = np.loadtxt(backfl)
        dists_forward_sqrt_val = np.tile(dists_forward_sqrt_val, [thresholds.shape[0], 1])
        dists_backward_sqrt_val = np.tile(dists_backward_sqrt_val, [thresholds.shape[0], 1])
        pre_sum_val = np.sum(np.less(dists_forward_sqrt_val, thresholds), axis=1)
        rec_sum_val = np.sum(np.less(dists_backward_sqrt_val, thresholds), axis=1)
        precision = pre_sum_val / (dists_forward_sqrt_val.shape[1])
        recall = rec_sum_val / (dists_backward_sqrt_val.shape[1])
        print("cat_id {}, obj_id {}: pre_sum {}, rec_sum {}, precision {}, recall {}"
              .format(cat_id, obj_id, pre_sum_val, rec_sum_val, precision, recall))
        precision_sum += precision
        recall_sum += recall
        count += 1
    return precision_sum / count, recall_sum / count, count


def get_points_distance(sampled_pc):
    """test_f_score.py:245-258: sampled_pc [1+V,N,3] -> float32 sqrt of the squared NN distances of every view to the
    ground truth (forward) and back, each flattened over all views (one nn_distance call with B = V)."""
    pc = np.ascontiguousarray(sampled_pc, np.float32)
    pred = pc[1:]
    src = np.ascontiguousarray(np.broadcast_to(pc[:1], pred.shape))
    dists_forward, _, dists_backward, _ = _engine().nn_distance(pred, src)
    return np.sqrt(dists_forward).reshape(-1), np.sqrt(dists_backward).reshape(-1)


def main(argv=None):
    global _DEVICE
    parser = argparse.ArgumentParser()
    parser.add_argument("--cal_dir", type=str, default="", help="target obj directory that needs to be tested")
    parser.add_argument("--gt_dir", type=str, required=True,
                        help="ground-truth directory <cat_id>/<obj_id>/ holding pnt_<N>.txt (eval_cd_emd --save_pnt)")
    parser.add_argument("--test_lst_dir", type=str, required=True, help="test mesh data list")
    parser.add_argument("--category", default="all", help="all, clean or one category name")
    parser.add_argument("--view_num", type=int, default=24, help="how many views do you want to create for each obj")
    parser.add_argument("--num_sample_points", type=int, default=2048, help="Sample Point Number for each obj to test")
    parser.add_argument("--batch_size", type=int, default=24, help="must equal view_num to compute distances")
    parser.add_argument("--truethreshold", type=float, default=2.5, help="if distance smaller than this value, its true")
    parser.add_argument("--gpu", type=int, default=0, help="CUDA device index")
    flags = parser.parse_args(argv)
    print(flags)
    _DEVICE = flags.gpu
    return cal_f_score_all_cat(select_cats(flags.category), flags.cal_dir, flags.gt_dir, flags.test_lst_dir, THRESHOLDS,
                               flags.truethreshold, view_num=flags.view_num, num_sample_points=flags.num_sample_points,
                               batch_size=flags.batch_size)


if __name__ == "__main__":
    main()
