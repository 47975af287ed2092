"""Test-set loader of the camera network, the reference's ``data/data_sdf_h5_queue_mask_imgh5_cammat.py``
``Pt_sdf_img``, for ``train_sdf_cam --test / --create``.

It is the SDF loader (data_sdf_h5_queue.Pt_sdf_img: queue, thread, epoch order, category limits) with the batches of
:232-334: the image is the view file's ``img_arr[:, :, :4] / 255`` (RGBA, no background handling; the network is fed
its RGB channels), the batch also holds ``RT`` (the view file's ``regress_mat``) and ``shifts`` (zeros), and the SDF
samples are always drawn with replacement by ``np.random.randint``.  The draws are the reference's, in its order:
``np.random.shuffle`` of the epoch order, then per view ``np.random.randint`` for ``pc`` and for ``sdf_pt``.
"""
from __future__ import annotations

import os

import numpy as np

from . import data_sdf_h5_queue


class Pt_sdf_img(data_sdf_h5_queue.Pt_sdf_img):
    def get_img(self, img_dir, num):
        """:161-180 (FLAGS.img_feat): the RGBA image as float32 / 255, trans_mat and RT = regress_mat."""
        with np.load(os.path.join(img_dir, "%02d.npz" % num)) as f:
            trans_mat = f["trans_mat"].astype(np.float32)
            RT = f["regress_mat"].astype(np.float32)
            img_arr = f["img_arr"][:, :, :4].astype(np.float32) / 255.
        return img_arr, trans_mat, RT

    def get_batch(self, index):
        """:232-334 without --shift and --rotation."""
        if index + self.batch_size > self.epoch_amount:
            index = index + self.batch_size - self.epoch_amount
        bs, F = self.batch_size, self.FLAGS
        batch_pc = np.zeros((bs, self.num_points, 3), np.float32)
        batch_sdf_pt = np.zeros((bs, self.gen_num_pt, 3), np.float32)
        batch_sdf_pt_rot = np.zeros((bs, self.gen_num_pt, 3), np.float32)
        batch_sdf_val = np.zeros((bs, self.gen_num_pt, 1), np.float32)
        batch_norm_params = np.zeros((bs, 4), np.float32)
        batch_sdf_params = np.zeros((bs, 6), np.float32)
        batch_img = np.zeros((bs, F.img_h, F.img_w, 4), np.float32)
        batch_trans_mat = np.zeros((bs, 4, 3), np.float32)
        batch_RT_mat = np.zeros((bs, 4, 3), np.float32)
        batch_shifts = np.zeros((bs, 2), np.float32)
        batch_cat_id, batch_obj_nm, batch_view_id = [], [], []
        for cnt, i in enumerate(range(index, index + bs)):
            ori_pt, _, sample_pt, sample_sdf_val, norm_params, sdf_params, img_dir, cat_id, obj, num = \
                self.getitem(self.order[i])
            img, trans_mat, RT = self.get_img(img_dir, num)
            cf_ref_choice = np.random.randint(ori_pt.shape[0], size=self.num_points)
            batch_pc[cnt, :, :] = ori_pt[cf_ref_choice, :]
            choice = np.random.randint(sample_pt.shape[0], size=self.gen_num_pt)
            batch_sdf_pt[cnt, ...] = sample_pt[choice, :]
            batch_sdf_val[cnt, :, 0] = sample_sdf_val[choice]
            batch_norm_params[cnt, ...] = norm_params
            batch_sdf_params[cnt, ...] = sdf_params
            batch_img[cnt, ...] = img
            batch_trans_mat[cnt, ...] = trans_mat
            batch_RT_mat[cnt, ...] = RT
            batch_cat_id.append(cat_id)
            batch_obj_nm.append(obj)
            batch_view_id.append(num)
        return {"pc": batch_pc, "sdf_pt": batch_sdf_pt, "sdf_pt_rot": batch_sdf_pt_rot, "sdf_val": batch_sdf_val,
                "norm_params": batch_norm_params, "sdf_params": batch_sdf_params, "img": batch_img,
                "trans_mat": batch_trans_mat, "RT": batch_RT_mat, "cat_id": batch_cat_id, "obj_nm": batch_obj_nm,
                "view_id": batch_view_id, "shifts": batch_shifts}
