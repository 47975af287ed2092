"""Test-set loader, the reference's ``data/data_sdf_h5_queue.py`` ``Pt_sdf_img`` for the inference drivers.

A background thread builds ``batch_data`` dicts (the layout of :256-303: pc, sdf_pt, sdf_pt_rot, sdf_val, norm_params,
sdf_params, img, trans_mat, cat_id, obj_nm, view_id) from the view files of create_img_h5 and the ``ori_sample.npz`` of
create_point_sdf_grid, and queues them; ``fetch`` takes the next one and ``shutdown`` stops it.  The random draws are the
reference's, in its order: ``np.random.shuffle`` of the epoch order (refill_data_order, with shuffle), then per view
``np.random.randint`` for ``pc`` and ``random.sample`` (or ``np.random.randint`` when the file holds fewer samples) for
``sdf_pt``.

Flags the reference reads without defining them in test_sdf_acc's parser (img_feat_onestream, augcolorfore,
augcolorback) count as False.  --alpha, --rot, --binary, --threedcnn and --multi_view are refused: they select ablation
branches, and --rot needs a host np.dot the device does not reproduce.
"""
from __future__ import annotations

import copy
import os
import queue
import random
import threading

import numpy as np

REFUSED_FLAGS = ("alpha", "rot", "binary", "threedcnn", "multi_view")


def check_flags(FLAGS):
    for flag in REFUSED_FLAGS:
        if getattr(FLAGS, flag, False):
            raise NotImplementedError("--%s is not supported by the test-set loader: it selects an ablation branch of the "
                                      "reference (or, for --rot, a host rotation of the samples)" % flag)


class Pt_sdf_img(threading.Thread):
    def __init__(self, FLAGS, listinfo=None, info=None, qsize=64, cats_limit=None, shuffle=True):
        check_flags(FLAGS)
        super().__init__(daemon=True)
        self.queue = queue.Queue(qsize)
        self.stopped = False
        self.bno = 0
        self.listinfo = listinfo
        self.num_points = FLAGS.num_points
        self.gen_num_pt = FLAGS.num_sample_points
        self.batch_size = FLAGS.batch_size
        self.img_dir = info["rendered_dir"]
        self.sdf_dir = info["sdf_dir"]
        self.data_num = len(self.listinfo)
        self.FLAGS = FLAGS
        self.shuffle = shuffle
        self.num_batches = int(self.data_num / self.FLAGS.batch_size)
        self.cats_limit, self.epoch_amount = self.set_cat_limit(cats_limit)
        self.data_order = list(range(len(listinfo)))
        self.order = self.data_order

    def set_cat_limit(self, cats_limit):
        epoch_amount = 0
        for cat, amount in cats_limit.items():
            cats_limit[cat] = min(self.FLAGS.cat_limit, amount)
            epoch_amount += cats_limit[cat]
        print("epoch_amount ", epoch_amount)
        print("cats_limit ", cats_limit)
        return cats_limit, epoch_amount

    def __len__(self):
        return self.epoch_amount

    def get_sdf_h5_filenm(self, cat_id, obj):
        return os.path.join(self.sdf_dir, cat_id, obj, "ori_sample.npz")

    def get_sdf_h5(self, sdf_file, cat_id, obj):
        """:147-168 on the .npz of create_point_sdf_grid."""
        with np.load(sdf_file) as f:
            if not all(k in f for k in ("pc_sdf_original", "pc_sdf_sample", "norm_params")):
                raise Exception(cat_id, obj, "no sdf and sample")
            ori_pt = f["pc_sdf_original"].astype(np.float32)[:, :3]
            sample_sdf = f["pc_sdf_sample"].astype(np.float32)
            if sample_sdf.shape[1] == 4:
                sample_pt, sample_sdf_val = sample_sdf[:, :3], sample_sdf[:, 3]
            else:
                sample_pt, sample_sdf_val = None, sample_sdf[:, 0]
            return ori_pt, None, sample_pt, sample_sdf_val, f["norm_params"], f["sdf_params"]

    def getitem(self, index):
        cat_id, obj, num = self.listinfo[index]
        ori_pt, ori_sdf_val, sample_pt, sample_sdf_val, norm_params, sdf_params = self.get_sdf_h5(
            self.get_sdf_h5_filenm(cat_id, obj), cat_id, obj)
        return (ori_pt, ori_sdf_val, sample_pt, sample_sdf_val, norm_params, sdf_params,
                os.path.join(self.img_dir, cat_id, obj), cat_id, obj, num)

    def get_img(self, img_dir, num):
        """:178-211 for the twostream model: the view file's image as float32 / 255 and its matrices."""
        with np.load(os.path.join(img_dir, "%02d.npz" % num)) as f:
            trans_mat = f["trans_mat"].astype(np.float32)
            regress_mat = f["regress_mat"].astype(np.float32)
            img_raw = f["img_arr"]
        img_arr = img_raw[:, :, :3].copy()
        if self.FLAGS.backcolorwhite:
            img_arr[img_raw[:, :, 3] == 0] = [255, 255, 255]
        img_arr = np.clip(img_arr, 0, 255)
        return img_arr.astype(np.float32) / 255., trans_mat, regress_mat

    def get_batch(self, index):
        """:256-303."""
        if index + self.batch_size > self.epoch_amount:
            index = index + self.batch_size - self.epoch_amount
        bs, F = self.batch_size, self.FLAGS
        batch_pc = np.zeros((bs, self.num_points, 3), np.float32)
        batch_sdf_pt = np.zeros((bs, self.gen_num_pt, 3), np.float32)
        batch_sdf_pt_rot = np.zeros((bs, self.gen_num_pt, 3), np.float32)
        batch_sdf_val = np.zeros((bs, self.gen_num_pt, 1), np.float32)
        batch_norm_params = np.zeros((bs, 4), np.float32)
        batch_sdf_params = np.zeros((bs, 6), np.float32)
        batch_img = np.zeros((bs, F.img_h, F.img_w, 3), np.float32)
        batch_regress_mat = np.zeros((bs, 4, 3), np.float32)
        batch_trans_mat = np.zeros((bs, 4, 3), np.float32)
        batch_cat_id, batch_obj_nm, batch_view_id = [], [], []
        for cnt, i in enumerate(range(index, index + bs)):
            ori_pt, _, sample_pt, sample_sdf_val, norm_params, sdf_params, img_dir, cat_id, obj, num = \
                self.getitem(self.order[i])
            img, trans_mat, regress_mat = self.get_img(img_dir, num)
            cf_ref_choice = np.random.randint(ori_pt.shape[0], size=self.num_points)
            batch_pc[cnt, :, :] = ori_pt[cf_ref_choice, :]
            if self.gen_num_pt > sample_pt.shape[0]:
                choice = np.random.randint(sample_pt.shape[0], size=self.gen_num_pt)
            else:
                choice = np.asarray(random.sample(range(sample_pt.shape[0]), self.gen_num_pt), dtype=np.int32)
            batch_sdf_pt[cnt, ...] = sample_pt[choice, :]
            batch_sdf_val[cnt, :, 0] = sample_sdf_val[choice]
            batch_sdf_pt_rot[cnt, ...] = sample_pt[choice, :]
            batch_norm_params[cnt, ...] = norm_params
            batch_sdf_params[cnt, ...] = sdf_params
            batch_img[cnt, ...] = img
            batch_regress_mat[cnt, ...] = regress_mat
            batch_trans_mat[cnt, ...] = trans_mat
            batch_cat_id.append(cat_id)
            batch_obj_nm.append(obj)
            batch_view_id.append(num)
        return {"pc": batch_pc, "sdf_pt": batch_sdf_pt, "sdf_pt_rot": batch_sdf_pt_rot, "sdf_val": batch_sdf_val,
                "norm_params": batch_norm_params, "sdf_params": batch_sdf_params, "img": batch_img,
                "trans_mat": batch_trans_mat, "cat_id": batch_cat_id, "obj_nm": batch_obj_nm, "view_id": batch_view_id}

    def refill_data_order(self):
        """:305-318."""
        temp_order = copy.deepcopy(self.data_order)
        cats_quota = dict(self.cats_limit)
        np.random.shuffle(temp_order)
        pointer = 0
        epoch_order = []
        while len(epoch_order) < self.epoch_amount:
            cat_id, _, _ = self.listinfo[temp_order[pointer]]
            if cats_quota[cat_id] > 0:
                epoch_order.append(temp_order[pointer])
                cats_quota[cat_id] -= 1
            pointer += 1
        return epoch_order

    def work(self, epoch, index):
        if index == 0 and self.shuffle:
            self.order = self.refill_data_order()
            print("data order reordered!")
        return self.get_batch(index)

    def run(self):
        per_epoch = self.num_batches * self.batch_size
        while per_epoch and self.bno // per_epoch < self.FLAGS.max_epoch and not self.stopped:
            try:
                item = self.work(self.bno // per_epoch, self.bno % per_epoch)
            except Exception as e:      # handed to fetch, which raises it in the caller's thread
                item = e
                self.stopped = True
            while True:
                try:
                    self.queue.put(item, timeout=0.1)
                    break
                except queue.Full:
                    if self.stopped and not isinstance(item, Exception):
                        return
            self.bno += self.batch_size

    def fetch(self):
        if self.stopped and self.queue.empty():
            return None
        item = self.queue.get()
        if isinstance(item, Exception):
            raise item
        return item

    def shutdown(self):
        self.stopped = True
        while not self.queue.empty():
            self.queue.get()
        if self.is_alive():
            self.join()
