"""Python handle over the C-ABI context: one Engine = one CUDA device + one stream (not thread-safe)."""
from __future__ import annotations

import ctypes as C
import os
from typing import NamedTuple

import numpy as np

from . import _lib
from ._lib import DISN_DEVICE_PTR, PREC_BF16X3, PREC_F16F8, PREC_FP32, DisnConfig, check

_PREC = {"fp32": PREC_FP32, "bf16x3": PREC_BF16X3, "f16f8": PREC_F16F8}
TAP_HW = (224, 112, 56, 28, 14)
TAP_C = (64, 128, 256, 512, 512)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


class MeshCleanCounts(NamedTuple):
    """Result counts of Engine.clean_mesh: the cleaned mesh's size, the components found and the components kept."""
    n_verts: int
    n_faces: int
    n_components: int
    n_kept: int


def engine_config(device: int = 0, precision: str = "fp32", max_batch: int = 1, tanh: bool = False,
                  img_h: int = 137, img_w: int = 137, num_classes: int = 1024, sdf_weight: float = 10.0) -> DisnConfig:
    """The disn_config an Engine with these arguments is created with (no device needed)."""
    cfg = DisnConfig()
    _lib.load().disn_default_config(C.byref(cfg))
    cfg.device = device
    cfg.precision = _PREC[precision]
    cfg.max_batch = max_batch
    cfg.tanh_out = int(bool(tanh))
    cfg.img_h, cfg.img_w, cfg.num_classes = img_h, img_w, num_classes
    cfg.sdf_weight = sdf_weight
    # models/model_normalization.py:249-251 clamps projected points to the constant [0, 136] whatever FLAGS.img_h/img_w
    # are: on a smaller map the points beyond its edge get no features, on a larger one nothing is read beyond 136
    cfg.clamp_max = 136.0
    return cfg


class Engine:
    def __init__(self, device: int = 0, precision: str = "fp32", max_batch: int = 1, tanh: bool = False,
                 img_h: int = 137, img_w: int = 137, num_classes: int = 1024, sdf_weight: float = 10.0):
        self.lib = _lib.load()
        cfg = engine_config(device, precision, max_batch, tanh, img_h, img_w, num_classes, sdf_weight)
        self.cfg = cfg
        self._h = C.c_void_p()
        check(self.lib.disn_create(C.byref(cfg), C.byref(self._h)))
        self.batch = 0
        self.last_clean = None
        self.obj_fallbacks = 0      # files read_obj handed to the Python reader

    # -- lifetime -----------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self.lib.disn_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream: int | None):
        check(self.lib.disn_set_stream(self._h, C.c_void_p(cuda_stream or 0)))

    def synchronize(self):
        check(self.lib.disn_synchronize(self._h))

    def set_precision(self, precision: str):
        check(self.lib.disn_set_precision(self._h, _PREC[precision]))

    @property
    def launch_count(self) -> int:
        return int(self.lib.disn_launch_count(self._h))

    # -- weights ------------------------------------------------------------------------------
    def load_weights(self, weights: dict):
        """weights: TF variable name -> array (HWIO).  Unknown names are stored but unused."""
        for name, arr in weights.items():
            a = _f32(arr)
            shp = (C.c_int64 * a.ndim)(*a.shape)
            check(self.lib.disn_load_weight(self._h, name.encode(), a.ctypes.data_as(C.c_void_p), shp, a.ndim))
        check(self.lib.disn_finalize_weights(self._h))

    # -- decoder training ----------------------------------------------------------------------
    def train_begin(self, beta1: float = 0.5, beta2: float = 0.999, epsilon: float = 1e-8, wd: float = 1e-5,
                    mask_weight: float = 4.0, sdf_weight: float = 10.0):
        """Start training the decoder of the loaded weights with TF's Adam (disn_train_begin): zeroed slots,
        beta powers = betas.  The encoder stays frozen."""
        cfg = _lib.DisnTrainConfig(beta1, beta2, epsilon, wd, mask_weight, sdf_weight)
        check(self.lib.disn_train_begin(self._h, C.byref(cfg)))
        self._train_names = train_var_names()

    def train_step(self, imgs, pts, pts_rot, trans_mat, sdf_gt, lr: float) -> np.ndarray:
        """One training step (disn_train_step): imgs [B,H,W,3], pts / pts_rot [B,N,3], trans_mat [B,4,3], sdf_gt [B,N] =
        the fed ground truth (sdf_val - 0.003) -> float64 [5] in TRAIN_LOSS_KEYS order, from the forward pass before the
        update.  The encoded state is dropped: encode again before inference."""
        a, p, t, g = _f32(imgs), _f32(pts), _f32(trans_mat), _f32(sdf_gt)
        if a.ndim != 4 or p.ndim != 3 or p.shape[2] != 3:
            raise ValueError("imgs must be [B,H,W,C] and pts [B,N,3]")
        B, N, _ = p.shape
        pr = None if pts_rot is None else _f32(pts_rot)
        if a.shape[0] != B or t.size != B * 12 or g.size != B * N or (pr is not None and pr.shape != p.shape):
            raise ValueError("imgs, pts_rot, trans_mat and sdf_gt must match pts' batch and points")
        out = np.zeros(5, np.float64)
        ptr = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
        self.batch = 0
        check(self.lib.disn_train_step(self._h, ptr(a), a.shape[1], a.shape[2], a.shape[3], ptr(p), ptr(pr), ptr(t), ptr(g),
                                       B, N, float(lr), ptr(out)))
        return out

    def train_state(self) -> dict:
        """The training state by TF name: the 24 decoder variables, their `/Adam` and `/Adam_1` slots (TF shapes) and
        `beta1_power` / `beta2_power` (float32 scalars)."""
        st = {}
        for name in self._train_names:
            n = self._numel(name)
            for suffix in ("", "/Adam", "/Adam_1"):
                st[name + suffix] = self.train_get(name + suffix, n).reshape(train_var_shape(name, n))
        for name in ("beta1_power", "beta2_power"):
            st[name] = np.float32(self.train_get(name, 1)[0])
        return st

    def train_phase_ms(self) -> dict:
        """Device-event milliseconds of the last train_step's phases: encode, gather, forward, loss, backward, adam."""
        ms = (C.c_float * 6)()
        check(self.lib.disn_train_phase_ms(self._h, ms))
        return dict(zip(("encode", "gather", "forward", "loss", "backward", "adam"), list(ms)))

    def train_get(self, name: str, numel: int) -> np.ndarray:
        """A variable of the context by TF name, flat: a decoder variable or slot, a beta power, or a frozen encoder
        variable (read only) of numel elements."""
        out = np.empty(numel, np.float32)
        check(self.lib.disn_train_get(self._h, name.encode(), out.ctypes.data_as(C.c_void_p), numel))
        return out

    def _numel(self, name: str) -> int:
        scope, rest = name.split("/", 1)
        layer, kind = rest.rsplit("/", 1)
        cout = _TRAIN_COUT[layer]
        if kind == "biases":
            return cout
        cin = {"fold1/conv1": 3, "fold1/conv2": 64, "fold1/conv3": 256, "fold2/conv2": 512, "fold2/conv5": 256}.get(layer)
        if cin is None:
            cin = 512 + (self.cfg.num_classes if scope == "sdfprediction" else 1472)
        return cin * cout

    def load_train_state(self, state: dict):
        """Set whatever of train_state()'s names `state` holds (variables, slots, beta powers)."""
        for name, arr in state.items():
            a = _f32(arr).reshape(-1)
            check(self.lib.disn_train_set(self._h, name.encode(), a.ctypes.data_as(C.c_void_p), a.size))
        self.batch = 0

    # -- encoder ------------------------------------------------------------------------------
    def encode(self, imgs):
        a = _f32(imgs)
        if a.ndim != 4:
            raise ValueError("imgs must be [B,H,W,C]")
        B, H, W, Cc = a.shape
        check(self.lib.disn_encode(self._h, a.ctypes.data_as(C.c_void_p), B, H, W, Cc, 0))
        self.batch = B

    def encode_device(self, imgs_ptr: int, B: int, H: int, W: int, Cc: int = 3):
        """Device-pointer, asynchronous variant."""
        check(self.lib.disn_encode(self._h, C.c_void_p(imgs_ptr), B, H, W, Cc, DISN_DEVICE_PTR))
        self.batch = B

    def get_encoded(self, what: int) -> np.ndarray:
        B = self.batch
        cfg = self.cfg
        if what == 0:
            shape = (B, cfg.num_classes)
        elif 1 <= what <= 5:
            shape = (B, TAP_HW[what - 1], TAP_HW[what - 1], TAP_C[what - 1])
        elif what == 6:
            shape = (B, cfg.img_h, cfg.img_w, 512)
        elif what == 7:
            shape = (B, 512)
        elif what == 8:
            shape = (B, cfg.vgg_in, cfg.vgg_in, 3)
        else:
            raise ValueError(what)
        out = np.empty(shape, dtype=np.float32)
        check(self.lib.disn_get_encoded(self._h, what, out.ctypes.data_as(C.c_void_p), out.size))
        return out

    # -- points -------------------------------------------------------------------------------
    def eval_points(self, pts, trans_mat, pts_rot=None, want_uv: bool = False):
        """One `sess.run`: pts [B,N,3], trans_mat [B,4,3] -> pred_sdf [B,N,1] (and uv [B,N,2])."""
        p = _f32(pts)
        t = _f32(trans_mat)
        B, N, _ = p.shape
        pr = None if pts_rot is None else _f32(pts_rot)
        out = np.empty((B, N, 1), dtype=np.float32)
        uv = np.empty((B, N, 2), dtype=np.float32) if want_uv else None
        check(self.lib.disn_eval_points(
            self._h, p.ctypes.data_as(C.c_void_p), None if pr is None else pr.ctypes.data_as(C.c_void_p),
            t.ctypes.data_as(C.c_void_p), B, N, out.ctypes.data_as(C.c_void_p),
            None if uv is None else uv.ctypes.data_as(C.c_void_p), 0))
        return (out, uv) if want_uv else out

    def eval_points_ex(self, pts, trans_mat, pts_rot=None):
        """pred_sdf, sample_img_points, pred_sdf_value_global, pred_sdf_value_local (model_normalization.py:194-206)."""
        p, t = _f32(pts), _f32(trans_mat)
        B, N, _ = p.shape
        pr = None if pts_rot is None else _f32(pts_rot)
        out, g, l = (np.empty((B, N, 1), np.float32) for _ in range(3))
        uv = np.empty((B, N, 2), np.float32)
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        check(self.lib.disn_eval_points_ex(self._h, ptr(p), ptr(pr), ptr(t), B, N, ptr(out), ptr(uv), ptr(g), ptr(l)))
        return out, uv, g, l

    def point_img_feat(self, pts, trans_mat):
        """end_points['point_img_feat'] [B,N,1,1472] and sample_img_points [B,N,2] (model_normalization.py:170-190)."""
        p, t = _f32(pts), _f32(trans_mat)
        B, N, _ = p.shape
        feat = np.empty((B, N, 1, 1472), np.float32)
        uv = np.empty((B, N, 2), np.float32)
        check(self.lib.disn_point_img_feat(self._h, p.ctypes.data_as(C.c_void_p), t.ctypes.data_as(C.c_void_p), B, N,
                                           feat.ctypes.data_as(C.c_void_p), uv.ctypes.data_as(C.c_void_p)))
        return feat, uv

    def eval_features(self, pts_rot, global_feat, point_feat):
        """get_decoder (model_normalization.py:223-238): explicit [B,1,1,1024] / [B,N,1,1472] features ->
        (multi_pred_sdf, pred_sdf_value_global, pred_sdf_value_local), each [B,N,1]."""
        p = _f32(pts_rot)
        B, N, _ = p.shape
        g = _f32(global_feat).reshape(B, -1)
        f = _f32(point_feat).reshape(B, N, 1472)
        out, og, ol = (np.empty((B, N, 1), np.float32) for _ in range(3))
        ptr = lambda a: a.ctypes.data_as(C.c_void_p)
        check(self.lib.disn_eval_features(self._h, ptr(p), ptr(g), ptr(f), B, N, ptr(out), ptr(og), ptr(ol), 0))
        return out, og, ol

    def eval_points_device(self, pts_ptr: int, trans_mat_ptr: int, B: int, N: int, out_ptr: int,
                           uv_ptr: int = 0, pts_rot_ptr: int = 0):
        """Device-pointer, asynchronous variant (pointers from torch tensors' data_ptr())."""
        check(self.lib.disn_eval_points(self._h, C.c_void_p(pts_ptr), C.c_void_p(pts_rot_ptr or 0),
                                        C.c_void_p(trans_mat_ptr), B, N, C.c_void_p(out_ptr),
                                        C.c_void_p(uv_ptr or 0), DISN_DEVICE_PTR))

    def sdf_metrics(self, pts, trans_mat, sdf_val, iso_offset: float = 0.003, sdf_weight: float = 10.0,
                    mask_weight: float = 4.0, want_pred: bool = False):
        """Per-image metrics of test/test_sdf_acc.py at ground-truth samples (disn_sdf_metrics): pts [B,N,3], trans_mat
        [B,4,3], sdf_val [B,N] or [B,N,1] of the encoded batch -> (count int64 [B], wsum float64 [B], rsum float64 [B]),
        and pred_sdf [B,N,1] (bitwise eval_points's) with want_pred.  batch_losses turns them into the batch values."""
        p, t = _f32(pts), _f32(trans_mat)
        if p.ndim != 3 or p.shape[2] != 3:
            raise ValueError("pts must be [B,N,3]")
        B, N, _ = p.shape
        g = _f32(sdf_val)
        if g.size != B * N:
            raise ValueError("sdf_val must hold B*N values")
        cnt, ws, rs = np.empty(B, np.int64), np.empty(B, np.float64), np.empty(B, np.float64)
        pred = np.empty((B, N, 1), np.float32) if want_pred else None
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        check(self.lib.disn_sdf_metrics(self._h, ptr(p), ptr(t), ptr(g), B, N, float(iso_offset), float(sdf_weight),
                                        float(mask_weight), 0, ptr(pred), ptr(cnt), ptr(ws), ptr(rs)))
        return (cnt, ws, rs, pred) if want_pred else (cnt, ws, rs)

    def sdf_metrics_device(self, pts_ptr: int, trans_mat_ptr: int, sdf_val_ptr: int, B: int, N: int, count_ptr: int,
                           wsum_ptr: int, rsum_ptr: int, pred_ptr: int = 0, iso_offset: float = 0.003,
                           sdf_weight: float = 10.0, mask_weight: float = 4.0):
        """Device-pointer, asynchronous variant: int64 counts and float64 sums [B] at the given device addresses."""
        check(self.lib.disn_sdf_metrics(self._h, C.c_void_p(pts_ptr), C.c_void_p(trans_mat_ptr), C.c_void_p(sdf_val_ptr),
                                        B, N, float(iso_offset), float(sdf_weight), float(mask_weight), DISN_DEVICE_PTR,
                                        C.c_void_p(pred_ptr or 0), C.c_void_p(count_ptr), C.c_void_p(wsum_ptr),
                                        C.c_void_p(rsum_ptr)))

    def eval_grid(self, sdf_params, trans_mat, sdf_res: int, z0: int = 0, z1: int | None = None, out=None):
        """Dense grid slab -> [B, z1-z0, R, R] float32 = pred/sdf_weight (reference `result`, reshaped)."""
        sp = np.ascontiguousarray(sdf_params, dtype=np.float64).reshape(-1, 6)
        t = _f32(trans_mat)
        B = sp.shape[0]
        R = sdf_res + 1
        z1 = R if z1 is None else z1
        if out is None:
            out = np.empty((B, z1 - z0, R, R), dtype=np.float32)
        assert out.dtype == np.float32 and out.flags.c_contiguous and out.size == B * (z1 - z0) * R * R
        check(self.lib.disn_eval_grid(self._h, sp.ctypes.data_as(C.POINTER(C.c_double)),
                                      t.ctypes.data_as(C.c_void_p), B, sdf_res, z0, z1,
                                      out.ctypes.data_as(C.c_void_p), 0))
        return out

    def eval_grid_device(self, sdf_params, trans_mat_ptr: int, sdf_res: int, z0: int, z1: int, out_ptr: int):
        sp = np.ascontiguousarray(sdf_params, dtype=np.float64).reshape(-1, 6)
        check(self.lib.disn_eval_grid(self._h, sp.ctypes.data_as(C.POINTER(C.c_double)), C.c_void_p(trans_mat_ptr),
                                      sp.shape[0], sdf_res, z0, z1, C.c_void_p(out_ptr), DISN_DEVICE_PTR))

    # -- estimated camera ------------------------------------------------------------------------
    def cam_estimate(self, imgs, K=None, want_rt: bool = False):
        """demo/demo.py:195-258 cam_evl: imgs [B,H,W,3] -> pred_trans_mat [B,4,3] (this engine must hold the camera
        checkpoint's variables: vgg_16/* and cameraprediction/*).  load_weights_raw() skips the SDF-head checks."""
        a = _f32(imgs)
        B, H, W, Cc = a.shape
        tm = np.empty((B, 4, 3), np.float32)
        rt = np.empty((B, 4, 3), np.float32) if want_rt else None
        kk = None if K is None else _f32(K).reshape(9)
        check(self.lib.disn_cam_estimate(self._h, a.ctypes.data_as(C.c_void_p), B, H, W, Cc,
                                         None if kk is None else kk.ctypes.data_as(C.c_void_p),
                                         None if rt is None else rt.ctypes.data_as(C.c_void_p),
                                         tm.ctypes.data_as(C.c_void_p)))
        return (tm, rt) if want_rt else tm

    def cam_metrics(self, imgs, pts, trans_mat, RT, K=None):
        """The camera checkpoint score of cam_est/train_sdf_cam.py --test (disn_cam_metrics): imgs [B,H,W,3], pts
        [B,N,3], ground-truth trans_mat and RT (the view file's regress_mat) [B,4,3] -> (pred_trans_mat [B,4,3], pred_RT
        [B,4,3], sums float64 [B,5]).  The predictions are cam_estimate's bits; cam_losses turns the sums into the batch
        values."""
        a, p, t, r = _f32(imgs), _f32(pts), _f32(trans_mat), _f32(RT)
        if a.ndim != 4 or p.ndim != 3 or p.shape[2] != 3:
            raise ValueError("imgs must be [B,H,W,C] and pts [B,N,3]")
        B, H, W, Cc = a.shape
        if p.shape[0] != B or t.size != B * 12 or r.size != B * 12:
            raise ValueError("pts, trans_mat and RT must hold one entry per image")
        tm, rt, sums = np.empty((B, 4, 3), np.float32), np.empty((B, 4, 3), np.float32), np.empty((B, 5), np.float64)
        kk = None if K is None else _f32(K).reshape(9)
        ptr = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
        check(self.lib.disn_cam_metrics(self._h, ptr(a), B, H, W, Cc, ptr(kk), ptr(p), p.shape[1], ptr(t), ptr(r), ptr(rt),
                                        ptr(tm), ptr(sums)))
        return tm, rt, sums

    def load_weights_raw(self, weights: dict):
        """Upload variables without finalising the SDF heads (camera-net contexts have no sdfprediction/*)."""
        for name, arr in weights.items():
            a = _f32(arr)
            shp = (C.c_int64 * a.ndim)(*a.shape)
            check(self.lib.disn_load_weight(self._h, name.encode(), a.ctypes.data_as(C.c_void_p), shp, a.ndim))

    # -- mesh metrics -------------------------------------------------------------------------
    def nn_distance(self, xyz1, xyz2):
        """The reference's tf_nndistance.nn_distance(xyz1, xyz2): squared NN distances + indices, both ways."""
        a, b = _f32(xyz1), _f32(xyz2)
        B, N, _ = a.shape
        M = b.shape[1]
        d1, i1 = np.empty((B, N), np.float32), np.empty((B, N), np.int32)
        d2, i2 = np.empty((B, M), np.float32), np.empty((B, M), np.int32)
        check(self.lib.disn_nn_distance(self._h, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), B, N, M,
                                        d1.ctypes.data_as(C.c_void_p), i1.ctypes.data_as(C.c_void_p),
                                        d2.ctypes.data_as(C.c_void_p), i2.ctypes.data_as(C.c_void_p)))
        return d1, i1, d2, i2

    def chamfer_x1000(self, pred, src):
        """test/test_cd_emd.py:300-301: (mean forward + mean backward squared NN distance) * 1000, per batch item."""
        df, _, db, _ = self.nn_distance(pred, src)
        return (df.mean(axis=1) + db.mean(axis=1)) * np.float32(1000)

    def approx_match(self, xyz1, xyz2, cost=False):
        """The reference's tf_approxmatch.approx_match(xyz1, xyz2) (models/tf_ops/approxmatch/tf_approxmatch.py:12-20):
        match [B,N,M] float32, element (k,l) = mass moved from point k of xyz1 to point l of xyz2.  cost=True also returns
        match_cost(xyz1, xyz2, match) [B] from the same call."""
        a, b = _f32(xyz1), _f32(xyz2)
        B, N, _ = a.shape
        M = b.shape[1]
        m = np.empty((B, N, M), np.float32)
        cst = np.empty(B, np.float32) if cost else None
        check(self.lib.disn_approx_match(self._h, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), B, N, M,
                                         m.ctypes.data_as(C.c_void_p), cst.ctypes.data_as(C.c_void_p) if cost else None))
        return (m, cst) if cost else m

    def match_cost(self, xyz1, xyz2, match):
        """tf_approxmatch.match_cost(xyz1, xyz2, match) (tf_approxmatch.py:28-37): cost [B]."""
        a, b, m = _f32(xyz1), _f32(xyz2), _f32(match)
        B, N, _ = a.shape
        M = b.shape[1]
        assert m.shape == (B, N, M), m.shape
        cst = np.empty(B, np.float32)
        check(self.lib.disn_match_cost(self._h, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p),
                                       m.ctypes.data_as(C.c_void_p), B, N, M, cst.ctypes.data_as(C.c_void_p)))
        return cst

    def emd(self, src, pred):
        """test/test_cd_emd.py:307-308: match_cost(src, pred, approx_match(src, pred)) * 0.01 per batch item; the match
        matrix stays in HBM."""
        a, b = _f32(src), _f32(pred)
        B, N, _ = a.shape
        cst = np.empty(B, np.float32)
        check(self.lib.disn_approx_match(self._h, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), B, N, b.shape[1],
                                         None, cst.ctypes.data_as(C.c_void_p)))
        return cst * np.float32(0.01)

    def points_loss(self, sampled_pc):
        """get_points_loss of test/test_cd_emd.py:291-315: sampled_pc [1+V,N,3] = the ground-truth cloud followed by the
        clouds of V predicted views.  Returns (avg_cf, min_cf, arg_min_cf, avg_em, min_em, arg_min_em) over the views:
        Chamfer x1000 and approximate EMD x0.01 of every view against the ground truth."""
        pc = _f32(sampled_pc)
        pred = pc[1:]
        src = np.ascontiguousarray(np.broadcast_to(pc[:1], pred.shape))
        cf = self.chamfer_x1000(pred, src)
        em = self.emd(src, pred)
        return (np.float32(cf.mean()), np.float32(cf.min()), int(cf.argmin()),
                np.float32(em.mean()), np.float32(em.min()), int(em.argmin()))

    def f_score(self, pred, src, thresholds):
        """test/test_f_score.py:231-236: precision / recall = fraction of sqrt NN distances (pred->src / src->pred)
        below each threshold; F = 2PR/(P+R).  pred, src: [1,N,3] / [1,M,3].  Distances come from the CUDA NN kernel."""
        df, _, db, _ = self.nn_distance(pred, src)
        th = np.asarray(thresholds, np.float32)[:, None]
        p = (np.sqrt(df).reshape(1, -1) < th).mean(axis=1)
        r = (np.sqrt(db).reshape(1, -1) < th).mean(axis=1)
        return p, r, 2 * p * r / np.maximum(p + r, 1e-30)

    # -- marching cubes -----------------------------------------------------------------------
    def marching_cubes(self, sdf, bbox, iso: float = 0.0, device_ptr: int | None = None, R: int | None = None,
                       fetch: bool = True):
        """sdf [R,R,R] (z,y,x) host array, or a device pointer -> (verts [V,3] float32, faces [F,3] int32 0-based).
        The welded mesh also stays in HBM as the resident mesh (write_mesh_obj, clean_mesh); fetch=False returns only
        the counts.  A failed call leaves the resident mesh empty."""
        bb = (C.c_double * 6)(*[float(v) for v in bbox])
        if device_ptr is None:
            a = _f32(sdf)
            R = a.shape[0]
            assert a.shape == (R, R, R)
            ptr, flags = a.ctypes.data_as(C.c_void_p), 0
        else:
            ptr, flags = C.c_void_p(device_ptr), DISN_DEVICE_PTR
        nv, nf = C.c_int64(0), C.c_int64(0)
        check(self.lib.disn_mc_run(self._h, ptr, R, bb, float(iso), flags, C.byref(nv), C.byref(nf)))
        if not fetch:
            return nv.value, nf.value
        return self._fetch(nv.value, nf.value)

    def write_mesh_obj(self, path: str):
        """OBJ of the resident mesh, as the last marching_cubes / load_mesh / clean_mesh call left it (reference mesher's
        output conventions)."""
        check(self.lib.disn_mc_write_obj(self._h, path.encode()))

    def load_mesh(self, verts, faces):
        """Upload a mesh (verts [V,3] float32, faces [F,3] 0-based) into the resident slot marching_cubes fills.  A face
        index outside [0, V) is refused and leaves the resident mesh as it was."""
        v = _f32(verts).reshape(-1, 3)
        f = np.ascontiguousarray(faces, np.int32).reshape(-1, 3)
        check(self.lib.disn_mesh_load(self._h, v.ctypes.data_as(C.c_void_p), len(v), f.ctypes.data_as(C.c_void_p), len(f)))

    def read_obj(self, path, parts: bool = False, load: bool = False):
        """create_sdf.read_obj(path), or read_obj_parts(path) with parts=True, parsed on the device (disn_obj_read): the
        same arrays bit for bit, and the same names.  The mesh stays resident, as after load_mesh.  A file outside the
        device reader's grammar (or one it finds invalid, or cannot open) is read by the Python reader instead, which
        raises what it raises; `obj_fallbacks` counts those files, and load=True then uploads what it returned (the
        resident mesh is empty otherwise)."""
        nv, nf, npart = C.c_int64(0), C.c_int64(0), C.c_int32(0)
        rc = self.lib.disn_obj_read(self._h, os.fsencode(path), _lib.DISN_OBJ_PARTS if parts else 0, C.byref(nv),
                                    C.byref(nf), C.byref(npart))
        if rc == _lib.DISN_ERR_OBJ_UNSUPPORTED:
            from .create_sdf import read_obj, read_obj_parts
            self.obj_fallbacks += 1
            mesh = read_obj_parts(path) if parts else read_obj(path)
            if load:
                self.load_mesh(mesh[0], mesh[1])
            return mesh
        check(rc)
        counts = np.zeros(2, np.int64)
        check(self.lib.disn_obj_read_stats(self._h, counts.ctypes.data_as(C.c_void_p), None))
        if counts[1]:       # a finite coordinate overflowed float32: numpy's own warning, as the cast in read_obj gives
            np.array([np.finfo(np.float64).max]).astype(np.float32)
        verts, faces = self._fetch(nv.value, nf.value)
        if not parts:
            return verts, faces
        pid = np.empty(nf.value, np.int32)
        off = np.empty(npart.value + 1, np.int64)
        check(self.lib.disn_obj_parts(self._h, pid.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), None, 0))
        buf = C.create_string_buffer(max(int(off[-1]), 1))
        check(self.lib.disn_obj_parts(self._h, None, None, buf, len(buf)))
        names, end = [], int(off[-1])
        for s in off[-2::-1]:           # a part's name ends where the next named part's begins (None has no bytes)
            names.append(None if s < 0 else buf.raw[s:end].decode("ascii"))
            end = end if s < 0 else int(s)
        return verts, faces, pid, names[::-1]

    def obj_read_stats(self):
        """The last successful disn_obj_read: coordinates converted on the host, coordinates that overflowed float32, and
        the milliseconds of its phases (device events: upload, lines, classify, parse; host clock: host)."""
        counts = np.zeros(2, np.int64)
        ms = (C.c_float * 5)()
        check(self.lib.disn_obj_read_stats(self._h, counts.ctypes.data_as(C.c_void_p), ms))
        return {"host_tokens": int(counts[0]), "overflows": int(counts[1]),
                "phase_ms": dict(zip(("upload", "lines", "classify", "parse", "host"), list(ms)))}

    def mesh_counts(self):
        """(n_verts, n_faces) of the resident mesh, read from the library's host-side state (no device work)."""
        nv, nf = C.c_int64(0), C.c_int64(0)
        check(self.lib.disn_mesh_counts(self._h, C.byref(nv), C.byref(nf)))
        return nv.value, nf.value

    def fetch_mesh(self):
        """The resident mesh (last marching_cubes / load_mesh / read_obj / mesh_grid_adaptive / clean_mesh /
        normalize_mesh, or a C-ABI call that wrote it) -> (verts, faces), sized by mesh_counts()."""
        return self._fetch(*self.mesh_counts())

    def _fetch(self, nv: int, nf: int):
        """The resident mesh, whose counts are nv / nf -> (verts [nv,3] float32, faces [nf,3] int32)."""
        verts = np.empty((nv, 3), dtype=np.float32)
        faces = np.empty((nf, 3), dtype=np.int32)
        if nv or nf:        # the library copies each array only when the resident mesh has entries
            check(self.lib.disn_mc_fetch(self._h, verts.ctypes.data_as(C.c_void_p), faces.ctypes.data_as(C.c_void_p)))
        return verts, faces

    def clean_mesh(self, dist_thresh: float = 0.5, num_thresh: float = 0.3, fetch: bool = True, want_labels: bool = False):
        """postprocessing/clean_smallparts.py:38-54 on the resident mesh, in place: drop every edge-connected component
        with n_c <= max n_c * num_thresh vertices or a centroid at distance >= dist_thresh from the origin.
        -> (verts, faces), plus the per-face component labels of the input mesh (sized by mesh_counts()) if
        want_labels; fetch=False returns the MeshCleanCounts instead of the mesh (and the labels).  The counts of the
        last call are in `last_clean`."""
        labels = np.empty(self.mesh_counts()[1], np.int32) if want_labels else None
        nc, nk, nv, nf = (C.c_int64(0) for _ in range(4))
        check(self.lib.disn_mesh_clean(self._h, float(dist_thresh), float(num_thresh),
                                       None if labels is None else labels.ctypes.data_as(C.c_void_p),
                                       C.byref(nc), C.byref(nk), C.byref(nv), C.byref(nf)))
        self.last_clean = MeshCleanCounts(nv.value, nf.value, nc.value, nk.value)
        if not fetch:
            return (self.last_clean, labels) if want_labels else self.last_clean
        verts, faces = self._fetch(nv.value, nf.value)
        return (verts, faces, labels) if want_labels else (verts, faces)

    def mesh_sdf(self, res: int, bbox=None, expand_rate: float = 1.2, sigma: float = 0.0, verts=None, faces=None,
                 device_ptr: int | None = None):
        """Signed distance field of the resident mesh (preprocessing/create_point_sdf_grid.py:200-210,
        computeDistanceField -s): (res+1)^3 grid over bbox (None = cube around the mesh AABB scaled by expand_rate),
        sign by exterior flood fill with wall threshold sigma (the reference's -g).  verts/faces, if given, are loaded
        first.  -> (grid [R,R,R] float32 (z,y,x), or None when written to device_ptr, bbox as a list of 6 floats)."""
        if verts is not None or faces is not None:
            self.load_mesh(verts, faces)
        R = res + 1
        bb = None if bbox is None else (C.c_double * 6)(*[float(v) for v in bbox])
        used = (C.c_double * 6)()
        if device_ptr is None:
            ok = res >= 1 and R ** 3 < 2 ** 31       # otherwise the library reports the bad resolution
            out = np.empty((R, R, R) if ok else (1,), np.float32)
            ptr, flags = out.ctypes.data_as(C.c_void_p), 0
        else:
            out, ptr, flags = None, C.c_void_p(device_ptr), DISN_DEVICE_PTR
        check(self.lib.disn_mesh_sdf(self._h, res, bb, float(expand_rate), float(sigma), ptr, used, flags))
        return out, list(used)

    def mesh_sdf_phase_ms(self):
        """Milliseconds of the last mesh_sdf's phases: BVH build, distance, edge rasterisation, flood fill and sign."""
        ms = (C.c_float * 4)()
        check(self.lib.disn_mesh_sdf_phase_ms(self._h, ms))
        return dict(zip(("build", "distance", "rasterise", "flood"), list(ms)))

    # -- per-object preprocessing: normalisation and field samples ------------------------------------------------
    def part_areas(self, part_ids=None, n_parts: int = 1):
        """Quantised part areas of the resident mesh (DESIGN.md §4.8): part_ids [n_faces] in [0, n_parts) or None (one
        part) -> (Q_p int64 [n_parts], shift s); Q_p is the exact sum of rint(area_f * 2^s) over the part's faces."""
        pid = None if part_ids is None else np.ascontiguousarray(part_ids, np.int32)
        q = np.empty(n_parts, np.int64)
        s = C.c_int32(0)
        check(self.lib.disn_mesh_part_areas(self._h, None if pid is None else pid.ctypes.data_as(C.c_void_p), n_parts,
                                            q.ctypes.data_as(C.c_void_p), C.byref(s)))
        return q, s.value

    def normalize_mesh(self, part_ids=None, n_parts: int = 1, amounts=None, draws=None, given=None,
                       want_samples: bool = False):
        """preprocessing/create_point_sdf_grid.py:169-198 get_normalize_mesh on the resident mesh: amounts [n_parts] and
        draws [N,3] = (face pick, r1, r2) in sample_surface's np.random order -> (centroid float64 [3], m) and, with
        want_samples, the surface samples [N,3] float64.  The resident vertices become float32((v - c) / m).
        given = (cx, cy, cz, m) skips the sampling and only transforms the vertices."""
        c, m = np.empty(3, np.float64), C.c_double(0.0)
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        if given is not None:
            g = np.ascontiguousarray(np.asarray(given, np.float64).reshape(4))
            check(self.lib.disn_mesh_normalize(self._h, None, 1, None, None, 0, ptr(g), ptr(c), C.byref(m), None))
            return c, m.value
        pid = None if part_ids is None else np.ascontiguousarray(part_ids, np.int32)
        amt = np.ascontiguousarray(amounts, np.int64).reshape(-1)
        dr = np.ascontiguousarray(draws, np.float64).reshape(-1, 3)
        smp = np.empty((len(dr), 3), np.float64) if want_samples else None
        check(self.lib.disn_mesh_normalize(self._h, ptr(pid), n_parts, ptr(amt), ptr(dr), len(dr), None, ptr(c),
                                           C.byref(m), ptr(smp)))
        return (c, m.value, smp) if want_samples else (c, m.value)

    def field_buffer(self, R: int) -> int:
        """Device address of the context's resident [R,R,R] field (grows only; valid until a larger request)."""
        out = C.c_void_p()
        check(self.lib.disn_field(self._h, R, C.byref(out)))
        return int(out.value)

    def band_samples(self, num_sample: int, bandwidth: float, iso_val: float, params, sdf_res: int, sdf=None,
                     device_ptr: int | None = None):
        """preprocessing/create_point_sdf_grid.py:74-113 sample_sdf on the device, bit for bit the host function for the
        same np.random state: the four bands of float32(sdf - iso) are compacted in HBM, the host applies the carry-over
        rule and draws np.random.randint exactly as the host function does, the device gathers the [n,4] rows.
        params: the float32 box of get_sdf; sdf: host [R,R,R] float32, or device_ptr (e.g. field_buffer).
        iso_val and bandwidth are taken as Python floats, as the reference passes them: numpy 2 then subtracts and
        compares in float32 (NEP 50), which is what the device does.  A float64 numpy scalar would make the host
        function compute in float64 instead, so both are converted with float() here and in the package's callers."""
        R = sdf_res + 1
        bw = float(bandwidth)
        iso_val = float(iso_val)
        percentages = [[-1. * bw, -1. * bw * 0.30, int(num_sample * 0.25)],
                       [-1. * bw * 0.30, 0, int(num_sample * 0.25)],
                       [0, bw * 0.30, int(num_sample * 0.25)],
                       [bw * 0.30, bw, int(num_sample * 0.25)]]
        edges = np.array([[p[0], p[1]] for p in percentages], np.float64).astype(np.float32)
        if device_ptr is None:
            a = _f32(sdf)
            assert a.size == R ** 3
            src, flags = a.ctypes.data_as(C.c_void_p), 0
        else:
            src, flags = C.c_void_p(device_ptr), DISN_DEVICE_PTR
        counts = np.zeros(4, np.int64)
        check(self.lib.disn_sdf_band_count(self._h, src, R, float(np.float32(iso_val)), edges.ctypes.data_as(C.c_void_p),
                                           flags, counts.ctypes.data_as(C.c_void_p)))
        k = np.zeros(4, np.int64)
        choices = []
        for i in range(4):
            n = int(counts[i])
            if n < percentages[i][2]:
                if i < 3:
                    percentages[i + 1][2] += percentages[i][2] - n
                percentages[i][2] = n
            if n == 0:
                continue
            choices.append(np.random.randint(n, size=percentages[i][2]).astype(np.int64))
            k[i] = percentages[i][2]
        ch = np.ascontiguousarray(np.concatenate(choices) if choices else np.zeros(0, np.int64))
        p = np.asarray(params, np.float32)
        axes = np.ascontiguousarray(np.concatenate(
            [np.linspace(p[a], p[3 + a], num=R).astype(np.float32) for a in range(3)]))
        out = np.empty((len(ch), 4), np.float32)
        check(self.lib.disn_sdf_band_gather(self._h, axes.ctypes.data_as(C.c_void_p), ch.ctypes.data_as(C.c_void_p),
                                            k.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
        self.last_band_counts = counts
        return out

    def sdf_strided(self, R: int, reduce: int, sdf=None, device_ptr: int | None = None):
        """create_point_sdf_fullgrid.py:70-96: every reduce-th value of the [R,R,R] field on each axis -> [M,M,M],
        M = (R-1)//reduce + 1."""
        M = (R - 1) // reduce + 1 if reduce >= 1 else 1
        out = np.empty((M, M, M), np.float32)
        if device_ptr is None:
            a = _f32(sdf)
            assert a.size == R ** 3
            src, flags = a.ctypes.data_as(C.c_void_p), 0
        else:
            src, flags = C.c_void_p(device_ptr), DISN_DEVICE_PTR
        check(self.lib.disn_sdf_strided(self._h, src, R, reduce, flags, out.ctypes.data_as(C.c_void_p)))
        return out

    def eval_grid_resident(self, sdf_params, trans_mat, sdf_res: int) -> int:
        """Whole [B,R,R,R] grid evaluated into the context's HBM buffer; returns its device address."""
        sp = np.ascontiguousarray(sdf_params, dtype=np.float64).reshape(-1, 6)
        t = _f32(trans_mat)
        out = C.c_void_p()
        check(self.lib.disn_eval_grid_resident(self._h, sp.ctypes.data_as(C.POINTER(C.c_double)),
                                               t.ctypes.data_as(C.c_void_p), sp.shape[0], sdf_res, C.byref(out)))
        return int(out.value)

    def eval_grid_indexed(self, sdf_params, trans_mat, sdf_res: int, idx, image: int = 0):
        """Grid points idx (linear (z*R + y)*R + x, any order) of encoded image `image` -> float32 [n], bitwise the
        values eval_grid gives at those points.  sdf_params [6] and trans_mat [4,3] belong to that image."""
        sp = np.ascontiguousarray(sdf_params, dtype=np.float64).reshape(6)
        t = _f32(trans_mat).reshape(4, 3)
        ix = np.ascontiguousarray(idx, dtype=np.int64).reshape(-1)
        if ix.size and (ix.min() < 0 or ix.max() >= 2 ** 31):
            raise ValueError("grid indices must lie in [0, 2^31)")
        ix = ix.astype(np.int32)
        out = np.empty(ix.size, np.float32)
        check(self.lib.disn_eval_grid_indexed(self._h, sp.ctypes.data_as(C.POINTER(C.c_double)), t.ctypes.data_as(C.c_void_p),
                                              image, sdf_res, ix.ctypes.data_as(C.c_void_p), ix.size,
                                              out.ctypes.data_as(C.c_void_p), 0))
        return out

    def eval_grid_indexed_device(self, sdf_params, trans_mat_ptr: int, sdf_res: int, idx_ptr: int, n: int, out_ptr: int,
                                 image: int = 0):
        """Device-pointer, asynchronous variant: int32 indices at idx_ptr, float32 results at out_ptr."""
        sp = np.ascontiguousarray(sdf_params, dtype=np.float64).reshape(6)
        check(self.lib.disn_eval_grid_indexed(self._h, sp.ctypes.data_as(C.POINTER(C.c_double)), C.c_void_p(trans_mat_ptr),
                                              image, sdf_res, C.c_void_p(idx_ptr), n, C.c_void_p(out_ptr), DISN_DEVICE_PTR))

    def eval_grid_adaptive(self, sdf_params, trans_mat, sdf_res: int, iso: float = 0.0, band: float = 1.0, image: int = 0):
        """Coarse-to-fine [R,R,R] grid of encoded image `image` (DESIGN.md §4.9), left in the context's HBM buffer ->
        (device address, points evaluated by the coarse lattice and by each level).  The network runs only in blocks that
        straddle iso or lie within band * (s/2) * |h| of it; the other points are interpolated.  band = inf is the dense
        grid."""
        sp = np.ascontiguousarray(sdf_params, dtype=np.float64).reshape(6)
        t = _f32(trans_mat).reshape(4, 3)
        out = C.c_void_p()
        counts = np.zeros(5, np.int64)
        nl = C.c_int32(0)
        check(self.lib.disn_eval_grid_adaptive(self._h, sp.ctypes.data_as(C.POINTER(C.c_double)), t.ctypes.data_as(C.c_void_p),
                                               image, sdf_res, float(iso), float(band), C.byref(out),
                                               counts.ctypes.data_as(C.c_void_p), C.byref(nl)))
        return int(out.value), [int(v) for v in counts[:nl.value]]

    def mesh_grid_adaptive(self, sdf_params, trans_mat, sdf_res: int, iso: float = 0.0, band: float = 1.0, image: int = 0,
                           fetch: bool = True):
        """Coarse-to-fine mesh of encoded image `image` without a dense grid (DESIGN.md §4.10): bit for bit the mesh
        marching_cubes makes of eval_grid_adaptive's grid, with memory proportional to the evaluated points; sdf_res up to
        2048.  The mesh stays resident (clean_mesh, write_mesh_obj) -> (verts, faces, level_counts), or with fetch=False
        ((n_verts, n_faces), level_counts).  A call that fails after its arguments are accepted leaves the resident mesh
        empty."""
        sp = np.ascontiguousarray(sdf_params, dtype=np.float64).reshape(6)
        t = _f32(trans_mat).reshape(4, 3)
        counts = np.zeros(5, np.int64)
        nl = C.c_int32(0)
        nv, nf = C.c_int64(0), C.c_int64(0)
        check(self.lib.disn_mesh_grid_adaptive(self._h, sp.ctypes.data_as(C.POINTER(C.c_double)),
                                               t.ctypes.data_as(C.c_void_p), image, sdf_res, float(iso), float(band),
                                               counts.ctypes.data_as(C.c_void_p), C.byref(nl), C.byref(nv), C.byref(nf)))
        levels = [int(v) for v in counts[:nl.value]]
        if not fetch:
            return (nv.value, nf.value), levels
        verts, faces = self._fetch(nv.value, nf.value)
        return verts, faces, levels

    def fetch(self, dev_ptr: int, shape, dtype=np.float32) -> np.ndarray:
        out = np.empty(shape, dtype=dtype)
        check(self.lib.disn_fetch(self._h, C.c_void_p(dev_ptr), out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    # -- cross-process device buffer (peer-store gather) --------------------------------------------
    def shared_alloc(self, nbytes: int):
        """-> (device pointer, 64-byte IPC handle): rank 0's whole-grid buffer the other ranks' kernels store into."""
        ptr = C.c_void_p()
        handle = C.create_string_buffer(64)
        check(self.lib.disn_shared_alloc(self._h, nbytes, C.byref(ptr), handle))
        return int(ptr.value), handle.raw

    def shared_open(self, handle: bytes) -> int:
        ptr = C.c_void_p()
        check(self.lib.disn_shared_open(self._h, C.create_string_buffer(handle, 64), C.byref(ptr)))
        return int(ptr.value)

    def shared_close(self, ptr: int, owner: bool):
        check(self.lib.disn_shared_close(self._h, C.c_void_p(ptr), int(owner)))

    def iou(self, verts1, faces1, verts2, faces2, dim: int = 110, want_grids: bool = False):
        """test/test_iou.py:208-233 iou_pymesh on two triangle meshes -> IoU (and the two occupancy grids)."""
        v1, v2 = _f32(verts1), _f32(verts2)
        f1, f2 = np.ascontiguousarray(faces1, np.int32), np.ascontiguousarray(faces2, np.int32)
        inter, uni = C.c_int64(0), C.c_int64(0)
        o1 = np.empty((dim, dim, dim), np.uint8) if want_grids else None
        o2 = np.empty((dim, dim, dim), np.uint8) if want_grids else None
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        check(self.lib.disn_iou(self._h, ptr(v1), len(v1), ptr(f1), len(f1), ptr(v2), len(v2), ptr(f2), len(f2), dim,
                                C.byref(inter), C.byref(uni), ptr(o1), ptr(o2)))
        val = inter.value / uni.value if uni.value else float("nan")
        return (val, inter.value, uni.value, o1, o2) if want_grids else val

    def iou_views(self, ref_verts, ref_faces, views, dim: int = 110, want_grids: bool = False):
        """iou_pymesh (test/test_iou.py:208-233) of one reference mesh against every mesh of `views`, a list of
        (verts, faces), in one call (disn_iou_views): the reference is voxelised once.  Returns (iou [V] float64,
        intersection [V] int64, union [V] int64), plus the occupancy grids [V+1,dim,dim,dim] uint8 (the reference's
        first) when want_grids.  iou[v] is intersection / union, NaN when the union is empty."""
        rv, rf = _f32(ref_verts), np.ascontiguousarray(ref_faces, np.int32)
        V = len(views)
        vs = [_f32(v).reshape(-1, 3) for v, _ in views]
        fs = [np.ascontiguousarray(f, np.int32).reshape(-1, 3) for _, f in views]
        voff = np.zeros(V + 1, np.int64)
        foff = np.zeros(V + 1, np.int64)
        voff[1:] = np.cumsum([len(v) for v in vs])
        foff[1:] = np.cumsum([len(f) for f in fs])
        verts = np.ascontiguousarray(np.concatenate(vs) if V else np.zeros((0, 3), np.float32), np.float32)
        faces = np.ascontiguousarray(np.concatenate(fs) if V else np.zeros((0, 3), np.int32), np.int32)
        inter, uni = np.zeros(max(V, 1), np.int64), np.zeros(max(V, 1), np.int64)
        grids = np.empty((V + 1, dim, dim, dim), np.uint8) if want_grids else None
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        check(self.lib.disn_iou_views(self._h, ptr(rv), len(rv), ptr(rf), len(rf), V, ptr(verts), ptr(voff), ptr(faces),
                                      ptr(foff), dim, ptr(inter), ptr(uni), ptr(grids)))
        inter, uni = inter[:V], uni[:V]
        with np.errstate(invalid="ignore", divide="ignore"):
            val = np.where(uni > 0, inter / np.maximum(uni, 1), np.nan)
        return (val, inter, uni, grids) if want_grids else (val, inter, uni)


TRAIN_LOSS_KEYS = ("accuracy", "sdf_loss_realvalue", "sdf_loss", "regularization", "overall_loss")
_TRAIN_COUT = {"fold1/conv1": 64, "fold1/conv2": 256, "fold1/conv3": 512, "fold2/conv1": 512, "fold2/conv2": 256,
               "fold2/conv5": 1}


def train_var_names():
    """The 24 decoder variables training updates, in the library's order (disn_train_var_name)."""
    lib = _lib.load()
    out = []
    for i in range(24):
        buf = C.create_string_buffer(128)
        check(lib.disn_train_var_name(i, buf, len(buf)))
        out.append(buf.value.decode())
    return out


def train_var_shape(name: str, numel: int):
    """TF's shape of a decoder variable (or of its Adam slots) with numel elements: [1,1,Cin,Cout] kernels, [Cout] biases."""
    base = name.split("/Adam")[0]
    cout = _TRAIN_COUT[base.split("/", 1)[1].rsplit("/", 1)[0]]
    return (cout,) if base.endswith("/biases") else (1, 1, numel // cout, cout)


def batch_losses(count, wsum, rsum, n_values: int):
    """The batch values of test_sdf_acc from per-image sdf_metrics results summed over n_values = B*N samples:
    (accuracy, sdf_loss_realvalue, sdf_loss) as float32.  accuracy equals np.mean of the 0/1 float32 agreements bit for
    bit (both operands are exact below 2^24)."""
    acc = np.float32(int(np.sum(count))) / np.float32(n_values)
    real = np.float32(float(np.sum(rsum)) / n_values)
    loss = np.float32(float(np.sum(wsum)) / n_values) * np.float32(1000)
    return acc, real, loss


CAM_LOSS_KEYS = ("rotpc_loss", "rot2d_loss", "rot3d_dist", "rot2d_dist", "rotmatrix_loss", "regularization",
                 "overall_loss")


def cam_losses(sums, n_points: int, regularization, loss_mode: str = "3D"):
    """The losses of cam_est/model_cam.py get_loss (:153-237) from per-image cam_metrics sums [B,5] over n_points points
    per image: (dict of float32 in CAM_LOSS_KEYS order, rot3d_dist_all [B], rot2d_dist_all [B]).  overall_loss follows
    --loss_mode: 3D rotpc, 2D rot2d, 3DM rotpc + 0.3 rotmatrix, anything else rot2d + rotpc + rotmatrix; plus the
    regularization constant of the checkpoint."""
    s = np.asarray(sums, np.float64).reshape(-1, 5)
    B = len(s)
    f32 = np.float32
    rotpc = f32(float(np.sum(s[:, 0])) / 2)                                   # l2_loss = sum / 2
    rot2d = f32(float(np.sum(s[:, 1])) / 2) / f32(10000.)
    rot3d_all = (s[:, 2] / n_points).astype(np.float32)                       # reduce_mean over the points
    rot2d_all = (s[:, 3] / n_points).astype(np.float32)
    rot3d = f32(np.mean(rot3d_all, dtype=np.float64))
    rot2d_dist = f32(np.mean(rot2d_all, dtype=np.float64))
    rotmatrix = f32(float(np.sum(s[:, 4])) / (12 * B))
    if loss_mode == "3D":
        loss = rotpc
    elif loss_mode == "2D":
        loss = rot2d
    elif loss_mode == "3DM":
        loss = rotpc + rotmatrix * f32(0.3)
    else:
        loss = rot2d + rotpc + rotmatrix
    reg = f32(regularization)
    vals = (rotpc, rot2d, rot3d, rot2d_dist, rotmatrix, reg, f32(loss + reg))
    return dict(zip(CAM_LOSS_KEYS, vals)), rot3d_all, rot2d_all


def write_dist(path: str, res: int, bbox, values):
    """C-ABI .dist writer (test/create_sdf.py:292-303 layout)."""
    v = _f32(values).reshape(-1)
    if v.size != (res + 1) ** 3:
        raise ValueError("values must hold (res+1)^3 samples")
    bb = (C.c_double * 6)(*[float(x) for x in bbox])
    check(_lib.load().disn_write_dist(path.encode(), res, bb, v.ctypes.data_as(C.c_void_p)))
