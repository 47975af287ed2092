"""Mirror of the reference's single-image demo (demo/demo.py): one 137x137 render -> (optionally estimated) camera ->
dense SDF grid -> mesh, on the CUDA path.  Same function names and argument meaning as the reference's module:

    read_img_get_transmat()      demo/demo.py:261-279   image -> batch_data {img, trans_mat, sdf_params}
    cam_evl(img_arr)             demo/demo.py:195-258   estimated-camera network -> pred_trans_mat
    create()                     demo/demo.py:123-193   build the graph, restore the checkpoint, run test_one_epoch
    create_obj(pred, params, dir, i)   demo/demo.py:355-363   .dist -> marching cubes at iso i -> <dir>/result.obj

The heavy lifting is create_sdf.py's (same chunk arithmetic, same session shim); this file only adds what the demo has on
top: the image loader, the hard-coded ground-truth camera of the shipped example and the --cam_est switch.
"""
from __future__ import annotations

import os

import numpy as np

from . import create_sdf as drv
from .engine import Engine
from .synth import DEMO_SDF_PARAMS, DEMO_TRANS_MAT

IMG_FILE = "./demo/03001627_17e916fc863540ee3def89b32cef8e45_20.png"    # demo/demo.py:262
CAM_WEIGHTS = None      # camera checkpoint variables (vgg_16/*, cameraprediction/*) for --cam_est


def default_flags(**kw):
    """argparse defaults of demo/demo.py:27-65 (on top of the driver's)."""
    kw.setdefault("sdf_res", 64)
    kw.setdefault("cam_log_dir", "./cam_est/checkpoint/cam_DISN")
    return drv.default_flags(**kw)


def cam_evl(img_arr, device: int = 0):
    """demo/demo.py:195-258: run the camera network on [B,137,137,3] images in [0,1] -> pred_trans_mat [B,4,3].
    Needs CAM_WEIGHTS (e.g. tf_checkpoint.load_checkpoint(FLAGS.cam_log_dir + '/model.ckpt'))."""
    if CAM_WEIGHTS is None:
        raise RuntimeError("Fail to load overall modelfile: set disn_b200.demo.CAM_WEIGHTS to the camera checkpoint's variables")
    eng = Engine(device=device, precision="bf16x3", max_batch=max(1, len(img_arr)))
    try:
        eng.load_weights_raw(CAM_WEIGHTS)
        pred_trans_mat_val = eng.cam_estimate(img_arr)
    finally:
        eng.close()
    print("pred_trans_mat_val", pred_trans_mat_val)
    return pred_trans_mat_val


def read_img_get_transmat(img_file: str | None = None, cam_est: bool | None = None):
    """demo/demo.py:261-279.  PNG (any channel count; alpha dropped like `[:, :, :3]`) -> float32 / 255."""
    import cv2
    img_file = img_file or IMG_FILE
    img = cv2.imread(img_file, cv2.IMREAD_UNCHANGED)
    if img is None:
        raise FileNotFoundError(img_file)
    if img.ndim == 2:
        img = np.repeat(img[:, :, None], 3, axis=2)
    img_arr = img.astype(np.uint8)[:, :, :3]
    batch_img = np.asarray([img_arr.astype(np.float32) / 255.])
    batch_data = {"img": batch_img}
    use_cam = drv.FLAGS.cam_est if (cam_est is None and drv.FLAGS is not None) else bool(cam_est)
    if use_cam:
        print("here we use our cam est network to estimate cam parameters:")
        batch_data["trans_mat"] = cam_evl(batch_img)
    else:
        print("here we use gt cam parameters")
        batch_data["trans_mat"] = DEMO_TRANS_MAT.copy()
    batch_data["sdf_params"] = np.asarray(DEMO_SDF_PARAMS, dtype=np.float64).reshape(1, 6).copy()
    batch_data["cat_id"], batch_data["obj_nm"], batch_data["view_id"] = ["demo"], ["obj"], [0]
    return batch_data


def create_obj(pred_sdf_val, sdf_params, dir, i):
    """demo/demo.py:355-363: writes <dir>/result.dist, meshes it at iso level `i` to <dir>/result.obj, removes the .dist."""
    os.makedirs(dir, exist_ok=True)
    obj_nm = "result"
    cube_obj_file = os.path.join(dir, obj_nm + ".obj")
    sdf_file = os.path.join(dir, obj_nm + ".dist")
    drv.to_binary((drv.RESOLUTION - 1), sdf_params, pred_sdf_val, sdf_file)
    drv.create_one_cube_obj("./isosurface/computeMarchingCubes", i, sdf_file, cube_obj_file)
    if os.path.exists(sdf_file):
        os.remove(sdf_file)                   # the reference shells out to `rm -rf`
    return cube_obj_file


def create(weights, img_file: str | None = None, flags=None, device: int = 0):
    """demo/demo.py:123-193 + :394-402: configure, read the image, run one epoch of the driver; returns the .obj paths."""
    drv.configure(flags or default_flags())
    batch_data = read_img_get_transmat(img_file)
    return drv.create(weights, [batch_data], device=device)
