"""Deterministic synthetic inputs for the SDF path (no dataset, no checkpoint): images, ShapeNet-style
cameras, and random-init weights keyed by the reference's TF variable names.

Camera convention restated from the reference's preprocessing (preprocessing/create_img_h5.py:14-63
getBlenderProj, :65-103 get_rotate_matrix, :106-123 get_norm_matrix, :183-185 composition):
``trans_mat = (K · RT · rot(-pi/2) · norm)^T`` with K = [[f,0,c],[0,f,c],[0,0,1]], f = 35·137/32,
c = 137/2.  tests/golden pins this module against the reference's own functions.
"""
from __future__ import annotations

import math

import numpy as np

IMG_H = IMG_W = 137
F_PIX = 35.0 * 137 / 32.0      # 149.84375 (cam_est/model_cam.py:28)
C_PIX = 137 / 2.0              # 68.5
CAM_MAX_DIST = 1.75

# demo/demo.py:272-276 -- the shipped ground-truth camera for the demo chair
DEMO_TRANS_MAT = np.asarray(
    [[[-68.453156, 5.5086656, -0.37556022],
      [-17.138561, -84.685486, -0.250198],
      [-47.284092, -3.6569588, 0.2493176],
      [101.133705, 101.34268, 1.4305686]]], dtype=np.float32)
DEMO_SDF_PARAMS = np.array([[-1, -1, -1, 1, 1, 1]], dtype=np.float64)   # demo/demo.py:278
# demo/demo.py:121 (commented cam_gt): az, el, 0, dist_ratio, 25
DEMO_CAM_GT = (326.421594487, 29.0316186116, 0.790311739218)


def intrinsics() -> np.ndarray:
    return np.array([[F_PIX, 0.0, C_PIX], [0.0, F_PIX, C_PIX], [0.0, 0.0, 1.0]], dtype=np.float64)


def blender_extrinsics(az_deg, el_deg, distance_ratio) -> np.ndarray:
    """3x4 [R|T] world->camera of the ShapeNet renderer (az/el in degrees), float64.  The sines and the camera distance
    are computed in the arguments' type, as getBlenderProj computes them: the view files pass the float32 values of
    rendering_metadata.txt (disn_b200/create_img_h5.py), so there they are float32."""
    a, e = np.radians(-az_deg), np.radians(-el_deg)
    sa, ca, se, ce = np.sin(a), np.cos(a), np.sin(e), np.cos(e)
    world2obj = np.array([[ca * ce, -sa, ca * se],
                          [sa * ce, ca, sa * se],
                          [-se, 0.0, ce]], dtype=np.float64).T
    eps = 4.371138828673793e-08
    cam_rot = np.array([[1.910685676922942e-15, eps, 1.0],
                        [1.0, -eps, -0.0],
                        [eps, 1.0, -eps]], dtype=np.float64)
    obj2cam = cam_rot.T
    flip = np.diag([1.0, -1.0, -1.0])
    R = flip @ (obj2cam @ world2obj)
    T = flip @ (-obj2cam @ np.array([[distance_ratio * CAM_MAX_DIST], [0.0], [0.0]], dtype=np.float64))
    return np.hstack([R, T])


def axis_rotation_matrix(angle: float) -> np.ndarray:
    """4x4 product neg·Rz·Rz·flipY·Rx used by the reference with angle = -pi/2."""
    c, s = math.cos(angle), math.sin(angle)
    rx = np.array([[1, 0, 0, 0], [0, c, -s, 0], [0, s, c, 0], [0, 0, 0, 1]], dtype=np.float64)
    rz = np.array([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], dtype=np.float64)
    flip_y = np.diag([1.0, -1.0, 1.0, 1.0])
    neg = np.diag([-1.0, -1.0, -1.0, 1.0])
    return neg @ rz @ rz @ flip_y @ rx


def norm_matrix(centre, m: float) -> np.ndarray:
    """T(centre)·S(m): maps the normalised [-1,1]^3 SDF frame back to the raw mesh frame."""
    M = np.diag([m, m, m, 1.0])
    T = np.eye(4)
    T[:3, 3] = centre
    return T @ M


def make_trans_mat(az_deg, el_deg, distance_ratio, m=1.0, centre=(0.0, 0.0, 0.0)) -> np.ndarray:
    """[4,3] float32 right-multiplied projection: [x,y,z,1]·trans_mat = (u·w, v·w, w)."""
    P = intrinsics() @ blender_extrinsics(az_deg, el_deg, distance_ratio) \
        @ axis_rotation_matrix(-math.pi / 2) @ norm_matrix(centre, m)
    return np.ascontiguousarray(P.T.astype(np.float32))


def synthetic_trans_mats(batch: int, seed: int = 4321) -> np.ndarray:
    """SURVEY.md 8d(ii): az U[0,360), el U[25,30], dist U[0.65,0.95], m U[0.4,0.6], centre U[-.05,.05]^3."""
    out = np.zeros((batch, 4, 3), dtype=np.float32)
    for b in range(batch):
        r = np.random.default_rng(seed + b)
        out[b] = make_trans_mat(r.uniform(0, 360), r.uniform(25, 30), r.uniform(0.65, 0.95),
                                r.uniform(0.4, 0.6), r.uniform(-0.05, 0.05, size=3))
    return out


def synthetic_images(batch: int, seed: int = 1234, smooth: bool = True) -> np.ndarray:
    """[B,137,137,3] float32 in [0,1] (like /255. renders, demo/demo.py:264)."""
    out = np.zeros((batch, IMG_H, IMG_W, 3), dtype=np.float32)
    for b in range(batch):
        img = np.random.default_rng(seed + b).random((IMG_H, IMG_W, 3), dtype=np.float32)
        if smooth:  # 3x3 box blur keeps some spatial structure; still in [0,1]
            p = np.pad(img, ((1, 1), (1, 1), (0, 0)), mode="edge")
            img = sum(p[i:i + IMG_H, j:j + IMG_W] for i in range(3) for j in range(3)) / np.float32(9.0)
        out[b] = img.astype(np.float32)
    return out


def weight_shapes(num_classes: int = 1024) -> dict:
    """TF variable name -> shape for every variable on the path (the checkpoint contract)."""
    cfg = [("conv1", 2, 64), ("conv2", 2, 128), ("conv3", 3, 256), ("conv4", 3, 512), ("conv5", 3, 512)]
    shapes, cin = {}, 3
    for blk, n, cout in cfg:
        for j in range(1, n + 1):
            shapes[f"vgg_16/{blk}/{blk}_{j}/weights"] = (3, 3, cin, cout)
            shapes[f"vgg_16/{blk}/{blk}_{j}/biases"] = (cout,)
            cin = cout
    for nm, shp in (("fc6", (7, 7, 512, 4096)), ("fc7", (1, 1, 4096, 4096)), ("fc8", (1, 1, 4096, num_classes))):
        shapes[f"vgg_16/{nm}/weights"] = shp
        shapes[f"vgg_16/{nm}/biases"] = (shp[-1],)
    for scope, cat in (("sdfprediction", 512 + num_classes), ("sdfprediction_imgfeat", 512 + 1472)):
        for nm, ci, co in (("fold1/conv1", 3, 64), ("fold1/conv2", 64, 256), ("fold1/conv3", 256, 512),
                           ("fold2/conv1", cat, 512), ("fold2/conv2", 512, 256), ("fold2/conv5", 256, 1)):
            shapes[f"{scope}/{nm}/weights"] = (1, 1, ci, co)
            shapes[f"{scope}/{nm}/biases"] = (co,)
    return shapes


_LINEAR = ("vgg_16/fc8/", "sdfprediction/fold2/conv5/", "sdfprediction_imgfeat/fold2/conv5/")


def make_weights(seed: int = 7, init: str = "he", num_classes: int = 1024) -> dict:
    """All variables of the path as float32 arrays.

    init="he":     N(0, 2/fan_in) for ReLU layers, N(0, 1/fan_in) for the three linear outputs,
                   biases N(0, 0.01) -- variance-preserving so |pred| = O(1) and a 1e-4 bar is meaningful.
    init="xavier": the reference's own initialisers (xavier-uniform weights, zero biases;
                   utils/tf_util.py:41,173-174) -- BASELINE config 0's literal random-init condition.
    """
    rng = np.random.default_rng(seed)
    W = {}
    for name, shp in weight_shapes(num_classes).items():
        if name.endswith("biases"):
            W[name] = (rng.standard_normal(shp, dtype=np.float32) * np.float32(0.01)) if init == "he" \
                else np.zeros(shp, dtype=np.float32)
            continue
        fan_in = int(np.prod(shp[:-1]))
        fan_out = int(shp[0] * shp[1] * shp[3])
        if init == "he":
            gain = 1.0 if any(name.startswith(p) for p in _LINEAR) else 2.0
            W[name] = rng.standard_normal(shp, dtype=np.float32) * np.float32(math.sqrt(gain / fan_in))
        elif init == "xavier":
            lim = math.sqrt(6.0 / (fan_in + fan_out))
            W[name] = rng.uniform(-lim, lim, size=shp).astype(np.float32)
        else:
            raise ValueError(init)
    return W
