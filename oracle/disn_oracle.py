"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the DISN two-stream SDF inference graph.

PARITY UNPINNED against TensorFlow itself (TF 1.x is not installable here, see
oracle/__init__.py).  Every function cites the reference file:line it restates; TF op
semantics follow SURVEY.md Appendix A (TF 1.10-1.15 CPU kernels).

All functions take ``dtype`` (np.float32 for the parity oracle, np.float64 for the
error-budget twin).  Convolutions use torch CPU ops as plain fp32/fp64 primitives.
"""
from __future__ import annotations

import math
import struct
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn.functional as F

# ----------------------------------------------------------------------------------------
# constants of the drivers (test/create_sdf.py:69-81, demo/demo.py:72-84)
# ----------------------------------------------------------------------------------------
SDF_WEIGHT = 10.0            # create_sdf.py:81
TWOSTREAM_CHUNK = 214669.0   # create_sdf.py:72
IMG_H = IMG_W = 137          # create_sdf.py:27-28
VGG_IN = 224                 # model_normalization.py:47 (img_size=224)
CLAMP_MAX = 136.0            # model_normalization.py:250

VGG_CFG = [  # models/CNN/vgg.py:187-196 -- (block, n_convs, out_channels)
    ("conv1", 2, 64), ("conv2", 2, 128), ("conv3", 3, 256), ("conv4", 3, 512), ("conv5", 3, 512)]
VGG_TAPS = ["vgg_16/conv1/conv1_2", "vgg_16/conv2/conv2_2", "vgg_16/conv3/conv3_3",
            "vgg_16/conv4/conv4_3", "vgg_16/conv5/conv5_3"]   # model_normalization.py:171-183
TAP_CHANNELS = [64, 128, 256, 512, 512]


def default_flags(**kw):
    """FLAGS namespace with the attributes get_model reads (model_normalization.py:20,66,76,81-214)."""
    d = dict(alpha=False, num_classes=1024, binary=False, threedcnn=False, img_feat_onestream=False,
             img_feat_twostream=True, multi_view=False, img_h=IMG_H, img_w=IMG_W, tanh=False,
             num_sample_points=1, sdf_res=64, batch_size=1)
    d.update(kw)
    return SimpleNamespace(**d)


def chunking(sdf_res: int):
    """create_sdf.py:69-77 -- (RESOLUTION, TOTAL_POINTS, SPLIT_SIZE, NUM_SAMPLE_POINTS)."""
    resolution = sdf_res + 1
    total = resolution ** 3
    split = int(np.ceil(total / TWOSTREAM_CHUNK))
    num_sample = int(np.ceil(total / split))
    return resolution, total, split, num_sample


# ----------------------------------------------------------------------------------------
# weight names / shapes: the checkpoint contract (SURVEY.md 8a)
# ----------------------------------------------------------------------------------------
def weight_shapes(num_classes: int = 1024):
    """name -> shape (HWIO for convs), in TF variable naming."""
    shapes = {}
    cin = 3
    for blk, n, cout in VGG_CFG:
        for j in range(1, n + 1):
            shapes[f"vgg_16/{blk}/{blk}_{j}/weights"] = (3, 3, cin, cout)
            shapes[f"vgg_16/{blk}/{blk}_{j}/biases"] = (cout,)
            cin = cout
    shapes["vgg_16/fc6/weights"] = (7, 7, 512, 4096)
    shapes["vgg_16/fc6/biases"] = (4096,)
    shapes["vgg_16/fc7/weights"] = (1, 1, 4096, 4096)
    shapes["vgg_16/fc7/biases"] = (4096,)
    shapes["vgg_16/fc8/weights"] = (1, 1, 4096, num_classes)
    shapes["vgg_16/fc8/biases"] = (num_classes,)
    for scope, cat in (("sdfprediction", 512 + num_classes), ("sdfprediction_imgfeat", 512 + 1472)):
        for nm, ci, co in (("fold1/conv1", 3, 64), ("fold1/conv2", 64, 256), ("fold1/conv3", 256, 512),
                           ("fold2/conv1", cat, 512), ("fold2/conv2", 512, 256), ("fold2/conv5", 256, 1)):
            shapes[f"{scope}/{nm}/weights"] = (1, 1, ci, co)
            shapes[f"{scope}/{nm}/biases"] = (co,)
    return shapes


LINEAR_LAYERS = ("vgg_16/fc8", "sdfprediction/fold2/conv5", "sdfprediction_imgfeat/fold2/conv5")


# ----------------------------------------------------------------------------------------
# TF op semantics (SURVEY.md Appendix A)
# ----------------------------------------------------------------------------------------
def tf_resize_bilinear(x: np.ndarray, out_h: int, out_w: int, dtype=np.float32) -> np.ndarray:
    """tf.image.resize_bilinear(x,[oh,ow]) with align_corners=False, legacy (no half-pixel).

    TF 1.x CPU kernel: scale = in/out (float32); in = i*scale; lo = floor(in);
    hi = min(lo+1, in-1); lerp = in - lo; value = top + (bottom-top)*ly, top = tl + (tr-tl)*lx.
    x: [B,H,W,C].
    """
    x = np.asarray(x, dtype=dtype)
    B, H, W, C = x.shape

    def weights(in_size, out_size):
        scale = np.float32(in_size) / np.float32(out_size) if (out_size > 0) else np.float32(0)
        i = np.arange(out_size, dtype=np.float32)
        src = (i * scale).astype(np.float32)
        lo = np.floor(src).astype(np.int64)
        hi = np.minimum(lo + 1, in_size - 1)
        lerp = (src - lo.astype(np.float32)).astype(np.float32)
        return lo, hi, lerp.astype(dtype)

    ylo, yhi, yl = weights(H, out_h)
    xlo, xhi, xl = weights(W, out_w)
    tl = x[:, ylo][:, :, xlo]
    tr = x[:, ylo][:, :, xhi]
    bl = x[:, yhi][:, :, xlo]
    br = x[:, yhi][:, :, xhi]
    xl_ = xl[None, None, :, None]
    yl_ = yl[None, :, None, None]
    top = tl + (tr - tl) * xl_
    bot = bl + (br - bl) * xl_
    return (top + (bot - top) * yl_).astype(dtype)


def tf_resampler(data: np.ndarray, warp: np.ndarray, dtype=np.float32) -> np.ndarray:
    """tf.contrib.resampler.resampler(data[B,H,W,C], warp[B,N,2]) -> [B,N,C].

    x = warp[...,0] (width axis), y = warp[...,1]; zero unless -1<x<W and -1<y<H;
    out = dx*dy*D(fx,fy) + (1-dx)*(1-dy)*D(cx,cy) + dx*(1-dy)*D(fx,cy) + (1-dx)*dy*D(cx,fy)
    with dx = cx - x, dy = cy - y and D == 0 outside the map.
    """
    data = np.asarray(data, dtype=dtype)
    warp = np.asarray(warp, dtype=dtype)
    B, H, W, C = data.shape
    N = warp.shape[1]
    out = np.zeros((B, N, C), dtype=dtype)
    for b in range(B):
        x = warp[b, :, 0]
        y = warp[b, :, 1]
        valid = (x > -1.0) & (y > -1.0) & (x < W) & (y < H)
        fx = np.floor(x).astype(np.int64)
        fy = np.floor(y).astype(np.int64)
        cx = fx + 1
        cy = fy + 1
        dx = (cx.astype(dtype) - x).astype(dtype)
        dy = (cy.astype(dtype) - y).astype(dtype)

        def D(ix, iy):
            ok = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
            v = data[b, np.clip(iy, 0, H - 1), np.clip(ix, 0, W - 1)]
            return v * ok[:, None].astype(dtype)

        one = dtype(1.0)
        res = ((dx * dy)[:, None] * D(fx, fy) + ((one - dx) * (one - dy))[:, None] * D(cx, cy)
               + (dx * (one - dy))[:, None] * D(fx, cy) + ((one - dx) * dy)[:, None] * D(cx, fy))
        out[b] = res * valid[:, None].astype(dtype)
    return out


def _conv2d_nhwc(x, w_hwio, b, padding, relu, dtype):
    """slim.conv2d: cross-correlation with HWIO weights, stride 1, SAME/VALID, bias, ReLU."""
    tdt = torch.float32 if dtype == np.float32 else torch.float64
    xt = torch.from_numpy(np.ascontiguousarray(x)).to(tdt).permute(0, 3, 1, 2)
    wt = torch.from_numpy(np.ascontiguousarray(w_hwio)).to(tdt).permute(3, 2, 0, 1).contiguous()
    bt = torch.from_numpy(np.ascontiguousarray(b)).to(tdt)
    pad = (w_hwio.shape[0] // 2) if padding == "SAME" else 0
    y = F.conv2d(xt, wt, bt, stride=1, padding=pad)
    if relu:
        y = torch.relu(y)
    return y.permute(0, 2, 3, 1).contiguous().numpy()


def _maxpool2(x, dtype):
    tdt = torch.float32 if dtype == np.float32 else torch.float64
    xt = torch.from_numpy(np.ascontiguousarray(x)).to(tdt).permute(0, 3, 1, 2)
    y = F.max_pool2d(xt, 2, 2)  # slim.max_pool2d([2,2]) stride 2 VALID
    return y.permute(0, 2, 3, 1).contiguous().numpy()


def vgg_16(img: np.ndarray, W: dict, dtype=np.float32):
    """slim vgg_16(img, num_classes, is_training=False, spatial_squeeze=False)
    (models/CNN/vgg.py:182-218; call at model_normalization.py:76).

    img: [B,224,224,3] in [0,1], no mean subtraction.  Returns (net[B,1,1,nc], end_points).
    """
    net = np.asarray(img, dtype=dtype)
    end_points = {}
    for blk, n, _ in VGG_CFG:
        for j in range(1, n + 1):
            nm = f"vgg_16/{blk}/{blk}_{j}"
            net = _conv2d_nhwc(net, W[nm + "/weights"], W[nm + "/biases"], "SAME", True, dtype)
            end_points[nm] = net
        net = _maxpool2(net, dtype)
        end_points[f"vgg_16/pool{blk[-1]}"] = net
    net = _conv2d_nhwc(net, W["vgg_16/fc6/weights"], W["vgg_16/fc6/biases"], "VALID", True, dtype)
    end_points["vgg_16/fc6"] = net
    net = _conv2d_nhwc(net, W["vgg_16/fc7/weights"], W["vgg_16/fc7/biases"], "VALID", True, dtype)
    end_points["vgg_16/fc7"] = net
    net = _conv2d_nhwc(net, W["vgg_16/fc8/weights"], W["vgg_16/fc8/biases"], "VALID", False, dtype)
    end_points["vgg_16/fc8"] = net
    return net, end_points


def get_img_points(sample_pc: np.ndarray, trans_mat_right: np.ndarray, dtype=np.float32):
    """model_normalization.py:241-251 -- [x,y,z,1]·T(4x3) -> (q0/q2, q1/q2) -> clamp [0,136]."""
    pc = np.asarray(sample_pc, dtype=dtype)
    T = np.asarray(trans_mat_right, dtype=dtype)
    homo = np.concatenate([pc, np.ones(pc.shape[:2] + (1,), dtype=dtype)], axis=-1)
    xyz = np.matmul(homo, T)
    xy = xyz[:, :, :2] / xyz[:, :, 2:3]
    return np.minimum(dtype(CLAMP_MAX), np.maximum(dtype(0.0), xy)).astype(dtype)


def conv2d_1x1(x: np.ndarray, w: np.ndarray, b: np.ndarray, relu: bool = True):
    """utils/tf_util.py:119-184 with kernel [1,1], VALID, bn=False: y = x·W[Cin,Cout] + b (ReLU)."""
    y = np.matmul(x, w.reshape(w.shape[-2], w.shape[-1])) + b
    return np.maximum(y, 0) if relu else y


def get_sdf_basic2(src_pc, globalfeats, W, scope="sdfprediction", dtype=np.float32):
    """models/sdfnet.py:69-92 -- global stream.  src_pc [B,N,3], globalfeats [B,1024] -> [B,N,1]."""
    g = lambda n: np.asarray(W[f"{scope}/{n}"], dtype=dtype)
    net = np.asarray(src_pc, dtype=dtype)
    for nm in ("fold1/conv1", "fold1/conv2", "fold1/conv3"):
        net = conv2d_1x1(net, g(nm + "/weights"), g(nm + "/biases"))
    B, N, _ = net.shape
    gf = np.asarray(globalfeats, dtype=dtype).reshape(B, 1, -1)
    concat = np.concatenate([net, np.broadcast_to(gf, (B, N, gf.shape[-1]))], axis=2)  # [net2, global]
    net = conv2d_1x1(concat, g("fold2/conv1/weights"), g("fold2/conv1/biases"))
    net = conv2d_1x1(net, g("fold2/conv2/weights"), g("fold2/conv2/biases"))
    return conv2d_1x1(net, g("fold2/conv5/weights"), g("fold2/conv5/biases"), relu=False)


def get_sdf_basic2_imgfeat_twostream(src_pc, point_feat, W, scope="sdfprediction_imgfeat", dtype=np.float32):
    """models/sdfnet.py:171-190 -- local stream.  point_feat [B,N,1472] -> [B,N,1]."""
    g = lambda n: np.asarray(W[f"{scope}/{n}"], dtype=dtype)
    net = np.asarray(src_pc, dtype=dtype)
    for nm in ("fold1/conv1", "fold1/conv2", "fold1/conv3"):
        net = conv2d_1x1(net, g(nm + "/weights"), g(nm + "/biases"))
    concat = np.concatenate([net, np.asarray(point_feat, dtype=dtype)], axis=2)      # [net2, point_feat]
    net = conv2d_1x1(concat, g("fold2/conv1/weights"), g("fold2/conv1/biases"))
    net = conv2d_1x1(net, g("fold2/conv2/weights"), g("fold2/conv2/biases"))
    return conv2d_1x1(net, g("fold2/conv5/weights"), g("fold2/conv5/biases"), relu=False)


def encode(imgs: np.ndarray, W: dict, FLAGS=None, dtype=np.float32):
    """model_normalization.py:47-79 + :171-183 -- image -> (global embedding, 5 resized 137x137 maps)."""
    FLAGS = FLAGS or default_flags()
    ref_img = np.asarray(imgs, dtype=dtype)
    if ref_img.shape[1] != VGG_IN or ref_img.shape[2] != VGG_IN:      # :65-72
        ref_img = tf_resize_bilinear(ref_img, VGG_IN, VGG_IN, dtype)
    net, ep = vgg_16(ref_img, {k: np.asarray(v, dtype=dtype) for k, v in W.items() if k.startswith("vgg_16")}, dtype)
    emb = net.reshape(net.shape[0], -1)                               # tf.squeeze axis [1,2] (:77)
    maps = [tf_resize_bilinear(ep[t], FLAGS.img_h, FLAGS.img_w, dtype) for t in VGG_TAPS]
    return SimpleNamespace(resized_ref_img=ref_img, img_embedding=emb, maps=maps, vgg_end_points=ep)


def decode(enc, sample_pc, sample_pc_rot, trans_mat, W, FLAGS=None, dtype=np.float32):
    """model_normalization.py:169-206,214-219 -- twostream branch given the encoder outputs."""
    FLAGS = FLAGS or default_flags()
    uv = get_img_points(sample_pc, trans_mat, dtype)                                   # :170
    feats = [tf_resampler(m, uv, dtype) for m in enc.maps]                             # :171-185
    point_img_feat = np.concatenate(feats, axis=2)                                     # :187-189
    pg = get_sdf_basic2(sample_pc_rot, enc.img_embedding, W, dtype=dtype)              # :194-197
    pl = get_sdf_basic2_imgfeat_twostream(sample_pc_rot, point_img_feat, W, dtype=dtype)  # :199-202
    pred = pg + pl                                                                     # :204
    if FLAGS.tanh:
        pred = np.tanh(pred)                                                           # :214-215
    return dict(pred_sdf=pred, pred_sdf_value_global=pg, pred_sdf_value_local=pl,
                sample_img_points=uv, point_img_feat=point_img_feat[:, :, None, :])


def get_model(imgs, sample_pc, sample_pc_rot, trans_mat, W, FLAGS=None, dtype=np.float32):
    """model_normalization.get_model (:47-221), twostream non-binary branch, one sess.run."""
    enc = encode(imgs, W, FLAGS, dtype)
    out = decode(enc, sample_pc, sample_pc_rot, trans_mat, W, FLAGS, dtype)
    out.update(ref_img=np.asarray(imgs), resized_ref_img=enc.resized_ref_img,
               img_embedding=enc.img_embedding, ref_feats_embedding_cnn=enc.img_embedding)
    return out


def get_loss(pred_sdf, gt_sdf, sdf_weight=10.0, mask_weight=4.0):
    """model_normalization.py:279-291 -- non-binary metrics (accuracy, sdf_loss, sdf_loss_realvalue)."""
    pred_sdf = np.asarray(pred_sdf, np.float32)
    gt_sdf = np.asarray(gt_sdf, np.float32)
    acc = np.mean(((gt_sdf > 0) == (pred_sdf > 0)).astype(np.float32))
    wm = (gt_sdf <= 0.01).astype(np.float32) * mask_weight + (gt_sdf > 0.01).astype(np.float32)
    sdf_loss = np.mean(np.abs(gt_sdf * sdf_weight - pred_sdf) * wm) * 1000
    real = np.mean(np.abs(gt_sdf - pred_sdf / sdf_weight))
    return dict(accuracy=acc, sdf_loss=sdf_loss, sdf_loss_realvalue=real)


# ----------------------------------------------------------------------------------------
# driver loop (test/create_sdf.py:224-303)
# ----------------------------------------------------------------------------------------
def grid_points(sdf_params, resolution: int) -> np.ndarray:
    """create_sdf.py:246-255 -- float64 linspace per axis, meshgrid(z,y,x,'ij'), (x,y,z), f32; x fastest."""
    x_ = np.linspace(sdf_params[0], sdf_params[3], num=resolution)
    y_ = np.linspace(sdf_params[1], sdf_params[4], num=resolution)
    z_ = np.linspace(sdf_params[2], sdf_params[5], num=resolution)
    z, y, x = np.meshgrid(z_, y_, x_, indexing="ij")
    return np.stack([x, y, z], axis=3).astype(np.float32).reshape(-1, 3)


def create_sdf_grid(imgs, trans_mat, sdf_params, W, sdf_res, FLAGS=None, dtype=np.float32,
                    rerun_encoder_per_chunk=False):
    """create_sdf.py:241-285 -- dense grid in SPLIT_SIZE chunks, reassembled, /SDF_WEIGHT (float64).

    Returns result [B, R^3, 1] float64.  ``rerun_encoder_per_chunk`` reproduces the reference's
    loop literally (whole graph incl. VGG per sess.run, :262-275).
    """
    FLAGS = FLAGS or default_flags(sdf_res=sdf_res)
    R, total, split, nsp = chunking(sdf_res)
    B = np.asarray(imgs).shape[0]
    extra = np.zeros((1, split * nsp - total, 3), dtype=np.float32)
    batch_points = np.zeros((split, 0, nsp, 3), dtype=np.float32)
    for b in range(B):
        pts = grid_points(sdf_params[b], R).reshape(1, -1, 3)
        pts = np.concatenate((pts, extra), axis=1).reshape(split, 1, -1, 3)
        batch_points = np.concatenate((batch_points, pts), axis=1)
    pred_all = np.zeros((split, B, nsp, 1))
    enc = None if rerun_encoder_per_chunk else encode(imgs, W, FLAGS, dtype)
    for sp in range(split):
        pc = batch_points[sp].reshape(B, -1, 3)
        e = encode(imgs, W, FLAGS, dtype) if rerun_encoder_per_chunk else enc
        pred_all[sp] = decode(e, pc, pc, trans_mat, W, FLAGS, dtype)["pred_sdf"]
    pred_all = np.swapaxes(pred_all, 0, 1).reshape(B, -1, 1)[:, :total, :]
    return pred_all / SDF_WEIGHT


def to_binary(res, pos, pred_sdf_val_all, sdf_file):
    """create_sdf.py:292-303 -- .dist: int32 -res,res,res; 6 float64 bbox; R^3 float32 (z,y,x C-order)."""
    with open(sdf_file, "wb") as f:
        f.write(struct.pack("i", -res))
        f.write(struct.pack("i", res))
        f.write(struct.pack("i", res))
        f.write(struct.pack("d" * len(pos), *pos))
        vals = np.asarray(pred_sdf_val_all, dtype=np.float64).reshape(-1)
        f.write(struct.pack("=%sf" % vals.shape[0], *vals))


# ----------------------------------------------------------------------------------------
# algebraic folds used by the CUDA path, restated on CPU so tests can check them separately
# ----------------------------------------------------------------------------------------
def folded_decode(enc, sample_pc, trans_mat, W, dtype=np.float64):
    """Same result as decode() in exact arithmetic, computed the way the CUDA path does:
    global feature -> per-image bias, VGG taps -> one projected 137x137x512 map gathered per point."""
    Wg = np.asarray(W["sdfprediction/fold2/conv1/weights"], dtype).reshape(-1, 512)
    Wl = np.asarray(W["sdfprediction_imgfeat/fold2/conv1/weights"], dtype).reshape(-1, 512)
    B = enc.img_embedding.shape[0]
    gbias = enc.img_embedding.astype(dtype) @ Wg[512:] + np.asarray(W["sdfprediction/fold2/conv1/biases"], dtype)
    off = 512
    pmap = 0
    for m, c in zip(enc.maps, TAP_CHANNELS):
        pmap = pmap + np.asarray(m, dtype) @ Wl[off:off + c]
        off += c
    uv = get_img_points(sample_pc, trans_mat, dtype)
    pfeat = tf_resampler(pmap, uv, dtype)          # [B,N,512]

    def stream(scope, extra):
        g = lambda n: np.asarray(W[f"{scope}/{n}"], dtype)
        net = np.asarray(sample_pc, dtype)
        for nm in ("fold1/conv1", "fold1/conv2", "fold1/conv3"):
            net = conv2d_1x1(net, g(nm + "/weights"), g(nm + "/biases"))
        w1 = g("fold2/conv1/weights").reshape(-1, 512)[:512]
        net = np.maximum(net @ w1 + extra, 0)
        net = conv2d_1x1(net, g("fold2/conv2/weights"), g("fold2/conv2/biases"))
        return conv2d_1x1(net, g("fold2/conv5/weights"), g("fold2/conv5/biases"), relu=False)

    pg = stream("sdfprediction", gbias.reshape(B, 1, 512))
    pl = stream("sdfprediction_imgfeat", pfeat + np.asarray(W["sdfprediction_imgfeat/fold2/conv1/biases"], dtype))
    return pg + pl


# ----------------------------------------------------------------------------------------
# estimated-camera path (cam_est/model_cam.py:47-109, models/posenet.py:22-36,91-124)
# ----------------------------------------------------------------------------------------
CAM_K = np.array([[149.84375, 0., 68.5], [0., 149.84375, 68.5], [0., 0., 1.]], dtype=np.float64)   # model_cam.py:28
CAM_T_OFFSET = np.array([-0.00193892, 0.00169222, 1.3949631])                                        # posenet.py:118


def cam_head_shapes():
    s = {}
    for head, dims in (("scale", (1024, 64, 32, 1)), ("ortho6d", (1024, 512, 256, 6)), ("translation", (1024, 128, 64, 3))):
        for i in range(3):
            s["cameraprediction/%s/fc%d/weights" % (head, i + 1)] = (dims[i], dims[i + 1])
            s["cameraprediction/%s/fc%d/biases" % (head, i + 1)] = (dims[i + 1],)
    return s


def rotation_from_ortho6d(poses):
    """models/posenet.py:22-36."""
    x_raw, y_raw = poses[:, 0:3], poses[:, 3:6]
    nrm = lambda v: v / np.maximum(np.sqrt((v * v).sum(1, keepdims=True)), 1e-8)
    x = nrm(x_raw)
    z = nrm(np.cross(x, y_raw))
    y = np.cross(z, x)
    return np.stack([x, y, z], axis=2)


def cam_estimate(imgs, W, K=CAM_K, dtype=np.float64):
    """model_cam.get_model (non-shift branch): -> (pred_RT [B,4,3], pred_trans_mat [B,4,3])."""
    img = np.asarray(imgs, dtype)
    if img.shape[1] != VGG_IN or img.shape[2] != VGG_IN:
        img = tf_resize_bilinear(img, VGG_IN, VGG_IN, dtype)
    net, _ = vgg_16(img, {k: np.asarray(v, dtype) for k, v in W.items() if k.startswith("vgg_16")}, dtype)
    g = net.reshape(net.shape[0], -1)

    def head(name):
        h = g
        for i in (1, 2, 3):
            h = h @ np.asarray(W["cameraprediction/%s/fc%d/weights" % (name, i)], dtype) + \
                np.asarray(W["cameraprediction/%s/fc%d/biases" % (name, i)], dtype)
            if i < 3:
                h = np.maximum(h, 0)
        return h

    scale = head("scale").reshape(-1, 1, 1) * np.eye(3)[None]
    R = rotation_from_ortho6d(head("ortho6d"))
    t = head("translation") + CAM_T_OFFSET
    Rs = scale @ R
    RT = np.concatenate([Rs, t[:, None, :]], axis=1)
    return RT, RT @ np.asarray(K, dtype).T


# Faults cam_pose can apply, so a test can show each one is visible to the camera tests' bounds.
CAM_FAULTS = ("offset_dropped", "offset_permuted", "K_not_transposed", "rows_not_columns", "z_unnormalised",
              "no_clamp", "scale_after_translation")


def cam_head_outputs(emb, W, mode="float64"):
    """The three fully-connected heads of posenet.get_cam_mat on embeddings [B, num_classes] -> (scale [B],
    ortho6d [B,6], translation [B,3]) before the offset.  "float64": float64 throughout; "float32-ops": the same float64
    values rounded once to float32 (a correctly rounded dot product: TF's float32 matmul pins no summation order)."""
    g = np.asarray(emb, np.float64)

    def head(name):
        h = g
        for i in (1, 2, 3):
            h = h @ np.asarray(W["cameraprediction/%s/fc%d/weights" % (name, i)], np.float64) + \
                np.asarray(W["cameraprediction/%s/fc%d/biases" % (name, i)], np.float64)
            if i < 3:
                h = np.maximum(h, 0)
        return h

    out = head("scale")[:, 0], head("ortho6d"), head("translation")
    return tuple(o.astype(np.float32) for o in out) if mode == "float32-ops" else out


def cam_pose(scale, ortho6d, translation, K=CAM_K, mode="float64", fault=None):
    """posenet.get_cam_mat after its heads (posenet.py:97,120-124, :13-36) and model_cam.py:102-103 -> (pred_RT [B,4,3],
    pred_trans_mat [B,4,3]).  "float64": every op in float64.  "float32-ops": every TF op rounded to float32 on its own,
    in TF's order -- square, reduce_sum (left to right), sqrt, maximum(., 1e-8), divide, cross (each product, then the
    difference), scale * I, matmul(scale * I, R), + offset, matmul(RT, K^T) (products, then left-to-right sums).
    `fault` (one of CAM_FAULTS) applies a deliberate mistake instead of the reference's step."""
    f = np.float32 if mode == "float32-ops" else np.float64
    assert mode in ("float64", "float32-ops") and (fault is None or fault in CAM_FAULTS)
    s = np.asarray(scale, f).reshape(-1)
    p = np.asarray(ortho6d, f)
    t = np.asarray(translation, f)
    Km = np.asarray(K, f).reshape(3, 3)
    B = s.shape[0]

    def normalize(v):
        sq = v * v
        mag = np.sqrt((sq[:, 0] + sq[:, 1]) + sq[:, 2])[:, None]
        if fault != "no_clamp":
            mag = np.maximum(mag, f(1e-8))
        with np.errstate(invalid="ignore", divide="ignore"):
            return v / mag

    def cross(a, b):
        return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                         a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)

    with np.errstate(over="ignore", invalid="ignore"):
        x = normalize(p[:, 0:3])
        z = cross(x, p[:, 3:6])
        if fault != "z_unnormalised":
            z = normalize(z)
        y = cross(z, x)
        R = np.stack([x, y, z], axis=1 if fault == "rows_not_columns" else 2)     # matrix[:, i, j] = (x, y, z)[j][i]
        S = s[:, None, None] * np.eye(3, dtype=f)[None]
        off = np.asarray(CAM_T_OFFSET, f)
        if fault == "offset_dropped":
            off = np.zeros(3, f)
        elif fault == "offset_permuted":
            off = off[[1, 2, 0]]
        tr = (t + off)[:, None, :]

        def matmul(A, Bm):          # [B,n,3] @ [3,m] or [B,3,m]: each product rounded, summed left to right
            Bm = np.broadcast_to(Bm, (A.shape[0],) + Bm.shape[-2:])
            return (A[:, :, 0, None] * Bm[:, None, 0, :] + A[:, :, 1, None] * Bm[:, None, 1, :]) + \
                A[:, :, 2, None] * Bm[:, None, 2, :]

        if fault == "scale_after_translation":
            RT = s[:, None, None] * np.concatenate([R, tr], axis=1)
        else:
            RT = np.concatenate([matmul(S, R), tr], axis=1)
        TM = matmul(RT, Km if fault == "K_not_transposed" else Km.T)
    assert RT.dtype == f and TM.dtype == f and RT.shape == (B, 4, 3)
    return RT, TM


def cam_heads(emb, W, K=CAM_K, mode="float64", fault=None):
    """model_cam.get_model's camera branch (non-shift) on given embeddings [B, num_classes] instead of the VGG's."""
    return cam_pose(*cam_head_outputs(emb, W, mode), K=K, mode=mode, fault=fault)
