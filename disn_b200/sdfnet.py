"""Mirror of the two reference MLP heads on the hot path (models/sdfnet.py:69-92 get_sdf_basic2,
:171-190 get_sdf_basic2_imgfeat_twostream).  In the reference these build 1x1-conv sub-graphs inside
get_model; on the CUDA path both heads live inside the fused point kernel.  Called on their own -- with placeholders
(symbolic, evaluated by Session.run) or with arrays (eager, on the engine given to set_engine) -- they run one stream of that
kernel through the explicit-feature entry point (disn_eval_features).

Layer contract (utils/tf_util.py:119-184 conv2d with kernel [1,1], VALID, bn=False: y = relu(x.W + b)):
    fold1/conv1 3->64, fold1/conv2 64->256, fold1/conv3 256->512,
    concat [point512 | global1024]  (get_sdf_basic2)         -> fold2/conv1 1536->512
    concat [point512 | point_feat1472] (..._imgfeat_twostream) -> fold2/conv1 1984->512
    fold2/conv2 512->256, fold2/conv5 256->1 (linear)
"""
from __future__ import annotations

import numpy as np

from .model_normalization import Placeholder, Tensor, _Graph

LAYERS = (("fold1/conv1", 3, 64, True), ("fold1/conv2", 64, 256, True), ("fold1/conv3", 256, 512, True),
          ("fold2/conv1", None, 512, True), ("fold2/conv2", 512, 256, True), ("fold2/conv5", 256, 1, False))

_ENGINE = None


def set_engine(engine):
    """Engine (with the SDF-head weights loaded) used when the heads are called eagerly on arrays."""
    global _ENGINE
    _ENGINE = engine


def _head(kind, src_pc, feats, feat_key, batch_size, bn):
    if bn:
        raise NotImplementedError("bn=True is not used at inference (test/create_sdf.py:169)")
    if isinstance(src_pc, Placeholder) or isinstance(feats, Placeholder):
        # symbolic: Session.run feeds the two placeholders and evaluates the head through disn_eval_features
        g = _Graph({"head_src_pc": src_pc, feat_key: feats}, None, None, None)
        return Tensor(kind, g, (batch_size, src_pc.shape[1] if hasattr(src_pc, "shape") else None, 1))
    if _ENGINE is None:
        raise RuntimeError("sdfnet heads called on arrays: call sdfnet.set_engine(engine) first")
    return eval_head(_ENGINE, kind, src_pc, feats)


def eval_head(engine, kind, src_pc, feats):
    """One head on explicit features through the decoder entry point: the other stream gets zero features and is ignored."""
    pts = np.ascontiguousarray(src_pc, np.float32)
    B, N, _ = pts.shape
    if kind == "head_global":
        out = engine.eval_features(pts, np.asarray(feats, np.float32).reshape(B, -1), np.zeros((B, N, 1472), np.float32))
        return out[1]
    out = engine.eval_features(pts, np.zeros((B, engine.cfg.num_classes), np.float32), np.asarray(feats, np.float32).reshape(B, N, 1472))
    return out[2]


def get_sdf_basic2(src_pc, globalfeats, is_training, batch_size, num_point, bn, bn_decay, wd=None):
    """models/sdfnet.py:69-92 -- global stream: src_pc [B,N,3], globalfeats [B,1024] (any shape with B*1024 elements)
    -> [B,N,1].  Placeholders give a symbolic tensor for Session.run; arrays are evaluated on the engine of set_engine()."""
    return _head("head_global", src_pc, globalfeats, "head_globalfeats", batch_size, bn)


def get_sdf_basic2_imgfeat_twostream(src_pc, point_feat, is_training, batch_size, num_point, bn, bn_decay, wd=None):
    """models/sdfnet.py:171-190 -- local stream: src_pc [B,N,3], point_feat [B,N,1,1472] -> [B,N,1]."""
    return _head("head_local", src_pc, point_feat, "head_point_feat", batch_size, bn)
