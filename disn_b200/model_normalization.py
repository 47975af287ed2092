"""Drop-in mirror of the reference's ``models/model_normalization.py`` call surface for the SDF-inference
hot path (twostream, non-binary branch), executed by the C-ABI library instead of a TF-1.x graph.

Same function names, argument meaning and end_points keys as the reference
(models/model_normalization.py:14 placeholder_inputs, :38 placeholder_features, :47 get_model,
:223 get_decoder, :241 get_img_points, :254 get_loss).  "Tensors" are light symbolic handles; a
:class:`Session` plays the role of ``tf.Session``: ``sess.run(fetches, feed_dict)`` maps the reference's
feeds (test/create_sdf.py:262-275) onto ``disn_encode`` + ``disn_eval_points``.

Out of scope (raise NotImplementedError, naming the flag): FLAGS.binary / threedcnn / img_feat_onestream /
multi_view / alpha -- ablation branches of the reference graph (SURVEY.md section 2).
"""
from __future__ import annotations

import hashlib

import numpy as np

from .engine import Engine

__all__ = ["placeholder_inputs", "placeholder_features", "get_model", "get_decoder", "get_img_points",
           "get_loss", "Session", "Placeholder", "Tensor"]


class Placeholder:
    """Stand-in for tf.placeholder: a named, shaped feed slot."""

    def __init__(self, name, shape, dtype=np.float32):
        self.name, self.shape, self.dtype = name, tuple(shape), dtype

    def get_shape(self):
        return self.shape

    def __repr__(self):
        return "Placeholder(%s, %s)" % (self.name, self.shape)


class Tensor:
    """Stand-in for a graph tensor: evaluated by Session.run."""

    def __init__(self, kind, graph, shape=None):
        self.kind, self.graph, self.shape = kind, graph, shape

    def __repr__(self):
        return "Tensor(%s)" % self.kind


class _Graph:
    def __init__(self, ref_dict, FLAGS, num_point, img_size):
        self.pl = ref_dict
        self.FLAGS = FLAGS
        self.num_point = num_point
        self.img_size = img_size


def placeholder_inputs(batch_size, num_points, img_size, num_sample_pc=256, scope="", FLAGS=None):
    """models/model_normalization.py:14-35 -- same keys, same shapes."""
    c = 4 if (FLAGS is not None and getattr(FLAGS, "alpha", False)) else 3
    return {
        "pc": Placeholder(scope + "/pc", (batch_size, num_points, 3)),
        "sample_pc": Placeholder(scope + "/sample_pc", (batch_size, num_sample_pc, 3)),
        "sample_pc_rot": Placeholder(scope + "/sample_pc_rot", (batch_size, num_sample_pc, 3)),
        "imgs": Placeholder(scope + "/imgs", (batch_size, img_size[0], img_size[1], c)),
        "sdf": Placeholder(scope + "/sdf", (batch_size, num_sample_pc, 1)),
        "sdf_params": Placeholder(scope + "/sdf_params", (batch_size, 6)),
        "trans_mat": Placeholder(scope + "/trans_mat", (batch_size, 4, 3)),
    }


def placeholder_features(batch_size, num_sample_pc=256, scope=""):
    """models/model_normalization.py:38-45."""
    return {
        "ref_feats_embedding_cnn": Placeholder(scope + "/ref_feats_embedding_cnn", (batch_size, 1, 1, 1024)),
        "point_img_feat": Placeholder(scope + "/point_img_feat", (batch_size, num_sample_pc, 1, 1472)),
    }


def _check_flags(FLAGS):
    if FLAGS is None:
        raise ValueError("FLAGS is required (the reference reads FLAGS.img_feat_twostream, img_h, ...)")
    for flag in ("binary", "threedcnn", "img_feat_onestream", "multi_view", "alpha"):
        if getattr(FLAGS, flag, False):
            raise NotImplementedError("FLAGS.%s selects an ablation branch of the reference graph that is outside "
                                      "the CUDA hot path (SURVEY.md section 2)" % flag)
    if not getattr(FLAGS, "img_feat_twostream", False):
        raise NotImplementedError("only the --img_feat_twostream graph (the DISN model) is implemented")


def get_model(ref_dict, num_point, is_training, bn=False, bn_decay=None, img_size=224, wd=1e-5, FLAGS=None):
    """models/model_normalization.py:47-221 -- returns the same end_points keys (symbolic)."""
    _check_flags(FLAGS)
    if bn:
        raise NotImplementedError("bn=True is never used by the inference drivers (test/create_sdf.py:169)")
    g = _Graph(ref_dict, FLAGS, num_point, img_size)
    B = ref_dict["imgs"].shape[0]
    N = ref_dict["sample_pc"].shape[1]
    ep = {
        "ref_pc": ref_dict["pc"],
        "ref_sdf": ref_dict["sdf"],
        "ref_img": Tensor("ref_img", g, ref_dict["imgs"].shape),
        "resized_ref_img": Tensor("resized_ref_img", g, (B, img_size, img_size, 3)),
        "img_embedding": Tensor("img_embedding", g, (B, FLAGS.num_classes)),
        "ref_feats_embedding_cnn": Tensor("img_embedding", g, (B, FLAGS.num_classes)),
        "pred_sdf_value_global": Tensor("pred_sdf_value_global", g, (B, N, 1)),
        "pred_sdf_value_local": Tensor("pred_sdf_value_local", g, (B, N, 1)),
        "pred_sdf": Tensor("pred_sdf", g, (B, N, 1)),
        "sample_img_points": Tensor("sample_img_points", g, (B, N, 2)),
        "point_img_feat": Tensor("point_img_feat", g, (B, N, 1, 1472)),
    }
    return ep


def get_decoder(num_point, input_pls, feature_pls, bn=False, bn_decay=None, wd=None):
    """models/model_normalization.py:223-238 -- decoder fed with explicit features: feature_pls from
    placeholder_features() ([B,1,1,1024] global embedding, [B,N,1,1472] per-point image features), input_pls from
    placeholder_inputs() (only 'sample_pc_rot' is read).  Returns the symbolic multi_pred_sdf [B,N,1] (global + local).
    Session.run folds the features through fold2/conv1's feature rows and runs the ordinary point kernel (disn_eval_features)."""
    if bn:
        raise NotImplementedError("bn=True is never used by the inference drivers")
    g = _Graph(dict(input_pls, **feature_pls), None, num_point, None)
    B, N = input_pls["sample_pc_rot"].shape[:2]
    return Tensor("decoder_pred", g, (B, N, 1))


def get_img_points(sample_pc, trans_mat_right):
    """models/model_normalization.py:241-251 -- symbolic when given placeholders."""
    if isinstance(sample_pc, Placeholder):
        g = _Graph({"sample_pc": sample_pc, "trans_mat": trans_mat_right}, None, None, None)
        return Tensor("sample_img_points", g, sample_pc.shape[:2] + (2,))
    raise TypeError("get_img_points takes the placeholders of placeholder_inputs(); evaluate "
                    "end_points['sample_img_points'] through Session.run")


def get_loss(end_points, sdf_weight=10.0, regularization=True, mask_weight=4.0, num_sample_points=2048,
             FLAGS=None, batch_size=None):
    """models/model_normalization.py:254-300 -- metrics of the non-binary branch (:279-291).  The drivers build
    this and never fetch it at inference (test/create_sdf.py:171); the regularisation term needs the
    training graph and is not offered."""
    g = end_points["pred_sdf"].graph
    meta = dict(sdf_weight=sdf_weight, mask_weight=mask_weight)
    end_points["losses"] = {k: Tensor("loss:" + k, g) for k in ("accuracy", "sdf_loss_realvalue", "sdf_loss")}
    for t in end_points["losses"].values():
        t.meta = meta
    end_points["losses"]["overall_loss"] = end_points["losses"]["sdf_loss"]
    return end_points["losses"]["sdf_loss"], end_points


class Session:
    """Plays tf.Session for the hot path.  ``weights``: dict TF-variable-name -> array (the checkpoint
    contract, SURVEY.md 8a); like the reference's restore (test/create_sdf.py:186-192) missing variables are
    tolerated only in the sense that whatever was loaded is used -- the encoder refuses to run without its
    weights rather than silently using zeros."""

    def __init__(self, weights=None, device=0, precision="bf16x3", max_batch=8, engine=None):
        self.engine = engine or Engine(device=device, precision=precision, max_batch=max_batch)
        self._img_key = None
        if weights is not None:
            self.engine.load_weights(weights)

    def load_weights(self, weights):
        self.engine.load_weights(weights)
        self._img_key = None

    def close(self):
        self.engine.close()

    def _feed(self, feed_dict, pl):
        for k, v in feed_dict.items():
            if k is pl:
                return v
        return None

    def run(self, fetches, feed_dict=None):
        single = not isinstance(fetches, (list, tuple))
        flist = [fetches] if single else list(fetches)
        feed_dict = feed_dict or {}
        graph = next((f.graph for f in flist if isinstance(f, Tensor)), None)
        if graph is None:
            raise ValueError("nothing to run")
        pl = graph.pl
        imgs = self._feed(feed_dict, pl.get("imgs"))
        pts = self._feed(feed_dict, pl.get("sample_pc"))
        rot = self._feed(feed_dict, pl.get("sample_pc_rot"))
        tm = self._feed(feed_dict, pl.get("trans_mat"))
        kinds = [f.kind for f in flist]
        need_enc = any(k in ("pred_sdf", "img_embedding", "resized_ref_img", "point_img_feat", "pred_sdf_value_global",
                             "pred_sdf_value_local") or k.startswith("loss:") for k in kinds) and "decoder_pred" not in kinds
        if need_enc:
            if imgs is None:
                raise ValueError("imgs placeholder was not fed")
            imgs = np.ascontiguousarray(imgs, dtype=np.float32)
            key = (imgs.shape, hashlib.blake2b(imgs.tobytes(), digest_size=16).digest())
            if key != self._img_key:        # the reference re-runs VGG per chunk; once per image is enough
                self.engine.encode(imgs)
                self._img_key = key
        if any(k in ("head_global", "head_local") for k in kinds):      # sdfnet heads on their own (explicit features)
            from . import sdfnet
            res = []
            for f in flist:
                src = self._feed(feed_dict, f.graph.pl.get("head_src_pc"))
                feats = self._feed(feed_dict, f.graph.pl.get("head_globalfeats" if f.kind == "head_global" else "head_point_feat"))
                if src is None or feats is None:
                    raise ValueError("the head's src_pc / feature placeholders were not fed")
                res.append(sdfnet.eval_head(self.engine, f.kind, src, feats))
            return res[0] if single else res
        if "decoder_pred" in kinds:                     # get_decoder graph: explicit features, no encoder
            if len(set(kinds)) != 1:
                raise ValueError("fetch the decoder output on its own")
            f_rot = self._feed(feed_dict, pl.get("sample_pc_rot"))
            f_g = self._feed(feed_dict, pl.get("ref_feats_embedding_cnn"))
            f_p = self._feed(feed_dict, pl.get("point_img_feat"))
            if f_rot is None or f_g is None or f_p is None:
                raise ValueError("sample_pc_rot / ref_feats_embedding_cnn / point_img_feat placeholders were not fed")
            res = self.engine.eval_features(f_rot, f_g, f_p)[0]
            return res if single else [res for _ in flist]
        pred = uv = pg = plc = feat = None
        want_streams = any(k in ("pred_sdf_value_global", "pred_sdf_value_local") for k in kinds)
        if "point_img_feat" in kinds:
            if pts is None or tm is None or self._img_key is None and imgs is None:
                raise ValueError("sample_pc / trans_mat / imgs placeholders were not fed")
            feat, _uv = self.engine.point_img_feat(pts, tm)
        if want_streams:
            pred, uv, pg, plc = self.engine.eval_points_ex(pts, tm, pts_rot=rot)
        elif any(k in ("pred_sdf", "sample_img_points") or k.startswith("loss:") for k in kinds):
            if pts is None or tm is None:
                raise ValueError("sample_pc / trans_mat placeholders were not fed")
            if self._img_key is None:        # projection only: any encoded image will do
                self.engine.encode(np.zeros((np.asarray(pts).shape[0], 137, 137, 3), np.float32))
                self._img_key = "zeros"
            pred, uv = self.engine.eval_points(pts, tm, pts_rot=rot, want_uv=True)
        out = []
        for f in flist:
            k = f.kind
            if k == "pred_sdf":
                out.append(pred)
            elif k == "sample_img_points":
                out.append(uv if uv is not None else _uv)
            elif k == "pred_sdf_value_global":
                out.append(pg)
            elif k == "pred_sdf_value_local":
                out.append(plc)
            elif k == "point_img_feat":
                out.append(feat)
            elif k == "ref_img":
                out.append(np.asarray(imgs))
            elif k == "img_embedding":
                out.append(self.engine.get_encoded(0))
            elif k == "resized_ref_img":
                out.append(self.engine.get_encoded(8))
            elif k.startswith("loss:"):
                gt = self._feed(feed_dict, pl.get("sdf"))
                if gt is None:
                    raise ValueError("sdf placeholder was not fed")
                out.append(_loss_metric(k[5:], pred, np.asarray(gt, np.float32), **f.meta))
            else:
                raise NotImplementedError("%s is an intermediate of the reference graph that the fused kernel "
                                          "never materialises" % k)
        return out[0] if single else out


def _loss_metric(name, pred, gt, sdf_weight, mask_weight):
    """models/model_normalization.py:279-291 (host arithmetic on [B,N,1] arrays; not on the hot path)."""
    if name == "accuracy":
        return np.float32(np.mean(((gt > 0) == (pred > 0)).astype(np.float32)))
    if name == "sdf_loss_realvalue":
        return np.float32(np.mean(np.abs(gt - pred / np.float32(sdf_weight))))
    wm = (gt <= 0.01).astype(np.float32) * np.float32(mask_weight) + (gt > 0.01).astype(np.float32)
    return np.float32(np.mean(np.abs(gt * np.float32(sdf_weight) - pred) * wm) * 1000)
