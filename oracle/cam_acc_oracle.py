"""TEST INFRASTRUCTURE ONLY -- float32 restatement of the per-point terms of the camera losses that disn_cam_metrics
sums (cam_est/model_cam.py:111-123 get_img_points, :153-162 get_loss), in the kernel's op order."""
from __future__ import annotations

import numpy as np

CLAMP_MAX = 136.0            # model_cam.py:122, the reference's hard-coded clamp of the projections


def cam_metric_terms(pts, tm, RT, pred_tm, pred_RT):
    """Per-point float32 terms of the camera losses (get_img_points, get_loss) in
    disn_cam_metrics's op order: every product [p, 1] . M summed in k order, one float32 rounding per op.  pts [B,N,3],
    matrices [B,4,3] -> dict of float32 arrays: rotpc [B,N,3] (squares of h.pred_RT - h.RT), rot2d [B,N,2] (squares of
    xy_pred - xy_gt, unclamped), rot3d [B,N] (sqrt of the rotpc row sum), rot2d_dist [B,N] (distance of the [0, 136]
    clamped projections), rotmatrix [B,12] ((pred_tm - tm)^2)."""
    f32 = np.float32
    p = np.asarray(pts, f32)

    def homo(M):
        M = np.asarray(M, f32).reshape(-1, 4, 3)[:, None]
        return ((p[..., 0:1] * M[..., 0, :] + p[..., 1:2] * M[..., 1, :]) + p[..., 2:3] * M[..., 2, :]) + M[..., 3, :]

    sub = homo(pred_RT) - homo(RT)
    sq = sub * sub
    rot3d = np.sqrt((sq[..., 0] + sq[..., 1]) + sq[..., 2])
    u, v = homo(tm), homo(pred_tm)
    xy_gt, xy_pr = u[..., :2] / u[..., 2:3], v[..., :2] / v[..., 2:3]
    d = xy_pr - xy_gt
    clamp = lambda xy: np.minimum(f32(CLAMP_MAX), np.maximum(f32(0), xy))
    c = clamp(xy_gt) - clamp(xy_pr)
    c2 = c * c
    dm = np.asarray(pred_tm, f32).reshape(-1, 12) - np.asarray(tm, f32).reshape(-1, 12)
    out = {"rotpc": sq, "rot2d": d * d, "rot3d": rot3d, "rot2d_dist": np.sqrt(c2[..., 0] + c2[..., 1]),
           "rotmatrix": dm * dm}
    assert all(a.dtype == f32 for a in out.values())
    return out
