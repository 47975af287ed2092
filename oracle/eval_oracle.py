"""TEST INFRASTRUCTURE ONLY -- CPU stand-in for the Engine methods the evaluation drivers call (disn_b200/eval_cd_emd.py,
eval_f_score.py, eval_iou.py): points_loss, nn_distance, iou and iou_views, built on oracle/metrics_oracle.py with the
arithmetic of the CUDA path (Engine.points_loss's reductions; the voxeliser's float64 operations).  Tests hand it to a
driver by replacing the driver's module-level _engine().

voxel_cells / voxel_mesh_vertices give the occupied cells and the voxel mesh's vertices of the restated
pymesh.VoxelGrid, so that tests/golden/make_golden_eval.py can run the reference's own binning line on them.
"""
import numpy as np

from oracle import metrics_oracle as mo


def voxel_cells(verts, faces, dim=110):
    """Occupied cells [K,3] int (sorted) of one mesh at cell 2/dim: metrics_oracle.voxel_occupancy's cell set."""
    vg, voff = mo.voxel_window(dim)
    cell = 2.0 / dim
    V = np.asarray(verts, np.float32).astype(np.float64)
    vox = set()
    for f in np.asarray(faces):
        tri = V[f]
        lo, hi = tri.min(axis=0), tri.max(axis=0)
        k0 = np.clip(np.floor(lo / cell - 0.5), -voff, vg - voff).astype(int)
        k1 = np.clip(np.ceil(hi / cell + 0.5), -voff - 1, vg - voff - 1).astype(int)
        if np.any(k1 < k0):
            continue
        ks = np.stack(np.meshgrid(*[np.arange(k0[a], k1[a] + 1) for a in range(3)], indexing="ij"), axis=-1).reshape(-1, 3)
        hit = mo._tri_cube_overlap(ks.astype(np.float64) * cell, cell * 0.5, tri)
        vox.update(map(tuple, ks[hit]))
    return np.array(sorted(vox), np.int64).reshape(-1, 3)


def voxel_mesh_vertices(verts, faces, dim=110):
    """The 8 corners (k +- 1/2) * cell of every occupied cell, float64 [8K,3], computed as voxel_occupancy does."""
    ks = voxel_cells(verts, faces, dim).astype(np.float64)
    cell = 2.0 / dim
    return np.concatenate([(ks + (np.array(corner) - 0.5)) * cell for corner in np.ndindex(2, 2, 2)]).reshape(-1, 3)


class EvalTwin:
    """The evaluation methods of disn_b200.engine.Engine on the CPU."""

    def nn_distance(self, xyz1, xyz2):
        return mo.nn_distance(xyz1, xyz2)

    def points_loss(self, sampled_pc):
        """Engine.points_loss: Chamfer x1000 and EMD x0.01 of views 1.. against cloud 0; mean, min, argmin of each."""
        pc = np.ascontiguousarray(sampled_pc, np.float32)
        pred = pc[1:]
        src = np.ascontiguousarray(np.broadcast_to(pc[:1], pred.shape))
        cf = mo.chamfer_x1000(pred, src)
        em = mo.match_cost(src, pred, mo.approx_match(src, pred)) * np.float32(0.01)
        return (np.float32(cf.mean()), np.float32(cf.min()), int(cf.argmin()),
                np.float32(em.mean()), np.float32(em.min()), int(em.argmin()))

    def iou(self, verts1, faces1, verts2, faces2, dim=110, want_grids=False):
        a, b = mo.voxel_occupancy(verts1, faces1, dim), mo.voxel_occupancy(verts2, faces2, dim)
        inter, uni = int(np.logical_and(a, b).sum()), int(np.logical_or(a, b).sum())
        val = inter / uni if uni else float("nan")
        return (val, inter, uni, a, b) if want_grids else val

    def iou_views(self, ref_verts, ref_faces, views, dim=110, want_grids=False):
        ref = mo.voxel_occupancy(ref_verts, ref_faces, dim)
        grids = [ref] + [mo.voxel_occupancy(v, f, dim) for v, f in views]
        inter = np.array([np.logical_and(ref, g).sum() for g in grids[1:]], np.int64)
        uni = np.array([np.logical_or(ref, g).sum() for g in grids[1:]], np.int64)
        with np.errstate(invalid="ignore", divide="ignore"):
            val = np.where(uni > 0, inter / np.maximum(uni, 1), np.nan)
        return (val, inter, uni, np.stack(grids)) if want_grids else (val, inter, uni)
