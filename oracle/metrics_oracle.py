"""TEST INFRASTRUCTURE ONLY -- CPU oracle of the mesh-evaluation metrics next to the hot path.

nn_distance restates the reference's CPU kernel models/tf_ops/nn_distance/tf_nndistance.cpp:21-43 (`nnsearch`):
for each point of set 1 the minimum over set 2 of the float32 value (dx*dx + dy*dy) + dz*dz, first minimum wins.
It is PINNED against the reference itself: oracle/_ref/libref_nndistance.so is that file compiled in place
(oracle/Makefile, stub TF headers in oracle/ref_stubs) and tests/test_oracle_cpu.py compares the two bit for bit.
Chamfer: test/test_cd_emd.py:300-301; precision/recall/F: test/test_f_score.py:159-186,231-236.

approx_match / match_cost restate models/tf_ops/approxmatch/tf_approxmatch.cpp:23-85 (`approxmatch_cpu`) and :86-107
(`matchcost_cpu`), the approximate earth mover's distance of test/test_cd_emd.py:307-308; pinned the same way against
oracle/_ref/libref_approxmatch.so (tests/test_oracle_cpu.py) and through tests/golden/approxmatch_ref.npz on the GPU box.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(HERE, "_ref", "libref_nndistance.so")
REF_AM_LIB = os.path.join(HERE, "_ref", "libref_approxmatch.so")


def nn_distance(xyz1, xyz2):
    """xyz1 [B,N,3], xyz2 [B,M,3] float32 -> dist1 [B,N] f32, idx1 [B,N] i32, dist2 [B,M], idx2 [B,M]."""
    a = np.ascontiguousarray(xyz1, np.float32)
    b = np.ascontiguousarray(xyz2, np.float32)

    def one_way(p, q):
        d = (p[:, :, None, :] - q[:, None, :, :]).astype(np.float32)        # q - p has the same squares
        s = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]).astype(np.float32) + (d[..., 2] * d[..., 2]).astype(np.float32)
        s = s.astype(np.float32)
        idx = np.argmin(s, axis=2).astype(np.int32)                         # first minimum, like `d < best`
        return np.take_along_axis(s, idx[..., None].astype(np.int64), axis=2)[..., 0], idx

    d1, i1 = one_way(a, b)
    d2, i2 = one_way(b, a)
    return d1, i1, d2, i2


def ref_nn_distance(xyz1, xyz2):
    """The reference's own compiled CPU op (oracle/_ref); raises FileNotFoundError when it was not built."""
    if not os.path.exists(REF_LIB):
        raise FileNotFoundError(REF_LIB)
    lib = C.CDLL(REF_LIB)
    a = np.ascontiguousarray(xyz1, np.float32)
    b = np.ascontiguousarray(xyz2, np.float32)
    B, N, _ = a.shape
    M = b.shape[1]
    d1, i1 = np.empty((B, N), np.float32), np.empty((B, N), np.int32)
    d2, i2 = np.empty((B, M), np.float32), np.empty((B, M), np.int32)
    err = C.create_string_buffer(256)
    rc = lib.ref_nn_distance(B, N, M, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p),
                             d1.ctypes.data_as(C.c_void_p), i1.ctypes.data_as(C.c_void_p),
                             d2.ctypes.data_as(C.c_void_p), i2.ctypes.data_as(C.c_void_p), err, 256)
    if rc:
        raise ValueError(err.value.decode())
    return d1, i1, d2, i2


def approx_match(xyz1, xyz2):
    """tf_approxmatch.cpp:23-85.  xyz1 [B,N,3], xyz2 [B,M,3] float32 -> match [B,N,M] float32 (element (k,l) = mass moved from
    point k of set 1 to point l of set 2; the op declares the shape (B,M,N) but indexes k*m+l, so for N != M the layout is this).
    Eleven rounds j = 8..-2 of a soft assignment with weights expf(-4^j d^2) (level 0 in the last round); every point of set 1
    can give max(N,M)/N units, every point of set 2 can take max(N,M)/M (integer division).  Arithmetic: float32 coordinates
    widened to float64, the exponent rounded to float32, expf in float32, everything else float64, `match` accumulated
    in float32."""
    a = np.ascontiguousarray(xyz1, np.float32).astype(np.float64)
    b = np.ascontiguousarray(xyz2, np.float32).astype(np.float64)
    B, N, _ = a.shape
    M = b.shape[1]
    out = np.zeros((B, N, M), np.float32)
    for i in range(B):
        d2 = ((a[i][:, None, 0] - b[i][None, :, 0]) ** 2 + (a[i][:, None, 1] - b[i][None, :, 1]) ** 2) \
            + (a[i][:, None, 2] - b[i][None, :, 2]) ** 2
        satl = np.full(N, float(max(N, M) // N))
        satr = np.full(M, float(max(N, M) // M))
        for j in range(8, -3, -1):
            level = 0.0 if j == -2 else -float(np.float32(4.0) ** np.float32(j))
            e = np.exp((level * d2).astype(np.float32).astype(np.float64)).astype(np.float32)      # expf of a float32 argument
            w = e.astype(np.float64) * satr[None, :]
            s = 1e-9 + w.sum(axis=1)
            w = w / s[:, None] * satl[:, None]
            ss = 1e-9 + w.sum(axis=0)
            w = w * np.minimum(satr / ss, 1.0)[None, :]
            satl = np.maximum(satl - w.sum(axis=1), 0.0)
            out[i] = (out[i].astype(np.float64) + w).astype(np.float32)
            satr = np.maximum(satr - w.sum(axis=0), 0.0)
    return out


def match_cost(xyz1, xyz2, match):
    """tf_approxmatch.cpp:86-107: cost[b] = sum_kl sqrtf(|p_k - q_l|^2) * match[k,l]; distances and products in float32,
    the sum in float64, the result stored as float32."""
    a = np.ascontiguousarray(xyz1, np.float32)
    b = np.ascontiguousarray(xyz2, np.float32)
    mt = np.ascontiguousarray(match, np.float32)
    d = (b[:, None, :, :] - a[:, :, None, :]).astype(np.float32)
    s = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]).astype(np.float32) + d[..., 2] * d[..., 2]).astype(np.float32)
    t = (np.sqrt(s).astype(np.float32) * mt).astype(np.float32)
    return t.astype(np.float64).sum(axis=(1, 2)).astype(np.float32)


def emd(xyz1, xyz2):
    """test/test_cd_emd.py:307-308: match_cost(src, pred, approx_match(src, pred)) * 0.01 per batch item."""
    return match_cost(xyz1, xyz2, approx_match(xyz1, xyz2)) * np.float32(0.01)


def _ref_am():
    if not os.path.exists(REF_AM_LIB):
        raise FileNotFoundError(REF_AM_LIB)
    return C.CDLL(REF_AM_LIB)


def ref_approx_match(xyz1, xyz2):
    """The reference's own compiled CPU op (oracle/_ref); raises FileNotFoundError when it was not built."""
    lib = _ref_am()
    a = np.ascontiguousarray(xyz1, np.float32)
    b = np.ascontiguousarray(xyz2, np.float32)
    B, N, _ = a.shape
    M = b.shape[1]
    out = np.empty((B, N, M), np.float32)
    err = C.create_string_buffer(256)
    if lib.ref_approx_match(B, N, M, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p),
                            err, 256):
        raise ValueError(err.value.decode())
    return out


def ref_match_cost(xyz1, xyz2, match):
    lib = _ref_am()
    a = np.ascontiguousarray(xyz1, np.float32)
    b = np.ascontiguousarray(xyz2, np.float32)
    mt = np.ascontiguousarray(match, np.float32)
    B, N, _ = a.shape
    M = b.shape[1]
    out = np.empty(B, np.float32)
    err = C.create_string_buffer(256)
    if lib.ref_match_cost(B, N, M, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), mt.ctypes.data_as(C.c_void_p),
                          out.ctypes.data_as(C.c_void_p), err, 256):
        raise ValueError(err.value.decode())
    return out


def chamfer_x1000(pred, src):
    """test/test_cd_emd.py:300-301 -- (mean fwd + mean bwd squared NN distance) * 1000 per batch item."""
    df, _, db, _ = nn_distance(pred, src)
    return (df.mean(axis=1) + db.mean(axis=1)) * np.float32(1000)


def precision_recall_f(pred, src, thresholds):
    """test/test_f_score.py:231-236,185: fractions of sqrt-distances below each threshold, F = 2PR/(P+R)."""
    df, _, db, _ = nn_distance(pred, src)
    th = np.asarray(thresholds, np.float32)[:, None]
    p = (np.sqrt(df).reshape(1, -1) < th).mean(axis=1)
    r = (np.sqrt(db).reshape(1, -1) < th).mean(axis=1)
    return p, r, 2 * p * r / np.maximum(p + r, 1e-30)


# ----------------------------------------------------------------------------------------------------------------------
# IoU (test/test_iou.py:208-233).  pymesh.VoxelGrid is an un-vendored third-party dependency (no pinned version, cannot be
# loaded here): its voxeliser is restated -- cells k are cubes centred at k*cell with half-size cell/2 (PyMesh hash keys
# are round(x / cell_size)), occupied iff they overlap a triangle (closed 13-axis separating-axis test), voxel-mesh
# vertices = the 8 corners of every occupied cell.  The binning expression is the reference's.  PARITY UNPINNED vs PyMesh.
# disn_b200/csrc/iou.cu performs the same float64 operations in the same order, over the same window of cells.
# ----------------------------------------------------------------------------------------------------------------------
def _tri_cube_overlap(c, half, tri):
    """c [M,3] cube centres, tri [3,3] -> bool [M]; closed separating-axis test, same operation order as iou.cu."""
    v = tri[None, :, :] - c[:, None, :]                      # [M,3(vertex),3(axis)]
    ok = np.ones(len(c), bool)
    for a in range(3):
        mn = np.minimum(v[:, 0, a], np.minimum(v[:, 1, a], v[:, 2, a]))
        mx = np.maximum(v[:, 0, a], np.maximum(v[:, 1, a], v[:, 2, a]))
        ok &= ~((mn > half) | (mx < -half))
    e = np.stack([v[:, 1] - v[:, 0], v[:, 2] - v[:, 1], v[:, 0] - v[:, 2]], axis=1)     # [M,3(edge),3]
    nx = e[:, 0, 1] * e[:, 1, 2] - e[:, 0, 2] * e[:, 1, 1]
    ny = e[:, 0, 2] * e[:, 1, 0] - e[:, 0, 0] * e[:, 1, 2]
    nz = e[:, 0, 0] * e[:, 1, 1] - e[:, 0, 1] * e[:, 1, 0]
    d = nx * v[:, 0, 0] + ny * v[:, 0, 1] + nz * v[:, 0, 2]
    ok &= ~(np.abs(d) > half * (np.abs(nx) + np.abs(ny) + np.abs(nz)))

    def sep(ax, ay, az):
        p = [ax * v[:, k, 0] + ay * v[:, k, 1] + az * v[:, k, 2] for k in range(3)]
        r = half * (np.abs(ax) + np.abs(ay) + np.abs(az))
        return (np.minimum(p[0], np.minimum(p[1], p[2])) > r) | (np.maximum(p[0], np.maximum(p[1], p[2])) < -r)

    z = np.zeros(len(c))
    for i in range(3):
        ok &= ~sep(z, -e[:, i, 2], e[:, i, 1])
        ok &= ~sep(e[:, i, 2], z, -e[:, i, 0])
        ok &= ~sep(-e[:, i, 1], e[:, i, 0], z)
    return ok


def voxel_window(dim):
    """(vg, voff): the cells k in [-voff, vg - voff) per axis that iou.cu hashes.  A corner p of a cell lands in a bin iff
    (p + 1.1) / 2.4 * dim is in (-1, dim), so only cells with k * cell in (-1.1 - 2.4/dim - cell/2, 1.3 + cell/2), i.e.
    k in (-(0.55 dim + 1.7), 0.65 dim + 0.5), can contribute; the window covers that with more than a cell to spare."""
    voff, vhi = 11 * dim // 20 + 4, 13 * dim // 20 + 4
    return voff + vhi, voff


def voxel_occupancy(verts, faces, dim=110, vg=None, voff=None):
    """occupancy grid [dim,dim,dim] uint8 of one mesh (the `v1` of test/test_iou.py:215-217).  Cells outside
    [-voff, vg - voff) are skipped; by default the window of voxel_window(dim), which loses no occupied bin."""
    if vg is None:
        vg, voff = voxel_window(dim)
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
        hit = _tri_cube_overlap(ks.astype(np.float64) * cell, cell * 0.5, tri)
        vox.update(map(tuple, ks[hit]))
    occ = np.zeros((dim, dim, dim), np.uint8)
    if vox:
        ks = np.array(sorted(vox), np.float64)
        for corner in np.ndindex(2, 2, 2):
            p = (ks + (np.array(corner) - 0.5)) * cell
            ind = ((p + 1.1) / 2.4 * dim).astype(int)
            ok = np.all((ind >= 0) & (ind < dim), axis=1)
            occ[ind[ok, 0], ind[ok, 1], ind[ok, 2]] = 1
    return occ


def iou_voxel(verts1, faces1, verts2, faces2, dim=110):
    """test/test_iou.py:208-233 iou_pymesh: (intersection, union, iou)."""
    a, b = voxel_occupancy(verts1, faces1, dim), voxel_occupancy(verts2, faces2, dim)
    inter, union = int(np.logical_and(a, b).sum()), int(np.logical_or(a, b).sum())
    return inter, union, (float(inter) / union if union else float("nan"))
