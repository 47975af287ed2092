"""TEST INFRASTRUCTURE ONLY -- CPU twin of the CUDA small-part cleaning (disn_b200/csrc/mesh_clean.cu).

Reference: postprocessing/clean_smallparts.py:38-54 (clean_single_mesh): pymesh.separate_mesh(connectivity_type='auto'),
keep a component iff len(vertices) > max_len * num_thresh and |mean(vertices)| < dist_thresh, pymesh.merge_meshes.

PARITY UNPINNED against PyMesh (not installed; its semantics are restated from its documentation):
  * components: two faces are connected when they share an undirected edge {a,b}, a != b ('auto' == 'face' for a
    triangle surface mesh); a bow-tie vertex does not connect; a degenerate face connects through its non-degenerate
    edges only.  Numbered here in order of their smallest face index (PyMesh's own order is not mirrored).
  * n_c = number of distinct vertices referenced by the faces of c (unreferenced vertices belong to no component).
  * centroid = ((double)S / n_c) * 2^-32, S = int64 sum of rint(v * 2^32) over those vertices: exact integer sums,
    within 2^-33 of a float64 np.mean; norm = sqrt((x*x + y*y) + z*z).
  * the result holds the kept faces and the vertices they reference, both in their original order, faces renumbered;
    a vertex shared by two kept components appears once (merge_meshes would duplicate it, component by component).
Bit-for-bit definition the CUDA path reproduces (faces, vertices, per-face labels, component and kept counts).
"""
import numpy as np

COORD_LIMIT = 2.0 ** 30      # refuse max|v| * n_verts >= 2^30: the int64 sums could overflow


def components(faces, n_verts):
    """Per-face component label (dense, ordered by smallest face index) and the component count."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    F = len(f)
    if F == 0:
        return np.zeros(0, np.int32), 0
    a = np.concatenate([f[:, 0], f[:, 1], f[:, 2]])
    b = np.concatenate([f[:, 1], f[:, 2], f[:, 0]])
    fid = np.tile(np.arange(F, dtype=np.int64), 3)
    m = a != b
    a, b, fid = a[m], b[m], fid[m]
    key = np.minimum(a, b) * np.int64(max(n_verts, 1)) + np.maximum(a, b)
    order = np.argsort(key, kind="stable")
    key, fid = key[order], fid[order]
    same = key[1:] == key[:-1]
    u, v = fid[:-1][same], fid[1:][same]          # consecutive faces on one edge: enough for connectivity
    # hook-and-shortcut label propagation: hook every edge's larger root under the smaller, then jump pointers to roots
    L = np.arange(F, dtype=np.int64)
    while True:
        lu, lv = L[u], L[v]
        d = lu != lv
        if not d.any():
            break
        lo, hi = np.minimum(lu[d], lv[d]), np.maximum(lu[d], lv[d])
        np.minimum.at(L, hi, lo)
        while True:
            nxt = L[L]
            if np.array_equal(nxt, L):
                break
            L = nxt
    root = L == np.arange(F)
    dense = np.cumsum(root) - root
    return dense[L].astype(np.int32), int(root.sum())


def clean(verts, faces, dist_thresh=0.5, num_thresh=0.3):
    """-> dict(verts [V,3] float32, faces [F,3] int32, labels [F_in] int32, n_components, n_kept, counts, centroids)."""
    v = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
    f = np.ascontiguousarray(faces, np.int32).reshape(-1, 3)
    nv = len(v)
    if len(f) and (f.min() < 0 or f.max() >= nv):
        raise ValueError("face index outside [0, %d)" % nv)
    empty = dict(verts=np.zeros((0, 3), np.float32), faces=np.zeros((0, 3), np.int32), labels=np.zeros(0, np.int32),
                 n_components=0, n_kept=0, counts=np.zeros(0, np.int64), centroids=np.zeros((0, 3)))
    if len(f) == 0:
        return empty
    maxabs = float(np.abs(v).max())
    if not maxabs * nv < COORD_LIMIT:
        raise ValueError("max |coordinate| * n_verts = %r must stay below 2^30" % (maxabs * nv))
    labels, C = components(f, nv)
    # distinct (component, vertex) pairs, sorted by component then vertex
    pair = np.unique(np.repeat(labels.astype(np.int64), 3) * nv + f.reshape(-1).astype(np.int64))
    pc, pv = pair // nv, pair % nv
    starts = np.searchsorted(pc, np.arange(C))
    counts = np.diff(np.append(starts, len(pair)))
    q = np.rint(v.astype(np.float64) * 2.0 ** 32).astype(np.int64)
    S = np.add.reduceat(q[pv], starts, axis=0)
    cen = (S.astype(np.float64) / counts.astype(np.float64)[:, None]) * 2.0 ** -32
    norm = np.sqrt((cen[:, 0] * cen[:, 0] + cen[:, 1] * cen[:, 1]) + cen[:, 2] * cen[:, 2])
    keep = (counts.astype(np.float64) > np.float64(counts.max()) * np.float64(num_thresh)) & (norm < dist_thresh)
    fk = keep[labels]
    vk = np.zeros(nv, bool)
    vk[f[fk].reshape(-1)] = True
    vmap = np.cumsum(vk) - vk
    return dict(verts=v[vk], faces=vmap[f[fk]].astype(np.int32), labels=labels, n_components=C,
                n_kept=int(keep.sum()), counts=counts, centroids=cen)
