"""TEST INFRASTRUCTURE ONLY -- CPU twin of the CUDA signed distance field (disn_b200/csrc/mesh_sdf.cu).

Reference: preprocessing/create_point_sdf_grid.py:200-210 runs the closed binary isosurface/computeDistanceField
(`<obj> res res res -s -e <expand> -o X.dist -m 1 [-g sigma]`).  PARITY UNPINNED against that binary: it cannot run
here and its polygon-soup pipeline is not restated.  This module defines the field the CUDA path reproduces bit for bit
(DESIGN.md §4.7), brute force in float64, operation for operation:
  * grid: X, Y, Z = np.linspace(lo, hi, R).astype(float32) per axis (disn_eval_grid's tables), layout [z][y][x];
  * d(p) = float32(sqrt(min_f d2(p, f))), d2 from Ericson's closest point on a triangle (Real-Time Collision Detection
    §5.1.5) on the widened float32 coordinates; a face whose float64 cross product is exactly zero counts as its three
    edge segments; a NaN d2 never wins the minimum;
  * a grid edge is blocked when its closed segment crosses a closed face: for every axis a, lines along a through the
    projected face AABB; closed 2D edge-function test with each edge's endpoints in lexicographic (x,y,z) order and the
    value negated when reversed; crossing t = A_a - (n_b (s_b - A_b) + n_c (s_c - A_c)) / n_a (faces with n_a == 0 are
    skipped); every grid edge [G_i, G_i+1] with G_i <= t <= G_i+1 is blocked;
  * wall: d <= sigma; exterior: non-wall points connected to a non-wall boundary point through unblocked edges between
    non-wall points; result +d on exterior points, -d on all others.
"""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


def axes(bbox, R):
    return [np.linspace(bbox[a], bbox[3 + a], R).astype(np.float32) for a in range(3)]


def auto_bbox(verts, expand_rate=1.2):
    """Cube centred on the vertex AABB with side = largest extent * expand_rate."""
    v = np.asarray(verts, np.float32).reshape(-1, 3)
    lo, hi = v.min(axis=0).astype(np.float64), v.max(axis=0).astype(np.float64)
    ext = float(np.max(hi - lo))
    half = ext * expand_rate / 2.0
    c = (lo + hi) / 2.0
    return [float(c[0] - half), float(c[1] - half), float(c[2] - half),
            float(c[0] + half), float(c[1] + half), float(c[2] + half)]


# ---- distance ------------------------------------------------------------------------------------------------------
def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _sub(a, b):
    return [a[0] - b[0], a[1] - b[1], a[2] - b[2]]


def _d2(p, q):
    d = _sub(p, q)
    return _dot(d, d)


def _seg_d2(p, a, b):
    e = _sub(b, a)
    ee = _dot(e, e)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = _dot(_sub(p, a), e) / ee
    t = np.where(t < 0.0, 0.0, np.where(t > 1.0, 1.0, t))
    q = [a[i] + t * e[i] for i in range(3)]
    return np.where(ee == 0.0, _d2(p, a), _d2(p, q))


def _min(a, b):
    return np.where(b < a, b, a)          # NaN in b never wins


def tri_dist2(p, a, b, c):
    """Squared distance, float64.  p: 3 arrays [P,1]; a, b, c: 3 arrays [1,T] (broadcast) -> [P,T]."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        ab, ac = _sub(b, a), _sub(c, a)
        n = [ab[1] * ac[2] - ab[2] * ac[1], ab[2] * ac[0] - ab[0] * ac[2], ab[0] * ac[1] - ab[1] * ac[0]]
        degen = (n[0] == 0.0) & (n[1] == 0.0) & (n[2] == 0.0)
        ap = _sub(p, a)
        d1, d2 = _dot(ab, ap), _dot(ac, ap)
        bp = _sub(p, b)
        d3, d4 = _dot(ab, bp), _dot(ac, bp)
        vc = d1 * d4 - d3 * d2
        cp = _sub(p, c)
        d5, d6 = _dot(ab, cp), _dot(ac, cp)
        vb = d5 * d2 - d1 * d6
        va = d3 * d6 - d5 * d4
        v_ab = d1 / (d1 - d3)
        w_ac = d2 / (d2 - d6)
        w_bc = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        denom = 1.0 / ((va + vb) + vc)
        v, w = vb * denom, vc * denom
        bc = _sub(c, b)
        cands = [
            (d1 <= 0.0) & (d2 <= 0.0), lambda: _d2(p, a),
            (d3 >= 0.0) & (d4 <= d3), lambda: _d2(p, b),
            (vc <= 0.0) & (d1 >= 0.0) & (d3 <= 0.0), lambda: _d2(p, [a[i] + v_ab * ab[i] for i in range(3)]),
            (d6 >= 0.0) & (d5 <= d6), lambda: _d2(p, c),
            (vb <= 0.0) & (d2 >= 0.0) & (d6 <= 0.0), lambda: _d2(p, [a[i] + w_ac * ac[i] for i in range(3)]),
            (va <= 0.0) & ((d4 - d3) >= 0.0) & ((d5 - d6) >= 0.0),
            lambda: _d2(p, [b[i] + w_bc * bc[i] for i in range(3)]),
        ]
        out = _d2(p, [(a[i] + ab[i] * v) + ac[i] * w for i in range(3)])     # interior
        for k in range(len(cands) - 2, -1, -2):                                 # first region wins: apply in reverse
            out = np.where(cands[k], cands[k + 1](), out)
        if degen.any():
            seg = _min(_min(_seg_d2(p, a, b), _seg_d2(p, b, c)), _seg_d2(p, c, a))
            out = np.where(degen, seg, out)
    return out


def unsigned_distance(verts, faces, pts, chunk=1 << 22):
    """Brute-force d (float32) of float32 points [P,3] to the mesh."""
    v = np.asarray(verts, np.float32).reshape(-1, 3).astype(np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    P = np.asarray(pts, np.float32).reshape(-1, 3).astype(np.float64)
    T = len(f)
    A, B, Cc = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    best = np.full(len(P), np.inf)
    step_p = max(1, chunk // max(T, 1))
    for s in range(0, len(P), step_p):
        p = [P[s:s + step_p, i:i + 1] for i in range(3)]
        for t0 in range(0, T, chunk):
            sl = slice(t0, t0 + chunk)
            d2 = tri_dist2(p, [A[None, sl, i] for i in range(3)], [B[None, sl, i] for i in range(3)],
                           [Cc[None, sl, i] for i in range(3)])
            with np.errstate(invalid="ignore"):
                m = np.fmin.reduce(d2, axis=1)      # the minimum is order-free; a NaN d2 never wins
            best[s:s + step_p] = _min(best[s:s + step_p], m)
    return np.sqrt(best).astype(np.float32)


def grid_points(bbox, R):
    X, Y, Z = axes(bbox, R)
    z, y, x = np.meshgrid(Z, Y, X, indexing="ij")
    return np.stack([x.reshape(-1), y.reshape(-1), z.reshape(-1)], axis=1)


def band_distance(verts, faces, bbox, R, r):
    """d on the grid, exact wherever it is <= r (inf where it is certainly > r): every face is evaluated only against the
    grid points inside its AABB dilated by r (plus a relative slack far above the rounding of the computed distance)."""
    G = [g.astype(np.float64) for g in axes(bbox, R)]
    v = np.asarray(verts, np.float32).reshape(-1, 3).astype(np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    best = np.full(R ** 3, np.inf)
    m = r * (1 + 2.0 ** -20) + 2.0 ** -24 * max(1.0, float(np.abs(v).max()), max(abs(x) for x in bbox))
    for tri in f:
        t = v[tri]
        lo, hi = t.min(axis=0) - m, t.max(axis=0) + m
        rng = [np.arange(np.searchsorted(G[a], lo[a], "left"), np.searchsorted(G[a], hi[a], "right")) for a in range(3)]
        if any(len(q) == 0 for q in rng):
            continue
        zi, yi, xi = np.meshgrid(rng[2], rng[1], rng[0], indexing="ij")
        idx = ((zi * R + yi) * R + xi).reshape(-1)
        p = [G[0][xi.reshape(-1)][:, None], G[1][yi.reshape(-1)][:, None], G[2][zi.reshape(-1)][:, None]]
        d2 = tri_dist2(p, *[[t[k, i:i + 1][None, :] for i in range(3)] for k in range(3)])[:, 0]
        best[idx] = _min(best[idx], d2)
    d = np.sqrt(best).astype(np.float32)
    d[d > np.float32(r)] = np.inf
    return d


# ---- blocked edges ----------------------------------------------------------------------------------------------------
def _lex_less(p, q):
    return (p[0] < q[0]) | ((p[0] == q[0]) & ((p[1] < q[1]) | ((p[1] == q[1]) & (p[2] < q[2]))))


def _edge_fn(P, Q, b, c, sb, sc):
    rev = _lex_less(Q, P)
    u = [np.where(rev, Q[i], P[i]) for i in range(3)]
    w = [np.where(rev, P[i], Q[i]) for i in range(3)]
    e = (w[b] - u[b]) * (sc - u[c]) - (w[c] - u[c]) * (sb - u[b])
    return np.where(rev, -e, e)


def blocked_edges(verts, faces, bbox, R):
    """uint8 [R^3]: bit a set when the grid edge from the point along +a is blocked."""
    G32 = axes(bbox, R)
    G = [g.astype(np.float64) for g in G32]
    v32 = np.asarray(verts, np.float32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    tri32 = v32[f]                                   # [F,3 vertices,3 coords]
    tri = tri32.astype(np.float64)
    A, B, C = tri[:, 0], tri[:, 1], tri[:, 2]
    n = np.stack([(B - A)[:, 1] * (C - A)[:, 2] - (B - A)[:, 2] * (C - A)[:, 1],
                  (B - A)[:, 2] * (C - A)[:, 0] - (B - A)[:, 0] * (C - A)[:, 2],
                  (B - A)[:, 0] * (C - A)[:, 1] - (B - A)[:, 1] * (C - A)[:, 0]], axis=1)
    bits = np.zeros(R ** 3, np.uint8)
    for a in range(3):
        b, c = (a + 1) % 3, (a + 2) % 3
        j0 = np.searchsorted(G[b], tri32[:, :, b].min(axis=1).astype(np.float64), "left")
        j1 = np.searchsorted(G[b], tri32[:, :, b].max(axis=1).astype(np.float64), "right")
        k0 = np.searchsorted(G[c], tri32[:, :, c].min(axis=1).astype(np.float64), "left")
        k1 = np.searchsorted(G[c], tri32[:, :, c].max(axis=1).astype(np.float64), "right")
        nj, nk = np.maximum(j1 - j0, 0), np.maximum(k1 - k0, 0)
        cnt = np.where(n[:, a] != 0.0, nj * nk, 0)
        fi = np.repeat(np.arange(len(f)), cnt)
        if len(fi) == 0:
            continue
        local = np.arange(len(fi)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        j = j0[fi] + local % nj[fi]
        k = k0[fi] + local // nj[fi]
        sb, sc = G[b][j], G[c][k]
        P = [A[fi, i] for i in range(3)]
        Q = [B[fi, i] for i in range(3)]
        S = [C[fi, i] for i in range(3)]
        e0 = _edge_fn(Q, S, b, c, sb, sc)
        e1 = _edge_fn(S, P, b, c, sb, sc)
        e2 = _edge_fn(P, Q, b, c, sb, sc)
        inside = ((e0 >= 0) & (e1 >= 0) & (e2 >= 0)) | ((e0 <= 0) & (e1 <= 0) & (e2 <= 0))
        fi, j, k, sb, sc = fi[inside], j[inside], k[inside], sb[inside], sc[inside]
        t = A[fi, a] - (n[fi, b] * (sb - A[fi, b]) + n[fi, c] * (sc - A[fi, c])) / n[fi, a]
        i0 = np.maximum(np.searchsorted(G[a], t, "left") - 1, 0)
        i1 = np.minimum(np.searchsorted(G[a], t, "right") - 1, R - 2)
        reps = np.maximum(i1 - i0 + 1, 0)
        ii = np.repeat(i0, reps) + (np.arange(reps.sum()) - np.repeat(np.cumsum(reps) - reps, reps))
        q = [None, None, None]
        q[a], q[b], q[c] = ii, np.repeat(j, reps), np.repeat(k, reps)
        idx = (q[2].astype(np.int64) * R + q[1]) * R + q[0]
        bits[idx] |= np.uint8(1 << a)
    return bits


def exterior(d, bits, R, sigma):
    """bool [R^3]: non-wall points connected to a non-wall boundary point through open edges."""
    free = ~(d.astype(np.float64) <= sigma)
    idx = np.arange(R ** 3).reshape(R, R, R)
    rows, cols = [], []
    for a, sl in enumerate([(slice(None), slice(None), slice(0, R - 1)), (slice(None), slice(0, R - 1), slice(None)),
                            (slice(0, R - 1), slice(None), slice(None))]):
        i = idx[sl].reshape(-1)
        j = i + (1, R, R * R)[a]
        ok = free[i] & free[j] & ((bits[i] >> a) & 1 == 0)
        rows.append(i[ok])
        cols.append(j[ok])
    r, c = np.concatenate(rows), np.concatenate(cols)
    g = coo_matrix((np.ones(len(r), np.int8), (r, c)), shape=(R ** 3, R ** 3))
    _, lab = connected_components(g, directed=False)
    bnd = np.zeros((R, R, R), bool)
    bnd[0], bnd[-1], bnd[:, 0], bnd[:, -1], bnd[:, :, 0], bnd[:, :, -1] = (True,) * 6
    bnd = bnd.reshape(-1) & free
    reached = np.zeros(lab.max() + 1, bool)
    reached[lab[bnd]] = True
    return free & reached[lab]


def mesh_sdf(verts, faces, res, bbox=None, expand_rate=1.2, sigma=0.0, dist=None):
    """-> (float32 [R,R,R] signed field, bbox).  dist: precomputed unsigned grid distances (default brute force)."""
    R = res + 1
    bbox = auto_bbox(verts, expand_rate) if bbox is None else [float(x) for x in bbox]
    d = unsigned_distance(verts, faces, grid_points(bbox, R)) if dist is None else np.asarray(dist, np.float32).reshape(-1)
    ext = exterior(d, blocked_edges(verts, faces, bbox, R), R, sigma)
    return np.where(ext, d, -d).astype(np.float32).reshape(R, R, R), bbox


def sign_from_band(verts, faces, res, bbox, sigma=0.0):
    """Exterior mask [R^3] needing distances only where they can be <= sigma (large grids)."""
    R = res + 1
    d = band_distance(verts, faces, bbox, R, sigma)
    return exterior(d, blocked_edges(verts, faces, bbox, R), R, sigma)


def winding_number(verts, faces, pts, chunk=1 << 22):
    """Generalised winding number (Jacobson et al. 2013, solid angles by Van Oosterom & Strackee), float64."""
    v = np.asarray(verts, np.float64).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    P = np.asarray(pts, np.float64).reshape(-1, 3)
    out = np.zeros(len(P))
    step = max(1, chunk // max(len(f), 1))
    for s in range(0, len(P), step):
        p = P[s:s + step, None, :]
        a, b, c = v[f[:, 0]][None] - p, v[f[:, 1]][None] - p, v[f[:, 2]][None] - p
        la, lb, lc = (np.linalg.norm(x, axis=2) for x in (a, b, c))
        det = np.einsum("pti,pti->pt", a, np.cross(b, c))
        den = la * lb * lc + np.einsum("pti,pti->pt", a, b) * lc + np.einsum("pti,pti->pt", b, c) * la \
            + np.einsum("pti,pti->pt", c, a) * lb
        out[s:s + step] = (2.0 * np.arctan2(det, den)).sum(axis=1) / (4.0 * np.pi)
    return out
