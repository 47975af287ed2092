"""TEST INFRASTRUCTURE ONLY -- CPU twins of the CUDA surface-sample normalisation (disn_b200/csrc/mesh_normalize.cu) and
of the band / strided field samplers (disn_b200/csrc/sdf_sample.cu).

Reference: preprocessing/create_point_sdf_grid.py:169-198 get_normalize_mesh (trimesh.sample.sample_surface per part,
np.mean centroid, max norm, (v - c) / m) and :74-113 sample_sdf; create_point_sdf_fullgrid.py:70-96.  The definitions
below (DESIGN.md §4.8) are what the CUDA path reproduces bit for bit; they differ from trimesh only where trimesh's float
cumulative areas put a pick on a different face (unpinned: trimesh is not installed) and in the fixed-point centroid, whose
distance from np.mean is bounded in tests/test_mesh_norm_cpu.py:
  * a_f = 0.5 * sqrt((cx*cx + cy*cy) + cz*cz), c = (v1 - v0) x (v2 - v0), float64 on the widened float32 vertices;
  * Q_f = rint(a_f * 2^s) (int64), s = 62 - frexp(a_max * n_faces)[1] (0 when a_max = 0); faces scanned in part order;
  * n_p = Q_p * total // sum Q (exact integers);
  * pick k = floor(u * 2^53), t = k * Q_p >> 53 (Python ints), face = first of part p with cumulative Q > t;
  * r1, r2: if r1 + r2 > 1 both minus 1, then abs; p = (e1 * r1 + e2 * r2) + v0;
  * c = (float(S) / N) * 2^-32 with S = sum rint(p * 2^32); m = max sqrt((dx*dx + dy*dy) + dz*dz);
  * vertices -> float32((v - c) / m).
"""
import math

import numpy as np

TOTAL = 16384


def face_areas(verts, faces):
    v = np.asarray(verts, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64)
    v0, v1, v2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    e1, e2 = v1 - v0, v2 - v0
    cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    return 0.5 * np.sqrt((cx * cx + cy * cy) + cz * cz)


def shift_for(a_max, n_faces):
    return 62 - math.frexp(float(a_max) * float(n_faces))[1] if a_max > 0 else 0


def part_scan(verts, faces, part_ids=None, n_parts=1):
    """-> dict(q=part totals (Python ints), shift, order (faces in part order), incl (int64 inclusive scan in that
    order), start (part offsets into order), areas)."""
    a = face_areas(verts, faces)
    nf = len(a)
    pid = np.zeros(nf, np.int64) if part_ids is None else np.asarray(part_ids, np.int64)
    if len(pid) and (pid.min() < 0 or pid.max() >= n_parts):
        raise ValueError("part id out of range")
    s = shift_for(a.max() if nf else 0.0, nf)
    order = np.argsort(pid, kind="stable")
    q = np.rint(np.ldexp(a[order], s)).astype(np.int64)
    incl = np.cumsum(q)
    start = np.concatenate([[0], np.cumsum(np.bincount(pid, minlength=n_parts))]).astype(np.int64)
    tot = [int(incl[start[p + 1] - 1]) - (int(incl[start[p] - 1]) if start[p] else 0) if start[p + 1] > start[p] else 0
           for p in range(n_parts)]
    return dict(q=tot, shift=s, order=order, incl=incl, start=start, areas=a)


def amounts(part_q, total=TOTAL):
    q = [int(x) for x in part_q]
    qs = sum(q)
    return [x * total // qs if qs else 0 for x in q]


def sample(verts, faces, scan, amts, draws):
    """Surface samples [N,3] float64 for the draws [N,3] = (pick, r1, r2), parts in order."""
    v = np.asarray(verts, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64)
    draws = np.asarray(draws, np.float64).reshape(-1, 3)
    incl, start, order = scan["incl"], scan["start"], scan["order"]
    face = np.empty(len(draws), np.int64)
    j = 0
    for p, n in enumerate(amts):
        if n == 0:
            continue
        Q = scan["q"][p]
        b, e = int(start[p]), int(start[p + 1])
        base = int(incl[b - 1]) if b else 0
        T = np.array([base + ((int(u * 2.0 ** 53) * Q) >> 53) for u in draws[j:j + n, 0]], np.int64)
        face[j:j + n] = order[b + np.searchsorted(incl[b:e], T, side="right")]
        j += n
    v0, v1, v2 = v[f[face, 0]], v[f[face, 1]], v[f[face, 2]]
    r1, r2 = draws[:, 1:2].copy(), draws[:, 2:3].copy()
    flip = (r1 + r2 > 1.0)
    r1[flip] -= 1.0
    r2[flip] -= 1.0
    r1, r2 = np.abs(r1), np.abs(r2)
    return ((v1 - v0) * r1 + (v2 - v0) * r2) + v0, face


def centroid_radius(samples):
    p = np.asarray(samples, np.float64)
    N = len(p)
    if np.abs(p).max() * N >= 2.0 ** 30:
        raise ValueError("int64 range of the fixed-point sums")
    S = [int(x) for x in np.rint(p * 2.0 ** 32).astype(np.int64).sum(axis=0, dtype=np.int64)]
    c = np.array([(float(s) / N) * 2.0 ** -32 for s in S])
    d = p - c
    m = float(np.max(np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])))
    return c, m


def transform(verts, c, m):
    return ((np.asarray(verts, np.float32).astype(np.float64) - np.asarray(c, np.float64)) / float(m)).astype(np.float32)


def normalize(verts, faces, part_ids, n_parts, amts, draws):
    """-> (centroid [3] float64, m, samples [N,3] float64, normalised vertices float32)."""
    scan = part_scan(verts, faces, part_ids, n_parts)
    pts, _ = sample(verts, faces, scan, amts, draws)
    c, m = centroid_radius(pts)
    return c, m, pts, transform(verts, c, m)


# ---- field samplers ----------------------------------------------------------------------------------------------------
def band_edges(bandwidth):
    """(lo, hi) of sample_sdf's four bands as float32, the thresholds numpy 2 compares a float32 array against."""
    bw = bandwidth
    e = [[-1. * bw, -1. * bw * 0.30], [-1. * bw * 0.30, 0], [0, bw * 0.30], [bw * 0.30, bw]]
    return np.array(e, np.float64).astype(np.float32)


def band_lists(sdf, iso, edges):
    dis = np.asarray(sdf, np.float32).reshape(-1) - np.float32(iso)
    return [np.nonzero((dis >= lo) & (dis < hi))[0] for lo, hi in edges]


def band_gather(sdf, R, axes, lists, choices, k):
    vals = np.asarray(sdf, np.float32).reshape(-1)
    idx = np.concatenate([lists[b][np.asarray(choices[b], np.int64)] for b in range(4) if k[b]] or [np.zeros(0, np.int64)])
    x, y, z = axes
    return np.stack([x[idx % R], y[(idx // R) % R], z[idx // (R * R)], vals[idx]], axis=1).astype(np.float32)


def sample_sdf(num_sample, bandwidth, iso, params, sdf_res, sdf):
    """The device band sampler's whole path on the twins: lists -> carry-over rule and np.random.randint on the host ->
    gather (the tables the host sample_sdf builds from the float32 params)."""
    R = sdf_res + 1
    lists = band_lists(sdf, iso, band_edges(bandwidth))
    want = [int(num_sample * 0.25)] * 4
    k, choices = [0] * 4, [None] * 4
    for i in range(4):
        n = len(lists[i])
        if n < want[i]:
            if i < 3:
                want[i + 1] += want[i] - n
            want[i] = n
        if n == 0:
            continue
        choices[i] = np.random.randint(n, size=want[i])
        k[i] = want[i]
    p = np.asarray(params, np.float32)
    axes = [np.linspace(p[a], p[3 + a], num=R).astype(np.float32) for a in range(3)]
    return band_gather(sdf, R, axes, lists, choices, k)


def strided(sdf, reduce):
    return np.ascontiguousarray(np.asarray(sdf, np.float32)[::reduce, ::reduce, ::reduce])
