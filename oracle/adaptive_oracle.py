"""NumPy twin of the coarse-to-fine SDF grid (disn_b200/csrc/adaptive.cu, DESIGN.md §4.9).

Given the dense float32 field the network would produce, `refine` returns what the device computes: which points are
evaluated, how many per level, and the filled grid, bit for bit.  `values` is the fill rule at any set of points; the
mesher's twin (oracle/adaptive_mesh_oracle.py) reads its cell corners with it.  Definitions (shared with the kernel):
  * s0 = the largest power of two <= 16 that divides res; s0 = 1 gives the dense grid.  The stride-s0 lattice is
    evaluated first, then levels s = s0, s0/2, ..., 2;
  * level s classifies the blocks of size s (closed cubes of lattice points, origin a multiple of s): all blocks at the
    first level, afterwards only the children of active parents.  A block is active when its 8 corners are not all on one
    side of iso (marching cubes' v < iso) or some corner has |v - iso| <= tau_s in float32, with
    tau_s = float32(band * (s/2) * sqrt(hx^2 + hy^2 + hz^2)) in float64 and h = (max - min) / res per axis;
  * the stride-s/2 points of the active blocks that are not yet evaluated are the level's points (ascending linear index);
  * fill: a point never evaluated is the trilinear interpolation (x, then y, then z; (1-t)*a + t*b with float32 rounding
    per operation) of the corners of the finest classified inactive block that contains it; among several such blocks of
    one level, the first in (z, y, x) order, each axis trying the block that starts at or below the point first.
"""
from __future__ import annotations

import math

import numpy as np


def coarse_stride(res: int) -> int:
    """s0: the largest power of two <= 16 that divides res (1: no refinement, the dense grid)."""
    s = 16
    while s > 1 and res % s:
        s //= 2
    return s


def tau(band: float, s: int, sdf_params, res: int) -> np.float32:
    """Activity threshold of level s: band * (s/2) * |h| in float64, rounded to float32."""
    p = [float(v) for v in sdf_params]
    hx, hy, hz = (p[3] - p[0]) / res, (p[4] - p[1]) / res, (p[5] - p[2]) / res
    with np.errstate(over="ignore"):
        return np.float32(float(band) * (s // 2) * math.sqrt(hx * hx + hy * hy + hz * hz))


def _lerp(t, a, b):
    one = np.float32(1)
    return (one - t) * a + t * b


def classify(field, s: int, iso, t, parent=None):
    """Block states of level s: 0 = not classified (its parent is not active), 1 = inactive, 2 = active."""
    res = field.shape[0] - 1
    nb = res // s
    V = field[::s, ::s, ::s]
    iso = np.float32(iso)
    below = np.zeros((nb, nb, nb), np.int32)
    near = np.zeros((nb, nb, nb), bool)
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                c = V[dz:dz + nb, dy:dy + nb, dx:dx + nb]
                below += c < iso
                near |= np.abs(c - iso) <= t
    active = ((below != 0) & (below != 8)) | near
    if parent is None:
        classified = np.ones_like(active)
    else:
        classified = parent.repeat(2, 0).repeat(2, 1).repeat(2, 2) == 2
    return np.where(classified, np.where(active, 2, 1), 0).astype(np.uint8)


def refine(field, sdf_params, iso: float = 0.0, band: float = 1.0, want_states: bool = False):
    """field: dense float32 [R,R,R] (z, y, x) -> (evaluated mask bool [R,R,R], points per level [coarse, level s0, ...,
    level 2], filled float32 grid) and, with want_states, the (s, block states) of every level."""
    F = np.ascontiguousarray(field, np.float32)
    R = F.shape[0]
    res = R - 1
    s0 = coarse_stride(res)
    if s0 == 1:
        out = (np.ones(F.shape, bool), [R ** 3], F.copy())
        return out + ([],) if want_states else out
    mask = np.zeros(F.shape, bool)
    mask[::s0, ::s0, ::s0] = True
    counts = [int(mask.sum())]
    states = []
    parent = None
    s = s0
    while s >= 2:
        nb = res // s
        st = classify(F, s, iso, tau(band, s, sdf_params, res), parent)
        h = s // 2
        lat = np.zeros((2 * nb + 1,) * 3, bool)
        act = st == 2
        for a in range(3):
            for b in range(3):
                for c in range(3):
                    lat[a:a + 2 * nb:2, b:b + 2 * nb:2, c:c + 2 * nb:2] |= act
        sub = mask[::h, ::h, ::h]                  # a view: updating it marks the points evaluated
        counts.append(int((lat & ~sub).sum()))
        sub |= lat
        states.append((s, st))
        parent = st
        s //= 2
    z, y, x = np.unravel_index(np.arange(F.size), F.shape)
    out = values(F, mask, states, res, z, y, x).reshape(F.shape)
    return (mask, counts, out, states) if want_states else (mask, counts, out)


def values(F, mask, states, res, z, y, x):
    """Values of the dense adaptive grid at points (z, y, x): F where evaluated (mask), else the trilinear fill of the
    finest classified inactive block, first candidate in (z, y, x) order (the fill rule)."""
    z, y, x = (np.asarray(v, np.int64) for v in (z, y, x))
    out = np.empty(len(z), np.float32)
    ev = mask[z, y, x]
    out[ev] = F[z[ev], y[ev], x[ev]]
    todo = np.flatnonzero(~ev)
    zz, yy, xx = z[todo], y[todo], x[todo]
    done = np.zeros(len(todo), bool)
    for s, st in reversed(states):                 # finest level first
        nb = res // s
        cand = []
        for c in (zz, yy, xx):
            q0 = c // s
            v0 = q0 < nb
            v1 = (c % s == 0) & (q0 >= 1)
            cand.append(((np.where(v0, q0, q0 - 1), q0 - 1), v0.astype(np.int64) + v1))
        (cz, kz), (cy, ky), (cx, kx) = cand
        for a in (0, 1):
            for b in (0, 1):
                for d in (0, 1):
                    ok = ~done & (a < kz) & (b < ky) & (d < kx)
                    if not ok.any():
                        continue
                    qz, qy, qx = cz[a][ok], cy[b][ok], cx[d][ok]
                    hit = st[qz, qy, qx] == 1
                    sel = np.flatnonzero(ok)[hit]
                    if not len(sel):
                        continue
                    oz, oy, ox = qz[hit] * s, qy[hit] * s, qx[hit] * s
                    inv = np.float32(1) / np.float32(s)
                    tx = (xx[sel] - ox).astype(np.float32) * inv
                    ty = (yy[sel] - oy).astype(np.float32) * inv
                    tz = (zz[sel] - oz).astype(np.float32) * inv
                    czv = []
                    for kk in (0, 1):
                        zk = oz + kk * s
                        c0 = _lerp(tx, F[zk, oy, ox], F[zk, oy, ox + s])
                        c1 = _lerp(tx, F[zk, oy + s, ox], F[zk, oy + s, ox + s])
                        czv.append(_lerp(ty, c0, c1))
                    out[todo[sel]] = _lerp(tz, czv[0], czv[1])
                    done[sel] = True
    assert done.all(), "a point outside every inactive block was never evaluated"
    return out
