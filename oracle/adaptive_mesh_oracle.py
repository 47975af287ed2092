"""NumPy twin of the coarse-to-fine mesher (disn_b200/csrc/adaptive_mesh.cu, DESIGN.md §4.10).

It builds the mesh from the refinement's block states and evaluated values alone (never from the dense filled grid of
oracle/adaptive_oracle.refine): the candidate cells K, their corner values by the fill rule, the crossing edges sorted
by edge id, faces cell by cell in table order.  The result must equal mc_oracle.marching_cubes of the dense adaptive grid
bit for bit.  K is the union of
  (i)   every cell of an active block of the last level (s = 2);
  (ii)  every cell of an inactive block (any level s) with a corner in an active block of level s;
  (iii) every cell of an inactive block with a corner v such that |v - iso| <= max|corner| * 2^-21 + 2^-126 (float64):
        only there can the fill's roundings put an interpolated value on the other side of iso than its corners (at
        iso = 0, corners of -2^-149 interpolate to -0, which is not below 0).
"""
from __future__ import annotations

import numpy as np

from oracle import adaptive_oracle as ao
from oracle import mc_oracle as mo


def _cells(block, s):
    return block.repeat(s, 0).repeat(s, 1).repeat(s, 2)


def candidates(F, states, res, iso, rule_ii: bool = True, rule_iii: bool = True):
    """K as a bool array over the cells [res, res, res] (cell = unit cube at its lowest corner (z, y, x)); rule_ii /
    rule_iii = False leave those rules out (negative controls)."""
    K = np.zeros((res,) * 3, bool)
    iso64 = np.float64(np.float32(iso))
    for li, (s, st) in enumerate(states):
        nb = res // s
        act, inact = st == 2, st == 1
        if li == len(states) - 1:
            K |= _cells(act, s)                                               # (i)
        V = F[::s, ::s, ::s].astype(np.float64)                               # block corners (evaluated)
        corners = [V[dz:dz + nb, dy:dy + nb, dx:dx + nb] for dz in (0, 1) for dy in (0, 1) for dx in (0, 1)]
        amax = np.max(np.abs(corners), axis=0)
        margin = amax * 2.0 ** -21 + 2.0 ** -126
        near = np.any([np.abs(c - iso64) <= margin for c in corners], axis=0)
        if rule_iii:
            K |= _cells(inact & near, s)                                      # (iii)
        if not rule_ii:
            continue
        loc = np.arange(res) % s
        pad = np.pad(act, 1)
        for dz in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    if dz == dy == dx == 0:
                        continue
                    nact = pad[1 + dz:1 + dz + nb, 1 + dy:1 + dy + nb, 1 + dx:1 + dx + nb]
                    allow = [(d == 0) | ((d == -1) & (loc == 0)) | ((d == 1) & (loc == s - 1)) for d in (dz, dy, dx)]
                    K |= _cells(inact & nact, s) & allow[0][:, None, None] & allow[1][None, :, None] \
                        & allow[2][None, None, :]                             # (ii)
    return K


def mesh(field, sdf_params, iso: float = 0.0, band: float = 1.0, rule_ii: bool = True, rule_iii: bool = True,
         want_K: bool = False):
    """-> (verts float32 [V,3], faces int32 [F,3], level counts) and, with want_K, the candidate cells K."""
    F = np.ascontiguousarray(field, np.float32)
    R = F.shape[0]
    res = R - 1
    mask, counts, _, states = ao.refine(F, sdf_params, iso=iso, band=band, want_states=True)
    if ao.coarse_stride(res) == 1:                 # the dense grid
        v, f = mo.marching_cubes(F, sdf_params, iso)
        return (v, f, counts, np.ones((res,) * 3, bool)) if want_K else (v, f, counts)
    K = candidates(F, states, res, iso, rule_ii, rule_iii)
    cz, cy, cx = (v.astype(np.int64) for v in np.nonzero(K))          # ascending cell id
    iso32 = np.float32(iso)
    case = np.zeros(len(cz), np.int64)
    for k in range(8):
        v = ao.values(F, mask, states, res, cz + (k >> 2 & 1), cy + (k >> 1 & 1), cx + (k & 1))
        case |= (v < iso32).astype(np.int64) << k
    nt = mo.NTRI[case]
    keep = nt > 0
    cz, cy, cx, case, nt = cz[keep], cy[keep], cx[keep], case[keep], nt[keep]
    ids = []
    for e in range(12):
        ax, dx, dy, dz = (int(v) for v in mo.EDGE[e])
        k0 = dx + 2 * dy + 4 * dz
        cross = ((case >> k0) ^ (case >> (k0 + (1 << ax)))) & 1 == 1
        ids.append((((cz[cross] + dz) * R + (cy[cross] + dy)) * R + (cx[cross] + dx)) * 3 + ax)
    E = np.unique(np.concatenate(ids)) if ids else np.zeros(0, np.int64)
    a = E % 3
    q = E // 3
    x, y, z = q % R, (q // R) % R, q // (R * R)
    v0 = ao.values(F, mask, states, res, z, y, x).astype(np.float64)
    v1 = ao.values(F, mask, states, res, z + (a == 2), y + (a == 1), x + (a == 0)).astype(np.float64)
    lo = np.asarray(sdf_params[:3], np.float64)
    h = (np.asarray(sdf_params[3:], np.float64) - lo) / np.float64(R - 1)
    t = (np.float64(iso32) - v0) / (v1 - v0)
    pos = lo[None, :] + np.stack([x, y, z], axis=1).astype(np.float64) * h[None, :]
    rows = np.arange(len(E))
    pos[rows, a] = pos[rows, a] + t * h[a]
    verts = pos.astype(np.float32)
    off = np.cumsum(nt) - nt
    faces = np.zeros((int(nt.sum()), 3), np.int64)
    for k in range(5):
        m = nt > k
        if not m.any():
            break
        for j in range(3):
            e = mo.TABLE[case[m], 3 * k + j]
            ax, dx, dy, dz = mo.EDGE[e, 0], mo.EDGE[e, 1], mo.EDGE[e, 2], mo.EDGE[e, 3]
            g = (((cz[m] + dz) * R + (cy[m] + dy)) * R + (cx[m] + dx)) * 3 + ax
            faces[off[m] + k, j] = np.searchsorted(E, g)
    out = (verts, faces.astype(np.int32), counts)
    return out + (K,) if want_K else out
