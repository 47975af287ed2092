"""TEST INFRASTRUCTURE ONLY -- the tensor-core point kernel (disn_b200/csrc/point_tc.cu) restated on the CPU.

`emulate` follows `point_tc_kernel` operation for operation wherever the kernel is deterministic:

* operands as `tc_pack_weights` (weights) and `store_pair` (activations) build them, per operand mode:
  "bf16x3"  x = hi + lo, both bf16 RN (lo = bf16 of the fp32 residual); products hi.hi + lo.hi + hi.lo;
  "f16f8"   h = fp16 RN; c1 = e5m2((a - h(a)) 2^s1) . e5m2(w 2^-s1); c2 = e5m2(fp16(h(a) fp16(2^-s2))) .
            e5m2((w - h(w)) 2^s2); products h.h + [bit 2l] c1 + [bit 2l+1] c2 in tensor layer l;
  e5m2 conversions RN and SATFINITE (a clamp to +-57344 before torch's overflowing cast);
* the float32 steps on the CUDA cores in kernel order: the fold1/conv1 fmaf chain, the epilogues
  fmaxf(acc + (bias [+ gather]), 0), the 4-tap gather as an fmaf chain in taps_of order, the fold2/conv5 dot products in
  the order of the accumulator fragment and its lane shuffles, (p0 + p1) + b6, tanhf, __fdiv_rn by out_div.

The one thing modelled rather than restated is the warpgroup MMA accumulation: every product and sum of a tensor layer is
taken in float64 and the layer output is rounded once to float32.  The distance of the kernel from this emulation is
therefore the hardware's fp32 accumulation order and nothing else.  fmaf is computed in float64 and rounded once; the
rare double rounding this admits is far below any bound the tests use.  mode "exact" rounds nothing (float64
throughout, the projection included) and equals the folded float64 oracle.

Padding rows of a partial tile (the kernel evaluates them as the point (0, 0, 0) without image features) are not
emulated; they only matter to the fp16 range guard, so callers that probe it use N % 64 == 0.
"""
from __future__ import annotations

import math

import numpy as np
import torch

MODES = ("exact", "bf16x3", "f16f8")
CORR_DEFAULT = 0xDF          # point_tc.cu: every correction but the second product of fold2/conv1
E5M2_MAX = 57344.0
SCOPES = ("sdfprediction", "sdfprediction_imgfeat")       # stream 0 (global), stream 1 (local)
LAYERS = ("fold1/conv2", "fold1/conv3", "fold2/conv1", "fold2/conv2")   # the four tensor layers
LAYER_K = (64, 256, 512, 512)
LAYER_N = (256, 512, 512, 256)
_CHUNK = 8192


# ------------------------------------------------------------------------------------------ quantizers
def q_bf16(x: torch.Tensor) -> torch.Tensor:
    return x.float().to(torch.bfloat16)


def q_f16(x: torch.Tensor) -> torch.Tensor:
    return x.float().to(torch.float16)


def q_e5m2(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> e5m2, round to nearest even, SATFINITE (|x| beyond the largest finite value gives +-57344)."""
    return x.float().clamp(-E5M2_MAX, E5M2_MAX).to(torch.float8_e5m2)


def _f64(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float64)


def fma32(a, b, c):
    """fmaf on float32 tensors: exact product, one float64 sum, rounded to float32."""
    return (_f64(a) * _f64(b) + _f64(c)).float()


# ------------------------------------------------------------------------------------------ scale rule
def lround(x: float) -> int:
    """std::lround: nearest integer, halves away from zero (np.round rounds halves to even)."""
    a = abs(x)
    f = math.floor(a)
    r = f + 1 if a - f >= 0.5 else f
    return int(math.copysign(r, x))


def layer_scales(w32: np.ndarray):
    """(s1, s2) of one tensor layer from its float32 weights (rows 0..K-1), as tc_pack_weights derives them."""
    w = np.asarray(w32, np.float32).astype(np.float64)
    rms = math.sqrt(float((w * w).sum()) / w.size)
    L = lround(math.log2(rms)) if rms > 0 else -4
    return min(24, max(-8, 10 + L)), min(28, max(-8, 12 + L))


def layer_weights(W: dict, s: int, l: int) -> np.ndarray:
    """Rows 0..K-1 of the [Cin, Cout] matrix of tensor layer l of stream s (fold2/conv1: its point-feature rows)."""
    w = np.asarray(W["%s/%s/weights" % (SCOPES[s], LAYERS[l])], np.float32)
    return np.ascontiguousarray(w.reshape(-1, w.shape[-1])[:LAYER_K[l]])


def act_scales(W: dict) -> np.ndarray:
    """The kernel's act_scale[stream][layer] = {2^s1, 2^-s2}, float32 [2, 4, 2]."""
    t = np.zeros((2, 4, 2), np.float32)
    for s in range(2):
        for l in range(4):
            s1, s2 = layer_scales(layer_weights(W, s, l))
            t[s, l] = (2.0 ** s1, 2.0 ** -s2)
    return t


def weight_operands(W: dict, mode: str):
    """[stream][layer] -> dict of [K, N] operand tensors in their storage dtype, as tc_pack_weights packs them:
    bf16x3 {"hi", "lo"} (bfloat16); f16f8 {"h", "e1", "e2"} (float16, float8_e5m2, float8_e5m2)."""
    out = []
    for s in range(2):
        row = []
        for l in range(4):
            w = torch.from_numpy(layer_weights(W, s, l))
            if mode == "bf16x3":
                hi = q_bf16(w)
                row.append({"hi": hi, "lo": q_bf16(w - hi.float())})
            elif mode == "f16f8":
                s1, s2 = layer_scales(w.numpy())
                h = q_f16(w)
                row.append({"h": h, "e1": q_e5m2(w * 2.0 ** -s1), "e2": q_e5m2((w - h.float()) * 2.0 ** s2)})
            else:
                raise ValueError(mode)
        out.append(row)
    return out


def act_operands_f16f8(a: torch.Tensor, sc_lo: float, sc_hi: float):
    """store_pair<MODE_F16F8> of float32 activations: (h, e5m2 residual, e5m2 copy).  The copy is scaled by an fp16
    multiply (__hmul2 by the fp16 of sc_hi), so it goes subnormal -- and rounds there -- for small h."""
    h = q_f16(a)
    lo = q_e5m2((a - h.float()) * np.float32(sc_lo))
    sc_h = q_f16(torch.tensor(float(sc_hi))).float()
    g = q_e5m2(q_f16(h.float() * sc_h))          # h * 2^-k is exact in float32; one rounding to fp16
    return h, lo, g


def act_operands_bf16x3(a: torch.Tensor):
    hi = q_bf16(a)
    return hi, q_bf16(a - hi.float())


# ------------------------------------------------------------------------------------------ CUDA-core steps
def project_f32(pts: np.ndarray, trans_mat: np.ndarray, clamp_max: float) -> np.ndarray:
    """common.cuh project(): [x,y,z,1] . T with fmaf in k order, fp32 division, clamp to [0, clamp_max].  [B,N,2]"""
    p = torch.from_numpy(np.asarray(pts, np.float32))
    T = torch.from_numpy(np.asarray(trans_mat, np.float32).reshape(-1, 12))
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    q = []
    for c in range(3):
        t = [T[:, c + 3 * i, None] for i in range(4)]
        q.append(fma32(z, t[2], fma32(y, t[1], x * t[0])) + t[3])
    uv = torch.stack([q[0] / q[2], q[1] / q[2]], dim=-1)
    return torch.clamp(uv, min=0.0).clamp(max=np.float32(clamp_max)).numpy()


def project_f64(pts, trans_mat, clamp_max: float) -> np.ndarray:
    p = np.asarray(pts, np.float64)
    T = np.asarray(trans_mat, np.float64).reshape(-1, 4, 3)
    xyz = np.einsum("bnk,bkc->bnc", p, T[:, :3]) + T[:, 3][:, None, :]
    return np.minimum(clamp_max, np.maximum(0.0, xyz[..., :2] / xyz[..., 2:3]))


def _gather(pm: torch.Tensor, uv: torch.Tensor, exact: bool) -> torch.Tensor:
    """taps_of + the epilogue's fmaf chain: pm [H,W,512] (float32), uv [n,2] -> [n,512]."""
    H, Wd, C = pm.shape
    u, v = uv[:, 0], uv[:, 1]
    ok = (u > -1) & (v > -1) & (u < Wd) & (v < H)
    fx, fy = torch.floor(u).long(), torch.floor(v).long()
    cx, cy = fx + 1, fy + 1
    dx, dy = cx.to(u.dtype) - u, cy.to(v.dtype) - v
    one = torch.ones((), dtype=u.dtype)
    wts = (dx * dy, (one - dx) * (one - dy), dx * (one - dy), (one - dx) * dy)
    taps = ((fx, fy), (cx, cy), (fx, cy), (cx, fy))
    flat = pm.reshape(-1, C)
    acc = torch.zeros((uv.shape[0], C), dtype=torch.float64 if exact else torch.float32)
    for (tx, ty), wk in zip(taps, wts):
        valid = ok & (tx >= 0) & (tx < Wd) & (ty >= 0) & (ty < H)
        m = flat[(ty.clamp(0, H - 1) * Wd + tx.clamp(0, Wd - 1))]
        wk = torch.where(valid, wk, torch.zeros_like(wk))[:, None]
        acc = acc + _f64(wk) * _f64(m) if exact else fma32(wk, m, acc)
    return acc


def _conv5(a5: torch.Tensor, w6: torch.Tensor, b6, exact: bool) -> torch.Tensor:
    """fold2/conv5 dot product: lane q of warpgroup h sums columns 128h + 8j + 2q + {0,1} (j = 0..15) with fmaf, the
    lanes combine as (q0 + q1) + (q2 + q3), the warpgroups as (p0 + p1) + b6."""
    if exact:
        return a5 @ _f64(w6) + float(b6)
    n = a5.shape[0]
    h = torch.arange(2).view(2, 1, 1, 1)
    q = torch.arange(4).view(1, 4, 1, 1)
    j = torch.arange(16).view(1, 1, 16, 1)
    c = torch.arange(2).view(1, 1, 1, 2)
    cols = (h * 128 + 8 * j + 2 * q + c).reshape(2, 4, 32)       # [h, q, step]
    pr = torch.zeros((n, 2, 4), dtype=torch.float32)
    for st in range(32):
        col = cols[:, :, st]
        pr = fma32(a5[:, col], w6[col], pr)
    p = (pr[..., 0] + pr[..., 1]) + (pr[..., 2] + pr[..., 3])
    return (p[:, 0] + p[:, 1]) + torch.tensor(b6, dtype=torch.float32)


# ------------------------------------------------------------------------------------------ the kernel
def emulate(W: dict, pts, trans_mat, pmap, gbias, mode: str = "f16f8", *, pts_rot=None, uv=None,
            corr_mask: int = CORR_DEFAULT, act_scale=None, keep_hi_lo: bool = True, clamp_max: float = 136.0,
            tanh: bool = False, out_div: float = 1.0):
    """point_tc_kernel<mode> on pts [B,N,3] (float32; pts_rot feeds the MLP when given), trans_mat [B,4,3] and the
    device's own encoder products pmap [B,H,W,512] (get_encoded(6)) and gbias [B,512] (get_encoded(7)).

    uv [B,N,2]: the projected points to gather at (the kernel's out_uv); default: project_f32 (project_f64 in "exact").
    corr_mask (f16f8): bit 2l keeps c1 of tensor layer l, bit 2l+1 keeps c2.  act_scale [2,4,2] overrides the activation
    multipliers (default: act_scales(W), derived like the weights' own scales).  keep_hi_lo=False drops hi.lo (bf16x3).

    Returns dict(pred [B,N], global [B,N], local [B,N], uv [B,N,2], act_max (largest fp32 activation the f16f8 kernel
    converts to fp16), overflow (an fp16 A operand is +inf: the kernel raises DISN_STATUS_FP16_OVERFLOW))."""
    if mode not in MODES:
        raise ValueError(mode)
    exact = mode == "exact"
    fdt = torch.float64 if exact else torch.float32
    pts = np.asarray(pts, np.float32)
    B, N, _ = pts.shape
    prot = pts if pts_rot is None else np.asarray(pts_rot, np.float32)
    if uv is None:
        uv = project_f64(pts, trans_mat, clamp_max) if exact else project_f32(pts, trans_mat, clamp_max)
    uv_t = torch.from_numpy(np.asarray(uv, np.float64 if exact else np.float32))
    pm = torch.from_numpy(np.asarray(pmap, np.float64 if exact else np.float32))
    gb = torch.from_numpy(np.asarray(gbias, np.float64 if exact else np.float32))
    sc = act_scales(W) if act_scale is None else np.asarray(act_scale, np.float32)
    g = lambda s, n: torch.from_numpy(np.asarray(W["%s/%s" % (SCOPES[s], n)], np.float32).reshape(-1)).to(fdt)

    # weight operands as float64 matrices [K, N]
    if exact:
        wops = [[(_f64(torch.from_numpy(layer_weights(W, s, l))),) for l in range(4)] for s in range(2)]
    else:
        wops = [[tuple(_f64(t) for t in ops.values()) for ops in row] for row in weight_operands(W, mode)]

    def tensor_layer(a, s, l):
        """a [n,K] (fdt) -> layer output before bias: float64 products and sums, rounded once to float32."""
        wo = wops[s][l]
        if exact:
            return a @ wo[0]
        if mode == "bf16x3":
            hi, lo = act_operands_bf16x3(a)
            hi, lo = _f64(hi), _f64(lo)
            out = hi @ wo[0] + lo @ wo[0]
            if keep_hi_lo:
                out = out + hi @ wo[1]
            return out.float()
        h, e1, e2 = act_operands_f16f8(a, sc[s, l, 0], sc[s, l, 1])
        out = _f64(h) @ wo[0]
        if (corr_mask >> (2 * l)) & 1:
            out = out + _f64(e1) @ wo[1]
        if (corr_mask >> (2 * l + 1)) & 1:
            out = out + _f64(e2) @ wo[2]
        return out.float()

    res = {k: np.zeros((B, N), np.float64 if exact else np.float32) for k in ("pred", "global", "local")}
    act_max = 0.0
    for b in range(B):
        for n0 in range(0, N, _CHUNK):
            n1 = min(N, n0 + _CHUNK)
            xr = torch.from_numpy(prot[b, n0:n1]).to(fdt)
            outs = []
            for s in range(2):
                w1 = g(s, "fold1/conv1/weights").view(3, 64)
                a = g(s, "fold1/conv1/biases").expand(n1 - n0, 64)
                for i in range(3):
                    a = a + xr[:, i:i + 1] * w1[i] if exact else fma32(xr[:, i:i + 1], w1[i], a)
                a = torch.clamp(a, min=0)
                for l in range(4):
                    act_max = max(act_max, float(a.max()))
                    acc = tensor_layer(a, s, l)
                    if l == 0:
                        bias = g(s, "fold1/conv2/biases")
                    elif l == 1:
                        bias = g(s, "fold1/conv3/biases")
                    elif l == 2 and s == 0:
                        bias = gb[b].to(fdt)
                    elif l == 2:
                        bias = g(s, "fold2/conv1/biases") + _gather(pm[b], uv_t[b, n0:n1], exact)
                    else:
                        bias = g(s, "fold2/conv2/biases")
                    a = torch.clamp(acc + bias, min=0)
                outs.append(_conv5(a, g(s, "fold2/conv5/weights"), g(s, "fold2/conv5/biases").item(), exact))
            r = outs[0] + outs[1]
            if tanh:
                r = torch.tanh(_f64(r)).to(fdt)
            res["pred"][b, n0:n1] = (r / torch.tensor(out_div, dtype=fdt)).numpy()
            res["global"][b, n0:n1] = outs[0].numpy()
            res["local"][b, n0:n1] = outs[1].numpy()
    res["uv"] = np.asarray(uv)
    res["act_max"] = act_max
    res["overflow"] = mode == "f16f8" and act_max >= 65520.0
    return res
