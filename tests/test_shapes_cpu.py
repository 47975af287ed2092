"""CPU side of the shape sweep (tests/test_gpu_shapes.py): the float64 references and split-K rules the GPU sweep uses,
checks that its element-wise error bound is tight enough to reject the plausible kernel slips, and the IoU voxel
window of oracle/metrics_oracle.py against an unwindowed voxelisation."""
import numpy as np
import pytest

from oracle import metrics_oracle as mo

# Element-wise bounds of the encoder GEMMs against S = |A| @ |W| + |b| (float64), see tests/test_gpu_shapes.py.  fp32:
# sequential fmaf chains over up to K = 4608 (or K / splits), worst measured 2^-21.2 (H100 SXM, M = 4225, K = 1472
# unsplit).  bf16x3: the dropped lo*lo term and the bf16 rounding of lo cost about 2^-16 relative per product; worst
# measured 2^-17.6 (K = 64, where a few products dominate S).
FP32_BOUND = 2.0 ** -20
TC_BOUND = 2.0 ** -16
H100_SXM_SMS = 132
SPLITK_WS_ELEMS = 8 << 20          # encoder_alloc: split-K workspace of one image


# ----------------------------------------------------------------------------------------------------------------------
# split-K rules of launch_gemm (encoder.cu, fp32 CUDA-core) and launch_conv_tc (conv_tc.cu, bf16x3 tensor core)
# ----------------------------------------------------------------------------------------------------------------------
def fp32_splits(M, N, K, sms, ws_elems=SPLITK_WS_ELEMS):
    bn = 128 if N % 128 == 0 else 64
    ctas = (N // bn) * -(-M // 128)
    splits = 1
    if K % 8 == 0 and ctas < sms:
        want = min(-(-296 // ctas), max(K // 64, 1))
        splits = next(d for d in range(want, 0, -1) if (K // 8) % d == 0)
        if splits * M * N > ws_elems:
            splits = 1
    return splits


def tc_splits(M, N, K, sms, ws_elems=SPLITK_WS_ELEMS):
    tiles = -(-M // 128) * -(-N // 128)
    slices = K // 64
    if tiles >= sms:
        return 1
    want = -(-2 * sms // tiles)
    return next(d for d in range(min(want, slices), 0, -1) if slices % d == 0 and d * M * N <= ws_elems)


# ----------------------------------------------------------------------------------------------------------------------
# float64 references
# ----------------------------------------------------------------------------------------------------------------------
def im2col(x):
    """x [B,H,W,Cin] -> [B*H*W, 9*Cin]: 3x3 SAME patches, zero padding, column k = tap*Cin + ci with the taps (dy, dx)
    row-major (TF's HWIO weights reshaped to [9*Cin, Cout])."""
    B, H, W, Cin = x.shape
    pad = np.zeros((B, H + 2, W + 2, Cin), x.dtype)
    pad[:, 1:H + 1, 1:W + 1] = x
    cols = [pad[:, dy:dy + H, dx:dx + W, :] for dy in range(3) for dx in range(3)]
    return np.concatenate(cols, axis=3).reshape(B * H * W, 9 * Cin)


def gemm_ref(A, Wt, bias, relu):
    """-> (C, S): C = act(A @ W + b) and S = |A| @ |W| + |b|, both float64; A is the (im2col) matrix [M,K]."""
    A, Wt = A.astype(np.float64), Wt.astype(np.float64)
    C = A @ Wt
    S = np.abs(A) @ np.abs(Wt)
    if bias is not None:
        C += bias.astype(np.float64)
        S += np.abs(bias.astype(np.float64))
    return (np.maximum(C, 0.0) if relu else C), S


def make_case(shape, N, K, relu, bias, positive, seed):
    """Float32 operands of one sweep case: A (plain [M,K] for shape = M, NHWC for shape = (B, H, W, Cin)), W [K,N],
    b [N] or None.  Weights are zero-mean at scale 1/sqrt(K); with relu the activations are positive and the weights
    carry a mean of -0.7/K, so about a quarter of the outputs are positive and a ReLU applied to the split-K partials
    before their sum changes the result.  positive=True makes every activation > 0, so that a dropped or misplaced
    padding tap changes the border outputs."""
    rng = np.random.default_rng(seed)
    a_shape = (shape, K) if np.isscalar(shape) else tuple(shape)
    A = rng.uniform(0.05, 1.0, a_shape) if (positive or relu) else rng.standard_normal(a_shape)
    Wt = rng.standard_normal((K, N)) / np.sqrt(K)
    if relu:
        Wt -= 0.7 / K        # E[a] = 0.525: output mean ~ -0.37, output std ~ 0.59
    b = rng.standard_normal(N) * 0.5 if bias else None
    return A.astype(np.float32), Wt.astype(np.float32), None if b is None else b.astype(np.float32)


def as_matrix(A):
    return im2col(A.astype(np.float64)) if A.ndim == 4 else A.astype(np.float64)


def ratio(got, ref, S):
    """worst element-wise |got - ref| / S (S > 0 everywhere the operands are non-trivial)"""
    return float(np.max(np.abs(got.astype(np.float64) - ref) / np.maximum(S, 1e-300)))


def within(got, ref, S, bound, floor=0.0):
    return bool(np.all(np.abs(got.astype(np.float64) - ref) <= bound * S + floor))


# ----------------------------------------------------------------------------------------------------------------------
# the bf16x3 bound must reject the float64 result of each plausible slip
# ----------------------------------------------------------------------------------------------------------------------
def _im2col_wrapped(x):
    """A slip of the im2col gather: a horizontal tap that falls off the image row reads the neighbouring row instead of
    zero (row-major pixel index + dx without the x bounds check); vertical padding stays correct."""
    B, H, W, Cin = x.shape
    flat = x.reshape(B, H * W, Cin)
    cols = []
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            col = np.zeros((B, H, W, Cin), x.dtype)
            for y in range(H):
                if not 0 <= y + dy < H:
                    continue
                for xx in range(W):
                    p = (y + dy) * W + xx + dx
                    if 0 <= p < H * W:
                        col[:, y, xx] = flat[:, p]
            cols.append(col)
    return np.concatenate(cols, axis=3).reshape(B * H * W, 9 * Cin)


# (shape, N, K): plain M = 514 (an m-tile of 2 rows after four full ones, 23 slices of 64), two im2col layers with
# border-only columns (H = 3) and m-tiles that cover several images (B = 2, H*W = 35)
POWER_SHAPES = [(514, 192, 1472), ((1, 3, 17, 64), 128, 576), ((2, 7, 5, 128), 64, 1152)]


@pytest.mark.parametrize("case", range(len(POWER_SHAPES)))
def test_tc_bound_rejects_plausible_slips(case):
    shape, N, K = POWER_SHAPES[case]
    A, Wt, b = make_case(shape, N, K, relu=1, bias=1, positive=True, seed=900 + case)
    Am = as_matrix(A)
    W64, b64 = Wt.astype(np.float64), b.astype(np.float64)
    M = Am.shape[0]
    C, S = gemm_ref(A if A.ndim == 2 else Am, Wt, b, relu=1)
    assert within(C.astype(np.float32), C, S, TC_BOUND)           # the float32-rounded reference itself passes
    splits = tc_splits(M, N, K, H100_SXM_SMS)
    assert splits > 1
    slips = {}
    k0 = (K // 64 // 2) * 64                                       # one 64-wide K slice dropped
    Ad = Am.copy()
    Ad[:, k0:k0 + 64] = 0
    slips["k_slice_dropped"] = np.maximum(Ad @ W64 + b64, 0)
    slips["bias_twice"] = np.maximum(Am @ W64 + 2 * b64, 0)
    kper = K // splits                                             # ReLU on every split-K partial before the reduce
    part = sum(np.maximum(Am[:, s * kper:(s + 1) * kper] @ W64[s * kper:(s + 1) * kper], 0) for s in range(splits))
    slips["relu_before_splitk_sum"] = np.maximum(part + b64, 0)
    lo = (M - 1) // 128 * 128                                      # last (partial) m-tile's rows shifted by one
    sh = C.copy()
    sh[lo:] = np.roll(C[lo:], 1, axis=0)
    slips["last_mtile_rows_shifted"] = sh
    if A.ndim == 4:
        slips["padding_from_neighbour_row"] = np.maximum(_im2col_wrapped(A.astype(np.float64)) @ W64 + b64, 0)
    for name, wrong in slips.items():
        assert not within(wrong, C, S, TC_BOUND), name


def test_split_rules_cover_the_decoder_projection():
    """the explicit-feature decoder's projection (K = 1472 = 23 slices of 64, N = 512) splits 23 ways on the tensor
    cores up to B*N = 256 rows and not at all above; the fp32 kernel splits 23 ways up to 384 rows"""
    assert [tc_splits(m, 512, 1472, H100_SXM_SMS) for m in (1, 256, 257, 514)] == [23, 23, 1, 1]
    assert [fp32_splits(m, 512, 1472, H100_SXM_SMS) for m in (1, 256, 384, 385, 514)] == [23, 23, 23, 8, 8]


# ----------------------------------------------------------------------------------------------------------------------
# IoU voxel window
# ----------------------------------------------------------------------------------------------------------------------
def unwindowed(verts, faces, dim):
    """voxel_occupancy with a window wide enough for every vertex of the mesh"""
    voff = int(np.ceil(np.abs(np.asarray(verts, np.float64)).max() * dim / 2.0)) + 3
    return mo.voxel_occupancy(verts, faces, dim, vg=2 * voff, voff=voff)


def edge_triangles():
    """small triangles straddling each binning edge, -1.1 and 1.3, on every axis, plus one near x = 0.95"""
    base = np.array([[-0.02, 0.10, 0.10], [0.02, 0.20, 0.12], [0.0, 0.12, 0.25]])
    verts = []
    for axis in range(3):
        for edge in (-1.1, 1.3):
            t = np.roll(base, axis, axis=1)
            t[:, axis] += edge
            verts.append(t)
    verts.append(base + [0.95, 0.0, 0.0])
    v = np.concatenate(verts).astype(np.float32)
    return v, np.arange(len(v), dtype=np.int32).reshape(-1, 3)


def far_triangle():
    v = np.array([[0.94, -0.3, 0.2], [0.96, -0.25, 0.21], [0.95, -0.28, 0.3]], np.float32)
    return v, np.array([[0, 1, 2]], np.int32)


def test_old_fixed_window_lost_geometry_above_dim_122():
    """The former fixed window (160 cells from -80) covers |k * 2/dim| < 160/dim: enough at dim 110, nothing at x = 0.95
    at dim 256.  The dim-derived window keeps the triangle and equals an unwindowed voxelisation."""
    v, f = far_triangle()
    old110, old256 = (mo.voxel_occupancy(v, f, d, vg=160, voff=80) for d in (110, 256))
    new110, new256 = (mo.voxel_occupancy(v, f, d) for d in (110, 256))
    assert old110.sum() > 0 and np.array_equal(old110, new110)
    assert old256.sum() == 0 and new256.sum() > 0
    np.testing.assert_array_equal(new256, unwindowed(v, f, 256))
    assert mo.iou_voxel(v, f, v, f, 256)[2] == 1.0


@pytest.mark.parametrize("dim", [110, 128, 256, 512])
def test_voxel_window_equals_unwindowed_at_the_binning_edges(dim):
    v, f = edge_triangles()
    occ = mo.voxel_occupancy(v, f, dim)
    np.testing.assert_array_equal(occ, unwindowed(v, f, dim))
    # both edges are reached: bins 0 and dim - 1 on every axis
    for axis in range(3):
        proj = occ.any(axis=tuple(a for a in range(3) if a != axis))
        assert proj[0] and proj[dim - 1], axis
    vg, voff = mo.voxel_window(dim)
    cell = 2.0 / dim
    assert -voff * cell < -1.1 - 2.4 / dim - 1.5 * cell and (vg - voff - 1) * cell > 1.3 + 1.5 * cell
