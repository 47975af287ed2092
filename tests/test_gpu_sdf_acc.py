"""GPU tests of disn_sdf_metrics (Engine.sdf_metrics): the checkpoint score of test/test_sdf_acc.py at ground-truth samples.

pred comes from the point kernel in explicit-point mode and must be eval_points's bits; the per-image count must be exact
and each float64 sum must equal, within 2^-40 relative, an exactly rounded (math.fsum) sum of the same float32 terms formed
by numpy in TF's order.  The engine encodes at most 8 images, so batch 24 is covered through the driver (three calls of 8).
"""
import math

import numpy as np
import pytest
import torch

from disn_b200 import synth
from disn_b200.engine import batch_losses
from disn_b200.model_normalization import _loss_metric

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
ISO, SW, MW = 0.003, 10.0, 4.0


def _restated(pred, val):
    """float64 restatement: (count [B], wsum [B], rsum [B]) of the float32 terms, exactly summed."""
    p = pred.reshape(len(pred), -1)
    g = val.reshape(p.shape).astype(np.float32) - np.float32(ISO)
    cnt = ((g > 0) == (p > 0)).sum(axis=1)
    w = (g <= np.float32(0.01)).astype(np.float32) * np.float32(MW) + (g > np.float32(0.01)).astype(np.float32)
    wt = np.abs(g * np.float32(SW) - p) * w
    rt = np.abs(g - p / np.float32(SW))
    assert wt.dtype == rt.dtype == np.float32
    return cnt, np.array([math.fsum(r.astype(np.float64)) for r in wt]), np.array([math.fsum(r.astype(np.float64)) for r in rt])


def _inputs(B, N, seed):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-0.6, 0.6, size=(B, N, 3)).astype(np.float32)
    val = rng.uniform(-0.08, 0.08, size=(B, N)).astype(np.float32)
    val.reshape(-1)[::7] = np.float32(0.003)              # g = 0 exactly: a sign tie
    val.reshape(-1)[3::11] = np.float32(0.013)            # g next to the 0.01 mask threshold
    return synth.synthetic_images(B, seed=seed), synth.synthetic_trans_mats(B, seed=seed), pts, val


def _close(a, b):
    return np.all(np.abs(a - b) <= 2.0 ** -40 * np.abs(b))


@pytest.fixture(scope="module", params=["fp32", "bf16x3", "f16f8"])
def eng(request, he_weights):
    from disn_b200.engine import Engine
    e = Engine(device=0, precision=request.param, max_batch=8)
    e.load_weights(he_weights)
    yield e
    e.close()


@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("N", [1, 2048, 5000])
def test_sdf_metrics_host(eng, B, N):
    imgs, tm, pts, val = _inputs(B, N, 900 + 10 * B + N % 7)
    eng.encode(imgs)
    ref = eng.eval_points(pts, tm)
    cnt, ws, rs, pred = eng.sdf_metrics(pts, tm, val, want_pred=True)
    assert np.array_equal(pred.view(np.uint32), ref.view(np.uint32))
    c0, w0, r0 = _restated(ref, val)
    assert np.array_equal(cnt, c0)
    assert _close(ws, w0) and _close(rs, r0), (ws - w0, rs - r0)
    gt = (val - np.float32(ISO))[..., None]
    acc, real, loss = batch_losses(cnt, ws, rs, B * N)
    assert acc.dtype == np.float32 and acc.tobytes() == _loss_metric("accuracy", ref, gt, SW, MW).tobytes()
    for mine, name in ((real, "sdf_loss_realvalue"), (loss, "sdf_loss")):     # numpy's float32 mean: a few ulp apart
        assert abs(float(mine) - float(_loss_metric(name, ref, gt, SW, MW))) <= 1e-5 * abs(float(mine)) + 1e-30
    again = eng.sdf_metrics(pts, tm, val)
    for a, b in zip(again, (cnt, ws, rs)):
        assert a.tobytes() == b.tobytes()
    assert eng.sdf_metrics(pts, tm, val[..., None])[1].tobytes() == ws.tobytes()    # [B,N,1] as the loader holds it


@pytest.mark.parametrize("B,N", [(1, 2048), (8, 5000)])
def test_sdf_metrics_device_on_a_caller_stream(eng, B, N):
    imgs, tm, pts, val = _inputs(B, N, 4000 + B)
    eng.encode(imgs)
    cnt, ws, rs, pred = eng.sdf_metrics(pts, tm, val, want_pred=True)
    stream = torch.cuda.Stream(DEV)
    eng.set_stream(stream.cuda_stream)
    try:
        with torch.cuda.stream(stream):
            d = {k: torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for k, a in
                 (("img", imgs), ("tm", tm), ("pts", pts), ("val", val))}
            oc = torch.full((B,), -1, dtype=torch.int64, device=DEV)
            ow = torch.full((B,), float("nan"), dtype=torch.float64, device=DEV)
            orr = torch.full((B,), float("nan"), dtype=torch.float64, device=DEV)
            op = torch.full((B, N, 1), float("nan"), dtype=torch.float32, device=DEV)
            eng.encode_device(d["img"].data_ptr(), B, 137, 137, 3)
            eng.sdf_metrics_device(d["pts"].data_ptr(), d["tm"].data_ptr(), d["val"].data_ptr(), B, N, oc.data_ptr(),
                                   ow.data_ptr(), orr.data_ptr(), op.data_ptr())
            eng.synchronize()
            got = [t.cpu().numpy() for t in (oc, ow, orr, op)]
            # without a pred buffer the kernel writes the context's scratch; the sums are the same
            eng.sdf_metrics_device(d["pts"].data_ptr(), d["tm"].data_ptr(), d["val"].data_ptr(), B, N, oc.data_ptr(),
                                   ow.data_ptr(), orr.data_ptr())
            eng.synchronize()
            again = [t.cpu().numpy() for t in (oc, ow, orr)]
    finally:
        eng.set_stream(None)
    for a, b in zip(got, (cnt, ws, rs, pred)):
        assert a.tobytes() == b.tobytes()
    for a, b in zip(again, (cnt, ws, rs)):
        assert a.tobytes() == b.tobytes()


def test_sdf_metrics_refuses_bad_sizes(he_weights):
    import ctypes as C
    from disn_b200._lib import DisnError
    from disn_b200.engine import Engine
    e = Engine(device=0, precision="f16f8", max_batch=2)
    try:
        e.load_weights(he_weights)
        imgs, tm, pts, val = _inputs(2, 64, 77)
        with pytest.raises(DisnError, match="disn_encode has not been called"):
            e.sdf_metrics(pts, tm, val)
        e.encode(imgs)
        with pytest.raises(DisnError, match="N >= 1"):
            e.sdf_metrics(pts[:, :0], tm, val[:, :0])
        with pytest.raises(DisnError, match="batch differs"):
            e.sdf_metrics(pts[:1], tm[:1], val[:1])
        with pytest.raises(ValueError, match="B\\*N"):
            e.sdf_metrics(pts, tm, val[:, :10])
        with pytest.raises(DisnError, match="sdf_weight"):
            e.sdf_metrics(pts, tm, val, sdf_weight=0.0)
        out = [np.zeros(2, np.int64), np.zeros(2), np.zeros(2)]
        rc = e.lib.disn_sdf_metrics(e._h, pts.ctypes.data_as(C.c_void_p), tm.ctypes.data_as(C.c_void_p), None, 2, 64,
                                    0.003, 10.0, 4.0, 0, None, *[o.ctypes.data_as(C.c_void_p) for o in out])
        assert rc != 0 and b"null argument" in e.lib.disn_last_error()
        e.sdf_metrics(pts, tm, val)     # the context still works
    finally:
        e.close()


def test_sdf_metrics_reports_the_f16f8_overflow_status(he_weights):
    from tests.test_gpu_device_path import _scaled_heads
    from disn_b200._lib import DisnError
    from disn_b200.engine import Engine
    e = Engine(device=0, precision="f16f8", max_batch=1)
    try:
        e.load_weights(_scaled_heads(he_weights, 2.0 ** 17))
        imgs, tm, pts, val = _inputs(1, 500, 78)
        e.encode(imgs)
        with pytest.raises(DisnError, match="fp16 range"):
            e.sdf_metrics(pts, tm, val)
        e.set_precision("bf16x3")
        e.sdf_metrics(pts, tm, val)     # the status does not stick
    finally:
        e.close()


class _HostMetricEngine:
    """The GPU engine's encode and pred_sdf (eval_points), with the metric restated on the host."""

    def __init__(self, eng):
        self.eng = eng

    def encode(self, imgs):
        self.eng.encode(imgs)

    def sdf_metrics(self, pts, trans_mat, sdf_val, iso_offset=0.003, sdf_weight=10.0, mask_weight=4.0):
        assert (iso_offset, sdf_weight, mask_weight) == (ISO, SW, MW)
        return _restated(self.eng.eval_points(pts, trans_mat), np.asarray(sdf_val))


@pytest.mark.parametrize("bs", [24, 5])
def test_driver_end_to_end(he_weights, golden, tmp_path, capsys, bs):
    """test_sdf_acc on the golden's fixture with synthetic weights: batch 24 is scored as three encodes of 8, batch 5
    in one encode; the lines equal those of the same driver with the host restatement of the metric."""
    import random
    from disn_b200 import test_sdf_acc
    from disn_b200.engine import Engine
    from tests.test_sdf_acc_cpu import assert_same_lines, score_lines, write_fixture
    ref = golden["sdf_acc_ref"]
    root = write_fixture(ref, tmp_path)
    eng = Engine(device=0, precision="f16f8", max_batch=8)
    try:
        eng.load_weights(he_weights)
        runs = []
        for engine in (None, _HostMetricEngine(eng)):
            np.random.seed(5)
            random.seed(5)
            test_sdf_acc.main(["--view_dir", str(root / "views"), "--sdf_dir", str(root / "sdf"), "--test_lst_dir",
                               str(root / "lst"), "--log_dir", str(tmp_path / "log"), "--batch_size", str(bs),
                               "--img_feat_twostream", "--precision", "f16f8"], weights=he_weights, engine=engine)
            runs.append(score_lines(capsys.readouterr().out))
        assert len(runs[0]) == 96 // bs + 1
        assert_same_lines(runs[0], runs[1])
    finally:
        eng.close()


def test_create_sdf_cli_writes_one_obj_per_view(he_weights, golden, tmp_path):
    import glob
    import random
    from disn_b200 import create_sdf
    from tests.test_sdf_acc_cpu import write_fixture
    root = write_fixture(golden["sdf_acc_ref"], tmp_path)
    random.seed(3)
    written = create_sdf.main(["--view_dir", str(root / "views"), "--sdf_dir", str(root / "sdf"), "--test_lst_dir",
                               str(root / "lst"), "--log_dir", str(tmp_path / "log"), "--sdf_res", "16",
                               "--view_num", "2"], weights=he_weights)
    objs = sorted(glob.glob(str(tmp_path / "log" / "test_objs" / "17_0.0" / "*" / "*.obj")))
    assert len(objs) == 4 * 2 and sorted(written) == objs
    for p in objs:
        assert open(p).read().startswith("# Generated by the DISN marching-cubes post-pass")
