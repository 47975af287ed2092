"""CPU tests of the C-ABI boundary: the library builds, loads, exports every declared symbol, refuses to
run without a GPU (no silent fallback), and its host-only entry points behave."""
import ctypes as C
import os
import re
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions(header="disn_b200.h"):
    src = open(os.path.join(ROOT, "include", header)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(disn_[a-z_0-9]+)\s*\(", src)))


def test_library_builds_and_exports_every_declared_symbol():
    from disn_b200 import _lib
    lib = _lib.load()
    names = _declared_functions()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), "missing export " + n
    assert set(names) == set(_lib.EXPORTS), "python binding and header disagree"
    # diagnostics live in their own header / library; the product library must not export them
    tlib = _lib.load_test()
    tnames = _declared_functions("disn_b200_test.h")
    assert set(tnames) == set(_lib.TEST_EXPORTS)
    for n in tnames:
        assert hasattr(tlib, n) and not hasattr(lib, n), n


def test_write_dist_matches_golden(golden):
    from disn_b200.engine import write_dist
    g = golden["dist_roundtrip"]
    with tempfile.TemporaryDirectory() as td:
        fn = os.path.join(td, "c.dist")
        write_dist(fn, int(g["res"]), g["bbox"], g["values"])
        assert np.array_equal(np.fromfile(fn, dtype=np.uint8), g["file_bytes"])
    with pytest.raises(ValueError):
        write_dist("/tmp/x.dist", 3, g["bbox"], g["values"])


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from disn_b200.engine import Engine
    from disn_b200._lib import DisnError
    with pytest.raises(DisnError, match="no CUDA device|no CPU fallback"):
        Engine(device=0)


def test_default_config_values():
    from disn_b200 import _lib
    lib = _lib.load()
    cfg = _lib.DisnConfig()
    lib.disn_default_config(C.byref(cfg))
    assert (cfg.img_h, cfg.img_w, cfg.vgg_in, cfg.num_classes) == (137, 137, 224, 1024)
    assert cfg.clamp_max == 136.0 and cfg.sdf_weight == 10.0 and cfg.tanh_out == 0


@pytest.mark.parametrize("hw", [(137, 137), (64, 64), (128, 128), (137, 173), (173, 137), (256, 256)])
def test_engine_config_clamps_at_136_whatever_the_map_size(hw):
    """models/model_normalization.py:249-251 clamps projections to the constant [0, 136]; the map size only sets the
    size the taps are resized to."""
    from disn_b200.engine import engine_config
    cfg = engine_config(img_h=hw[0], img_w=hw[1], precision="f16f8", max_batch=2)
    assert (cfg.img_h, cfg.img_w) == hw and cfg.clamp_max == 136.0
    assert (cfg.precision, cfg.max_batch, cfg.vgg_in) == (2, 2, 224)


@pytest.mark.parametrize("hw", [(2048, 2048), (2049, 2049), (2, 2 ** 30), (65536, 65536)])
def test_create_refuses_a_map_of_2_31_elements_before_touching_a_device(hw):
    """The tensor-core point kernel addresses one image's [img_h, img_w, 512] map with 32-bit offsets: disn_create
    refuses img_h * img_w * 512 >= 2^31 before it looks for a device (so also on a machine without one) and names the
    limit.  65536 x 65536 would wrap a 32-bit product to 0."""
    from disn_b200 import _lib
    from disn_b200.engine import engine_config
    lib = _lib.load()
    h = C.c_void_p()
    cfg = engine_config(img_h=hw[0], img_w=hw[1])
    assert lib.disn_create(C.byref(cfg), C.byref(h)) != 0 and not h.value
    assert "img_h * img_w * 512 must stay below 2^31" in lib.disn_last_error().decode()
