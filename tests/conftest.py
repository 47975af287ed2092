import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a)")


@pytest.fixture(scope="session")
def golden():
    return {n[:-4]: np.load(os.path.join(GOLDEN, n), allow_pickle=False)
            for n in os.listdir(GOLDEN) if n.endswith(".npz")}


@pytest.fixture(scope="session")
def he_weights():
    from disn_b200 import synth
    return synth.make_weights(seed=7, init="he")


@pytest.fixture(scope="session")
def engine(he_weights):
    """fp32 engine with the He-scaled synthetic weights loaded (GPU tests only)."""
    from disn_b200.engine import Engine
    eng = Engine(device=0, precision="fp32", max_batch=2)
    eng.load_weights(he_weights)
    yield eng
    eng.close()
