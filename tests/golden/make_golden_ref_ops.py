"""Generate tests/golden/ref_ops_cpu.npz: the outputs of the REFERENCE's own CPU ops (oracle/_ref, compiled from the
reference's sources by oracle/Makefile) on exactly the inputs of tests/test_oracle_cpu.py's compiled-op comparisons, so that
those comparisons also run where the reference sources (and so oracle/_ref) are absent.

    make -C oracle && python tests/golden/make_golden_ref_ops.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import metrics_oracle as mo  # noqa: E402


def nn_case():
    rng = np.random.default_rng(0)
    a = rng.standard_normal((3, 257, 3)).astype(np.float32)
    b = rng.standard_normal((3, 100, 3)).astype(np.float32)
    b[1, 5] = b[1, 9]                       # exact tie: the first minimum must win
    return a, b


AM_SHAPES = ((2, 64, 64), (1, 96, 32), (1, 40, 100), (1, 7, 1))


def am_cases():
    rng = np.random.default_rng(3)
    for B, N, M in AM_SHAPES:
        yield (rng.uniform(-0.5, 0.5, (B, N, 3)).astype(np.float32), rng.uniform(-0.5, 0.5, (B, M, 3)).astype(np.float32))


def main():
    out = {}
    a, b = nn_case()
    for k, v in zip(("dist1", "idx1", "dist2", "idx2"), mo.ref_nn_distance(a, b)):
        out["nn_" + k] = v
    for i, (x, y) in enumerate(am_cases()):
        m = mo.ref_approx_match(x, y)
        out["am%d_match" % i] = m
        out["am%d_cost" % i] = mo.ref_match_cost(x, y, m)
    np.savez_compressed(os.path.join(HERE, "ref_ops_cpu.npz"), **out)
    print("ref_ops_cpu.npz:", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
