"""The point kernel's epilogues and fold1/conv1 prologue store at per-thread bases plus immediates
(disn_b200/csrc/point_tc_layout.cuh).  Those offsets are checked here against tc::sw128_offset / tc::sw64_offset, the
layout the MMAs read, for every thread and element: a host program built from the same header counts mismatches, and a
formula with a wrong bit must be caught."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "disn_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

PROGRAM = r"""
#include <cstdio>
#include "point_tc_layout.cuh"
using namespace disn::ptc;
int main() {
  int bad = store_offset_mismatches();
  // a deliberately wrong chunk XOR (bit 6 dropped) and a wrong SW64 row pattern must show up as mismatches
  int broken16 = 0, broken8 = 0;
  for (uint32_t r0 = 0; r0 < 56; ++r0)
    for (int j = 0; j < 16; ++j) {
      const uint32_t b16 = epi_base16(0, r0, 0), b8 = epi_base8(0, r0, 0);
      const uint32_t k = 8u * (j & 7);
      broken16 += ((b16 ^ ((uint32_t)(j & 3) << 4)) + (uint32_t)(j >> 3) * X_SLICE) !=
                  (uint32_t)(j >> 3) * X_SLICE + tc::sw128_offset(r0, k >> 3);
      broken8 += epi_off8(b8 ^ (((r0 >> 1) & 3u) << 4), 0, j, 0) != (uint32_t)(j >> 3) * X_SLICE + X_TILE +
                 tc::sw64_offset(r0, k >> 4) + (k & 15u);
    }
  std::printf("%d %d %d\n", bad, broken16, broken8);
  return 0;
}
"""


@pytest.fixture(scope="module")
def mismatches(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("tc_addressing")
    src, exe = d / "check.cu", d / "check"
    src.write_text(PROGRAM)
    subprocess.run([NVCC, "-std=c++17", "--expt-relaxed-constexpr", "-I", CSRC, str(src), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    return [int(v) for v in out]


def test_store_offsets_match_the_swizzled_layout(mismatches):
    assert mismatches[0] == 0


def test_a_wrong_swizzle_is_caught(mismatches):
    assert mismatches[1] > 0 and mismatches[2] > 0
