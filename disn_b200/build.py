"""Build libdisn_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdisn_b200.so")
TEST_LIB = os.path.join(HERE, "libdisn_b200_test.so")
SOURCES = ["api.cu", "encoder.cu", "point_fp32.cu", "point_tc.cu", "mc.cu", "chamfer.cu", "conv_tc.cu", "cam.cu", "iou.cu",
           "decoder.cu", "emd.cu", "mesh_clean.cu", "mesh_sdf.cu", "mesh_normalize.cu", "sdf_sample.cu"]
# diagnostics: selftests / probes, plus encoder.cu rebuilt with its debug GEMM harness -> libdisn_b200_test.so
DIAG_SOURCES = ["tc_selftest.cu", "tc_probe.cu"]
# voxel classification (iou.cu), the small-part keep rule (mesh_clean.cu) and the distances and edge crossings of the
# signed distance field (mesh_sdf.cu) and the face areas, surface samples and normalised vertices (mesh_normalize.cu) must
# match the float64 oracle operation for operation
EXTRA_FLAGS = {"iou.cu": ["--fmad=false"], "mesh_clean.cu": ["--fmad=false"], "mesh_sdf.cu": ["--fmad=false"],
               "mesh_normalize.cu": ["--fmad=false"]}
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC,-ffp-contract=off", "--expt-relaxed-constexpr", "-shared"]


def needs_build() -> bool:
    if not os.path.exists(LIB) or not os.path.exists(TEST_LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "disn_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src: str, obj: str, extra, verbose: bool):
    cmd = [NVCC] + [f for f in FLAGS if f != "-shared"] + list(extra) + ["-c", os.path.join(CSRC, src), "-o", obj]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose:
        sys.stderr.write(r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    from concurrent.futures import ThreadPoolExecutor
    jobs = [(src, os.path.join(CSRC, src.replace(".cu", ".o")), EXTRA_FLAGS.get(src, [])) for src in SOURCES + DIAG_SOURCES]
    jobs.append(("encoder.cu", os.path.join(CSRC, "encoder_diag.o"), ["-DDISN_DIAGNOSTICS"]))
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(lambda j: _compile(j[0], j[1], j[2], verbose), jobs))
    prod = objs[:len(SOURCES)]
    diag = [o for o in prod if not o.endswith("encoder.o")] + objs[len(SOURCES):]
    for out, oo in ((LIB, prod), (TEST_LIB, diag)):
        r = subprocess.run([NVCC, "-shared", "-o", out] + oo + ["-lcudart"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
