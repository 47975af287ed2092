#!/usr/bin/env python3
"""Static SASS report of the tensor-core point kernel; needs nvcc and cuobjdump, no GPU.

Compiles disn_b200/csrc/point_tc.cu with the library's nvcc flags into a temporary directory and prints, for each
operand-mode instantiation of point_tc_kernel: registers, spill stores and loads, whether ptxas serialised the warpgroup
MMAs (warning C7512), and instruction counts per segment of the kernel body, cut at every BAR.SYNC.

The kernel launches three warpgroups and splits the register file with setmaxnreg.  ptxas reports the launch count;
the report adds each role's budget from the SASS (USETMAXREG.TRY_ALLOC for the consumers, USETMAXREG.DEALLOC for the
producer) and the highest register each role's code uses, which shows whether the consumers really use more than the
launch count.  The producer's code (from its USETMAXREG.DEALLOC to its EXIT) is counted as its own segment and left
out of the consumer segments.

Every epilogue loop is fully unrolled, so a segment's static counts are the instructions each thread runs per tile
there; an MMA segment holds a `#pragma unroll 1` loop over K slices and its counts are per loop body.  Segments are
named from the kernel's structure: a segment with warpgroup MMAs is a layer's MMA loop, the segment after it that
layer's epilogue (L3: the fold2/conv5 dot product), and the segment before a stream's first MMA loop its fold1/conv1
prologue.  f16f8 compiles the two point streams apart (global, then local); bf16x3 shares them.  ptxas may move
register-only work (an epilogue's first bias adds, its address bases) above the BAR.SYNC into the preceding MMA
segment, so the MMA loops and the whole body are summed too.

  int   LOP3, IADD3, IMAD*, LEA*, SHF, VIADD, MOV: address and index arithmetic in these kernels
  GMMA  HGMMA (fp16 / bf16) and QGMMA (e5m2) warpgroup MMAs

usage: tools/sass_report.py [--src FILE] [--segments]
  --src FILE   report another version of point_tc.cu (compiled against this tree's headers)
  --segments   also print every segment, not only the named ones
"""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from disn_b200.build import CSRC, FLAGS, NVCC  # noqa: E402

MODES = {"0": "bf16x3", "1": "f16f8"}
INT_OPS = {"LOP3", "IADD3", "IMAD", "LEA", "SHF", "VIADD", "MOV"}
COLUMNS = ("total", "int", "LDG", "STS", "F2FP", "GMMA", "LDL/STL")
_INSN = re.compile(r"^\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z0-9_.]+)")
_REG = re.compile(r"\bR(\d+)\b")


def compile_kernel(src: str, tmp: str):
    obj = os.path.join(tmp, "point_tc.o")
    cmd = [NVCC, "-Xptxas=-v"] + [f for f in FLAGS if f != "-shared"] + ["-I", CSRC, "-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit("nvcc failed:\n" + r.stdout + r.stderr)
    cuobjdump = os.path.join(os.path.dirname(NVCC), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def ptxas_info(log: str):
    """kernel mode -> (registers, spill stores, spill loads, C7512 seen)"""
    info, mode = {}, None
    for line in log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?_Z\w*point_tc_kernelILi(\d)E", line)
        if m:
            mode = MODES[m.group(1)]
            info.setdefault(mode, [None, None, None, False])
            continue
        if "Function properties for" in line:   # a device function (mbar_wait_slow)
            mode = None
            continue
        if mode is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            info[mode][1], info[mode][2] = int(m.group(1)), int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            info[mode][0] = int(m.group(1))
    # the serialisation warning names its function
    for m in re.finditer(r"C7512[^\n]*point_tc_kernelILi(\d)E|point_tc_kernelILi(\d)E[^\n]*C7512", log):
        info[MODES[m.group(1) or m.group(2)]][3] = True
    if "C7512" in log and not any(v[3] for v in info.values()):
        for v in info.values():
            v[3] = True
    return info


def kernels(sass: str):
    """kernel mode -> list of (opcode, instruction text) in program order"""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : \w*point_tc_kernelILi(\d)E", line)
        if m:
            cur = out.setdefault(MODES[m.group(1)], [])
            continue
        if "Function :" in line:
            cur = None
            continue
        m = _INSN.match(line)
        if m and cur is not None:
            cur.append((m.group(1), line.split(";")[0]))
    return out


def max_reg(insns):
    """highest general register Rn the instructions name (-1 if none)"""
    return max((int(r) for _, text in insns for r in _REG.findall(text)), default=-1)


def split_roles(insns):
    """-> (consumer and common instructions, producer instructions, consumer budget, producer budget).  The producer
    region runs from USETMAXREG.DEALLOC to the next EXIT; budgets are None when the kernel has no setmaxnreg."""
    alloc = next((i for i, (op, _) in enumerate(insns) if op.startswith("USETMAXREG.TRY_ALLOC")), None)
    dealloc = next((i for i, (op, _) in enumerate(insns) if op.startswith("USETMAXREG.DEALLOC")), None)
    budget = lambda i: int(re.search(r"(0x[0-9a-f]+|\d+)\s*$", insns[i][1]).group(1), 0) if i is not None else None
    if dealloc is None:
        return insns, [], budget(alloc), None
    end = next((i for i in range(dealloc, len(insns)) if insns[i][0] == "EXIT"), len(insns) - 1)
    return insns[:dealloc] + insns[end + 1:], insns[dealloc:end + 1], budget(alloc), budget(dealloc)


def count(ops):
    c = dict.fromkeys(COLUMNS, 0)
    c["total"] = len(ops)
    for op in ops:
        base = op.split(".")[0]
        if base in INT_OPS:
            c["int"] += 1
        elif base == "LDG":
            c["LDG"] += 1
        elif base == "STS":
            c["STS"] += 1
        elif base == "F2FP":
            c["F2FP"] += 1
        elif base in ("HGMMA", "QGMMA"):
            c["GMMA"] += 1
        elif base in ("LDL", "STL"):
            c["LDL/STL"] += 1
    return c


def segments(ops):
    segs, cur = [], []
    for op in ops:
        if op.startswith("BAR.SYNC"):
            segs.append(cur)
            cur = []
        else:
            cur.append(op)
    segs.append(cur)
    return segs


def name_segments(segs, mode):
    """segment index -> name, from the MMA segments (4 per stream)"""
    mma = [i for i, s in enumerate(segs) if any(op.startswith(("HGMMA", "QGMMA")) for op in s)]
    streams = ["global", "local"] if len(mma) == 8 else ["both"]
    names = {}
    for n, i in enumerate(mma):
        stream, layer = streams[n // 4], n % 4
        names[i] = "%s L%d MMA loop" % (stream, layer)
        if i + 1 < len(segs) and i + 1 not in mma:
            names[i + 1] = "%s L%d epilogue" % (stream, layer) if layer < 3 else "%s L3 fold2/conv5" % stream
        if layer == 0 and i >= 1:
            names[i - 1] = "%s fold1/conv1 prologue" % stream
    return names


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--src", default=os.path.join(CSRC, "point_tc.cu"))
    ap.add_argument("--segments", action="store_true")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory(prefix="sass_report_") as tmp:
        log, sass = compile_kernel(os.path.abspath(args.src), tmp)
    info = ptxas_info(log)
    ks = kernels(sass)
    print("%s (nvcc flags of disn_b200/build.py)" % os.path.relpath(os.path.abspath(args.src), ROOT))
    for mode in ("bf16x3", "f16f8"):
        regs, st, ld, c7512 = info.get(mode, [None, None, None, False])
        print("\n== point_tc_kernel, %s: %s registers, %s B spill stores, %s B spill loads, C7512 %s"
              % (mode, regs, st, ld, "PRESENT (MMAs serialised)" if c7512 else "absent"))
        insns = ks.get(mode, [])
        rest, prod, b_cons, b_prod = split_roles(insns)
        if b_cons is None and b_prod is None:
            print("   one register budget: %s at launch (no setmaxnreg); highest register used R%d"
                  % (regs, max_reg(insns)))
        else:
            alloc = next(i for i, (op, _) in enumerate(rest) if op.startswith("USETMAXREG.TRY_ALLOC"))
            print("   register budgets: %s at launch; consumers setmaxnreg %s, highest register used R%d; "
                  "producer setmaxnreg %s, highest register used R%d"
                  % (regs, b_cons, max_reg(rest[alloc:]), b_prod, max_reg(prod)))
        segs = segments([op for op, _ in rest])
        names = name_segments(segs, mode)
        print("%-30s" % "segment" + "".join("%9s" % c for c in COLUMNS))
        epi = dict.fromkeys(COLUMNS, 0)
        mma = dict.fromkeys(COLUMNS, 0)
        body = count([op for s in segs for op in s])
        if prod:
            print("%-30s" % "   producer" + "".join("%9d" % v for v in count([op for op, _ in prod]).values()))
        spill_in = []
        for i, s in enumerate(segs):
            c = count(s)
            name = names.get(i)
            if name and ("epilogue" in name or "MMA" in name) and c["LDL/STL"]:
                spill_in.append(name)
            for tot, suffix in ((epi, "epilogue"), (mma, "MMA loop")):
                if name and name.endswith(suffix):
                    for k in COLUMNS:
                        tot[k] += c[k]
            if name or args.segments:
                print("%-30s" % ("%2d %s" % (i, name or "")) + "".join("%9d" % c[k] for k in COLUMNS))
        for label, tot in (("L0-L2 epilogues, sum", epi), ("MMA loops, sum", mma), ("kernel body", body)):
            print("%-30s" % ("   " + label) + "".join("%9d" % tot[k] for k in COLUMNS))
        print("   local loads/stores in an MMA loop or epilogue: %s" % (", ".join(spill_in) if spill_in else "none"))


if __name__ == "__main__":
    main()
