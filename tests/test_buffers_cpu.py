"""Every device and pinned allocation of the library is owned by the one buffer type of common.cuh: no other code may
call the CUDA allocators, so no code can free, forget or outlive another owner's memory.  The two IPC entry points are
the exception: they hand their allocation to the caller across processes."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "disn_b200", "csrc")
ALLOC = re.compile(r"\bcuda(?:Malloc\w*|Free\w*|HostAlloc)\b")


def _strip_comments(src):
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return re.sub(r"//[^\n]*", "", src)


def _cut_block(src, head):
    """Remove the brace-delimited block that starts at the first match of regex `head`; return (rest, block)."""
    m = re.search(head, src)
    assert m, "not found: " + head
    i = src.index("{", m.end())
    depth = 0
    for j in range(i, len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return src[:m.start()] + src[j + 1:], src[m.start():j + 1]
    raise AssertionError("unbalanced braces after " + head)


def test_cuda_allocators_only_inside_the_buffer_type():
    allowed = {
        "common.cuh": [r"class\s+Buffer\b"],
        "api.cu": [r"int\s+disn_shared_alloc\s*\(", r"int\s+disn_shared_close\s*\("],
    }
    files = sorted(glob.glob(os.path.join(CSRC, "*.cu*")))
    assert len(files) >= 10
    offenders = []
    for path in files:
        name = os.path.basename(path)
        src = _strip_comments(open(path).read())
        for head in allowed.get(name, []):
            src, block = _cut_block(src, head)
            assert ALLOC.search(block), "%s: %s no longer allocates; update this test" % (name, head)
        for m in ALLOC.finditer(src):
            offenders.append("%s:%d %s" % (name, src.count("\n", 0, m.start()) + 1, m.group(0)))
    assert not offenders, "raw CUDA allocation outside the buffer type: " + ", ".join(offenders)
