"""CPU tests of the OBJ reader's rules (disn_b200/csrc/obj_read.cu): the library's host coordinate converter against
Python's float() and numpy's float32 cast, the device's exact-conversion rule (its twin oracle/obj_oracle.py) against
float(), and the line / token split twin against Python's text-mode iteration and str.split()."""
import ctypes as C
import decimal
import lzma
import os

import numpy as np
import pytest

from oracle import obj_oracle as oo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEMO = os.path.join(ROOT, "tests", "golden", "demo_result.obj.xz")


def f32_bits(values):
    with np.errstate(over="ignore"):
        return np.array(values, np.float64).astype(np.float32).view(np.uint32)


def host_convert(toks):
    from disn_b200 import _lib
    lib = _lib.load_test()
    text = b"".join(toks)
    lens = np.array([len(t) for t in toks], np.int32)
    offs = np.concatenate([[0], np.cumsum(lens[:-1], dtype=np.int64)]).astype(np.int64)
    out = np.empty(len(toks), np.float32)
    if lib.disn_debug_obj_tokens(text, offs.ctypes.data_as(C.c_void_p), lens.ctypes.data_as(C.c_void_p), len(toks),
                                 out.ctypes.data_as(C.c_void_p)):
        raise _lib.DisnError(lib.disn_last_error().decode())      # the diagnostics library keeps its own message
    return out.view(np.uint32)


def midpoint_tokens(rng, n):
    """Decimal strings within a quarter double ulp of a float32 rounding midpoint: float64 rounding lands on the
    midpoint (then ties to even), while one rounding straight to float32 goes to the side of the decimal."""
    out = []
    ctx = decimal.Context(prec=60)
    for _ in range(n):
        f = np.float32(rng.uniform(0.5, 2.0) * 10.0 ** rng.integers(-30, 30))
        g = np.nextafter(f, np.float32(np.inf))
        mid = (float(f) + float(g)) / 2             # exact in float64
        q = decimal.Decimal(np.spacing(mid)) / 4
        d = ctx.add(decimal.Decimal(mid), q if rng.random() < 0.5 else -q)
        s = format(d, ".%de" % int(rng.integers(19, 26)))
        out.append(("-" if rng.random() < 0.3 else "") + s)
    return out


def corpus(seed=0, n=1_000_000):
    rng = np.random.default_rng(seed)
    toks = []
    k = n // 8
    vals = rng.standard_normal(k) * 10.0 ** rng.integers(-12, 12, k)
    toks += ["%g" % v for v in vals.astype(np.float32)]
    toks += ["%.9g" % v for v in vals[: k // 2].astype(np.float32)]
    toks += ["%.17g" % v for v in vals[k // 2:]]
    toks += ["%.18e" % v for v in vals]
    # 16-25 digit significands with random point positions and exponents
    for _ in range(k):
        nd = int(rng.integers(16, 26))
        digs = "".join(rng.choice(list("0123456789"), nd))
        p = int(rng.integers(0, nd + 1))
        s = digs[:p] + "." + digs[p:] if p < nd else digs
        if rng.random() < 0.5:
            s += "e%+d" % int(rng.integers(-40, 40))
        toks.append(("-" if rng.random() < 0.5 else "+" if rng.random() < 0.1 else "") + s)
    toks += midpoint_tokens(rng, k // 2)
    # subnormals of both types, out of range, signs, zeros and the forms the grammar allows
    sub = rng.uniform(1, 10, k // 4) * 10.0 ** rng.integers(-325, -300, k // 4)
    toks += ["%.*e" % (int(d), v) for d, v in zip(rng.integers(0, 20, k // 4), sub)]
    toks += ["%.9g" % v for v in (rng.uniform(1, 10, k // 4) * 10.0 ** rng.integers(-46, -37, k // 4))]
    fixed = ["1e400", "-1e400", "1e-400", "-1e-400", "1e39", "-3.5e38", "3.4028235e38", "3.40282357e38", "-0", "+0",
             "-0.0", "0e999999999999", "-0e-5", "+.5", "1.", "-1.e3", ".5e-3", "007", "00.00100", "inf", "-INF",
             "+Infinity", "iNfInItY", "nan", "-nan", "+NaN", "NAN", "2e-324", "3e-324", "4.9406564584124654e-324",
             "2.4703282292062328e-324", "1.401298464324817e-45", "7e-46", "7.00000000000001e-46",
             "9007199254740993", "9007199254740992", "123456789012345678901234567890", "1" + "0" * 400,
             "0." + "0" * 400 + "1", "1e2147483648", "1e-2147483649"]
    toks += fixed * 10
    while len(toks) < n:
        toks.append("%d" % int(rng.integers(-10 ** 9, 10 ** 9)))
    return toks


@pytest.fixture(scope="module")
def tokens():
    return corpus()


def test_host_converter_equals_float_then_float32(tokens):
    assert len(tokens) >= 1_000_000
    got = host_convert([t.encode() for t in tokens])
    want = f32_bits([float(t) for t in tokens])
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(tokens[i], hex(got[i]), hex(want[i])) for i in bad[:10]]


def test_midpoint_tokens_separate_double_from_single_rounding():
    """The corpus's midpoint tokens round to a float32 midpoint in float64, and about half of them round to the other
    float32 neighbour when rounded once, straight from the decimal."""
    differ = 0
    toks = midpoint_tokens(np.random.default_rng(1), 2000)
    for t in toks:
        x = abs(float(t))
        two = np.float32(x)
        lo = two if float(two) < x else np.nextafter(two, np.float32(0))
        hi = np.nextafter(lo, np.float32(np.inf))
        assert float(lo) + float(hi) == 2 * x
        one = lo if abs(decimal.Decimal(t)) < decimal.Decimal(x) else hi
        differ += one != two
    assert differ > 0.4 * len(toks)


def test_host_converter_refuses_tokens_outside_the_grammar():
    from disn_b200._lib import DisnError
    for t in [b"1_0", b"0x10", b"1e", b"1e+", b".", b"", b"+", b"--1", b"1.5.2", b"in", b"infinit", b"nan(1)", b"1e5x",
              b"e5", b"1d5", b" 1"]:
        with pytest.raises(DisnError, match="outside the OBJ reader's grammar"):
            host_convert([t])


def test_grammar_twin_accepts_what_float_accepts_in_ascii():
    ok = [b"1", b"-1.", b"+.5", b"1e5", b"1E-5", b"inf", b"-Infinity", b"nan", b"00.5e+07"]
    bad = [b"1_0", b"0x1", b"1e", b".e1", b"infinit", b"1 0"]
    assert all(oo.is_coordinate(t) for t in ok) and not any(oo.is_coordinate(t) for t in bad)
    for t in ok:
        float(t)


def test_fast_rule_twin_is_exact(tokens):
    picked = 0
    for t in tokens:
        v = oo.fast_value(t.encode())
        if v is not None:
            picked += 1
            w = float(t)
            assert np.float64(v).view(np.uint64) == np.float64(w).view(np.uint64), t
    assert picked > len(tokens) // 4


def test_fast_rule_takes_every_g_and_9g_token_of_mesh_coordinates():
    """disn_write_obj's %g, write_obj_exact's %.9g and the reference's demo/result.obj never reach the host."""
    rng = np.random.default_rng(2)
    v = np.concatenate([rng.uniform(-1, 1, 200_000), rng.uniform(-1000, 1000, 50_000),
                        rng.standard_normal(50_000) * 10.0 ** rng.integers(-10, 6, 50_000), [0.0, -0.0, 1e-10]])
    v = v.astype(np.float32)
    for fmt in ("%g", "%.9g"):
        for x in v:
            assert oo.fast_value((fmt % x).encode()) is not None, fmt % x
    with lzma.open(DEMO) as fh:
        for line in fh:
            tok = line.split()
            if tok and tok[0] == b"v":
                for t in tok[1:4]:
                    assert oo.fast_value(t) is not None, t


def test_line_and_token_split_twin_equals_python_text_mode(tmp_path):
    rng = np.random.default_rng(3)
    alphabet = [b"\r", b"\n", b"\r\n", b"\v", b"\f", b"\x1c", b"\x1d", b"\x1e", b"\x1f", b"\t", b" ", b"v", b"f", b"1",
                b"-", b"/", b"#", b"a", b"\x0b\r", b"\r\r\n"]
    p = tmp_path / "t.obj"
    for trial in range(3000):
        data = b"".join(alphabet[i] for i in rng.integers(0, len(alphabet), int(rng.integers(0, 60))))
        p.write_bytes(data)
        with open(p) as fh:
            want = [line.split() for line in fh]
        got = [[t.decode() for t in oo.tokens(line)] for line in oo.lines(data)]
        assert got == want, data
