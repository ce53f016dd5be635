"""CPU: the host side of the function filter -- the inner table hook against brute force,
AFFINE_FUNCTIONS against an ANF degree computation, gate_functions against lut_table and
gate2_table, allowed_fill and match_functions_allowed on hand-worked records, the argument checks
that need no device, and the header's declarations."""
import ctypes as C
import os

import numpy as np
import pytest

import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import graph, native

IN1, IN2, IN3 = 0xF0, 0xCC, 0xAA   # the three inputs as 3-input functions (lut_table numbering)


def _p3(x):
    return sum(3 ** j for j in range(8) if (x >> j) & 1)


def _brute_table(inner):
    fs = range(256) if inner is None else inner
    out = np.zeros(6561, dtype=np.uint8)
    for seen in range(256):
        for ones in range(256):
            if ones & ~seen:
                continue
            out[_p3(seen) + _p3(ones)] = any((f & seen) == ones for f in fs)
    return out


@pytest.mark.parametrize("which", ["all", "none", "empty", "single", "affine", "random1", "random2"])
def test_inner_table_equals_brute_force(which):
    rng = np.random.default_rng(len(which))
    inner = {"all": list(range(256)), "none": None, "empty": [], "single": [0x96],
             "affine": sorted(sb.AFFINE_FUNCTIONS)}.get(which)
    if which.startswith("random"):
        inner = sorted(int(f) for f in rng.choice(256, size=int(rng.integers(2, 40)), replace=False))
    got = sb.inner_table(inner)
    assert got.dtype == np.uint8 and got.shape == (6561,)
    assert np.array_equal(got, _brute_table(inner))
    if which in ("all", "none"):
        assert got.all()
    if which == "empty":
        assert not got.any()


def test_inner_table_rejects_a_null_output():
    lib = native.load_library()
    assert lib.sbg_inner_table(None, None) != 0


def _anf_degree(f):
    """Algebraic degree of a 3-input function from its algebraic normal form (Moebius transform)."""
    a = [(f >> m) & 1 for m in range(8)]
    for i in range(3):
        for m in range(8):
            if (m >> i) & 1:
                a[m] ^= a[m ^ (1 << i)]
    return max((bin(m).count("1") for m in range(8) if a[m]), default=0)


def test_affine_functions_have_degree_at_most_one():
    want = {f for f in range(256) if _anf_degree(f) <= 1}
    assert len(want) == 16
    assert set(sb.AFFINE_FUNCTIONS) == want
    assert {0x00, 0xFF, IN1, IN2, IN3, IN1 ^ IN2 ^ IN3, 0xFF ^ IN1} <= want
    assert 0x80 not in want   # AND of the three inputs


def _brute_gates(available):
    """lut_table(f, in1, in2, in3) == gate2_table(t, x, y) over 64-bit words of distinct inputs."""
    rng = np.random.default_rng(available)
    ins = [rng.integers(0, 2**63, size=4, dtype=np.uint64) for _ in range(3)]
    as_int = [sum(int(w) << (64 * i) for i, w in enumerate(x)) for x in ins]
    # inputs that realise every cell (a random 256-bit triple almost surely does; check it)
    cells = {((as_int[0] >> p) & 1) << 2 | ((as_int[1] >> p) & 1) << 1 | ((as_int[2] >> p) & 1)
             for p in range(256)}
    assert len(cells) == 8
    out = set()
    for f in range(256):
        tf = sum(int(w) << (64 * i) for i, w in enumerate(sb.lut_table(f, *ins)))
        for t in range(16):
            if not (available >> t) & 1:
                continue
            if any(graph.gate2_table(t, x, y) == tf for x in as_int for y in as_int):
                out.add(f)
    return out


@pytest.mark.parametrize("available", [194] + [1 << t for t in range(16)])
def test_gate_functions_equal_brute_force(available):
    assert set(sb.gate_functions(available)) == _brute_gates(available)


def test_gate_functions_194_is_and_or_xor():
    got = sb.gate_functions(194)
    for x, y in ((IN1, IN2), (IN1, IN3), (IN2, IN3)):
        assert {x & y, x | y, x ^ y} <= got
    assert 0x00 in got and IN1 in got       # XOR(x, x) and AND(x, x)
    assert 0xFF ^ IN1 not in got            # no inverter among AND, OR, XOR
    assert sb.gate_functions(0) == frozenset()
    for bad in (-1, 1 << 16):
        with pytest.raises(ValueError):
            sb.gate_functions(bad)


def test_allowed_fill_is_minimal():
    rng = np.random.default_rng(5)
    for _ in range(300):
        seen = int(rng.integers(0, 256))
        ones = int(rng.integers(0, 256)) & seen
        inner = None if rng.random() < 0.2 else \
            [int(f) for f in rng.choice(256, size=int(rng.integers(0, 30)), replace=False)]
        got = sb.allowed_fill(ones, seen, inner)
        cands = [f for f in (range(256) if inner is None else inner) if (f & seen) == ones]
        assert got == (min(cands) if cands else None)
    assert sb.allowed_fill(0x0F, 0xFF, [0x0F]) == 0x0F
    assert sb.allowed_fill(0x0F, 0xFF, [0x1F]) is None
    assert sb.allowed_fill(0x01, 0x03, [0xF0, 0x05, 0x0D]) == 0x05
    assert sb.allowed_fill(0, 0, []) is None
    assert sb.allowed_fill(0x80, 0x80) == 0x80


def _rec(width, fo, fm, fi, seen):
    r = np.zeros(1, dtype=sb.MATCH_DTYPE)[0]
    r["width"], r["func_outer"], r["func_middle"] = width, fo, fm
    r["func_inner"], r["inner_seen"] = fi, seen
    return r


def test_match_functions_allowed_by_hand():
    aff = sb.AFFINE_FUNCTIONS
    # 3-LUT: only inner counts; solved bits 0x96 & 0xF0 = 0x90, the XOR 0x96 completes them
    r3 = _rec(3, 0, 0, 0x90, 0xF0)
    assert sb.match_functions_allowed(r3, [], [], aff)
    assert sb.match_functions_allowed(r3, None, None, [0x96])
    assert not sb.match_functions_allowed(r3, None, None, [0x80, 0x0F])
    assert not sb.match_functions_allowed(r3, None, None, [])
    # 5-LUT: outer and inner count, middle does not
    r5 = _rec(5, 0x3C, 0, 0x01, 0x03)
    assert sb.match_functions_allowed(r5, aff, [], aff)          # 0x3C = in1 ^ in2; 0x55 completes
    assert not sb.match_functions_allowed(r5, [0x80], None, None)
    assert not sb.match_functions_allowed(r5, aff, None, [0x80])
    # 7-LUT: all three count
    r7 = _rec(7, 0xF0, 0x80, 0x00, 0x00)
    assert sb.match_functions_allowed(r7, aff, None, [0xE8])
    assert not sb.match_functions_allowed(r7, aff, aff, None)
    assert sb.match_functions_allowed(r7, None, [0x80], None)
    assert not sb.match_functions_allowed(r7, [0x0F], None, None)
    with pytest.raises(ValueError):
        sb.match_functions_allowed(_rec(4, 0, 0, 0, 0))


def test_function_filter_argument_checks():
    eng = sb.LutEngine.__new__(sb.LutEngine)   # no device: the checks run before the library
    for bad in ([256], [-1], [0.5], [True], "abc", [None], [[1]]):
        for role in ("outer", "middle", "inner"):
            with pytest.raises(ValueError):
                eng.set_function_filter(**{role: bad})


def test_header_declares_the_function_filter():
    with open(os.path.join(S.ROOT, "include", "sboxgates_b200.h")) as f:
        header = f.read()
    assert "int sbg_enum_set_functions(sbg_handle *h, const uint64_t *outer, const uint64_t " \
        "*middle,\n    const uint64_t *inner);" in header
    assert "int sbg_inner_table(const uint64_t *inner, uint8_t *out);" in header
    assert native.SIGNATURES["sbg_enum_set_functions"] == (
        C.c_int, [C.c_void_p, native.u64p, native.u64p, native.u64p])
    assert native.SIGNATURES["sbg_inner_table"] == (C.c_int, [native.u64p, C.POINTER(C.c_uint8)])
    lifetime = header[header.index("Cursor lifetime:"):header.index("Without a cursor")]
    assert "sbg_enum_set_functions ends it" in lifetime
    # the lines the depth filter's test reads are still there
    assert "sbg_enum_set_depth ends it, whatever the call returns." in lifetime
