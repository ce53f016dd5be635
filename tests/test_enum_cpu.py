"""Enumeration without a GPU: the CPU enumeration oracle against the oracle's first-match searches,
its order invariance, the Python decoding of matches into the reference's ret[10], and the
sbg_match layout against include/sboxgates_b200.h."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native

NONE = native.SBG_KEY_NONE


def _random_mask(rs, positions):
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, positions, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def _cases5():
    """(tables, target, mask, inbits) of search_5lut-sized states: n = 7-11, sparse random masks."""
    sbox = S.rijndael_sbox()
    rs = np.random.RandomState(51)
    for i in range(8):
        n = int(rs.choice([7, 8, 9, 10, 11]))
        inb = [] if i % 2 else [int(rs.randint(0, 8))]
        yield (S.synthetic_state(n, seed=5100 + i), S.sbox_target(sbox, i % 8),
               _random_mask(rs, int(rs.choice([8, 12, 16, 24]))), inb)


def _cases7():
    """7-LUT states with gate 0 excluded (no stale-cache rows) and the first entries of their
    phase-1 lists."""
    sbox = S.rijndael_sbox()
    rs = np.random.RandomState(71)
    out = []
    for i in range(6):
        n = int(rs.choice([8, 9, 10]))
        tabs = S.synthetic_state(n, seed=7100 + i)
        tgt = S.sbox_target(sbox, (3 * i) % 8)
        mask = _random_mask(rs, int(rs.choice([6, 10, 16])))
        inb = [0] if i % 2 else [0, int(rs.randint(1, 8))]
        lst, _ = S.oracle_filter7(tabs, tgt, mask, inb)
        if len(lst):
            out.append((tabs, tgt, mask, inb, lst[:2]))
    assert len(out) >= 3
    return out


def test_oracle_enum5_first_is_search5_key():
    for i, (tabs, tgt, mask, inb) in enumerate(_cases5()):
        order, _, _ = E.orders(i)
        total, keys, feasible = E.oracle_enum5(tabs, tgt, mask, inb, order, 4)
        first = S.oracle_search5_key(tabs, tgt, mask, inb, order)
        assert (keys[0] if keys else NONE) == first, i
        assert keys == sorted(set(keys)) and len(keys) == min(total, 4)
        assert feasible <= S.oracle_lib().orc_n_choose_k(tabs.shape[0], 5)


def test_oracle_enum7_first_is_decomp7_key():
    for i, (tabs, tgt, mask, inb, lst) in enumerate(_cases7()):
        _, outer, middle = E.orders(100 + i)
        total, keys = E.oracle_enum7(tabs, tgt, mask, lst, outer, middle, 3)
        first = S.oracle_decomp7_key(tabs, tgt, mask, lst, outer, middle)
        assert (keys[0] if keys else NONE) == first, i
        assert keys == sorted(set(keys)) and len(keys) == min(total, 3)


def test_oracle_totals_do_not_depend_on_orders():
    for i, (tabs, tgt, mask, inb) in enumerate(list(_cases5())[:4]):
        totals = {E.oracle_enum5(tabs, tgt, mask, inb, E.orders(s)[0], 0)[0] for s in (1, 2, 3)}
        assert len(totals) == 1, i
    tabs, tgt, mask, inb, lst = _cases7()[0]
    totals = {E.oracle_enum7(tabs, tgt, mask, lst[:1], *E.orders(s)[1:], 0)[0] for s in (4, 5)}
    assert len(totals) == 1


def _match(width, key, gates, fo, fm, fi, seen):
    m = np.zeros(1, dtype=sb.MATCH_DTYPE)[0]
    m["key"], m["func_outer"], m["func_middle"] = key, fo, fm
    m["func_inner"], m["inner_seen"], m["width"] = fi, seen, width
    m["gates"][:len(gates)] = gates
    return m


def test_match_to_ret_fills_like_result_to_ret():
    """The ret[10] of a match is what result5_to_ret / result7_to_ret give for the same solution,
    with the same RNG draws (one iff an inner cell is unseen)."""
    seed = bytes(range(128))
    for seen in (0xFF, 0x5A):
        r5 = native.SbgResult(found=1, func_outer=0x96, func_inner=0x12 & seen, inner_seen=seen)
        for i, g in enumerate([3, 9, 4, 1, 7]):
            r5.gates[i] = g
        a, b = sb.Xorshift1024(seed), sb.Xorshift1024(seed)
        want = sb.lut.result5_to_ret(r5, a).ret
        got = sb.match_to_ret(_match(5, 0, [3, 9, 4, 1, 7], 0x96, 0, 0x12 & seen, seen), b)
        assert got == want and a.draws == b.draws == (0 if seen == 0xFF else 1)
        r7 = native.SbgResult(found=1, func_outer=0x17, func_middle=0xE8, func_inner=0x40 & seen,
                              inner_seen=seen)
        for i, g in enumerate([2, 5, 8, 0, 6, 11, 10]):
            r7.gates[i] = g
        a, b = sb.Xorshift1024(seed), sb.Xorshift1024(seed)
        want = sb.lut.result7_to_ret(r7, a).ret
        got = sb.match_to_ret(_match(7, 0, [2, 5, 8, 0, 6, 11, 10], 0x17, 0xE8, 0x40 & seen, seen),
                              b)
        assert got == want and a.draws == b.draws


def test_decode_keys():
    assert sb.decode_key5((1234 << 12) | (7 << 8) | 200) == (1234, 7, 200)
    assert sb.decode_key7((99999 << 23) | (69 << 16) | (255 << 8) | 3) == (99999, 69, 255, 3)


def test_match_layout_against_header(tmp_path):
    """sbg_match as the C compiler lays it out from the header = the ctypes structure = the numpy
    dtype the Python layer reads the records with."""
    src = tmp_path / "layout.c"
    fields = ["key", "gates", "func_outer", "func_middle", "func_inner", "inner_seen", "width",
              "pad"]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "sboxgates_b200.h"\n'
                   "int main(void) {\n  printf(\"%zu %u\\n\", sizeof(sbg_match), "
                   "(unsigned)SBG_ENUM_MAX_MATCHES);\n"
                   + "".join('  printf("%%zu\\n", offsetof(sbg_match, %s));\n' % f for f in fields)
                   + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([os.environ.get("CC", "gcc"), "-I", os.path.join(S.ROOT, "include"), str(src),
                    "-o", str(exe)], check=True, capture_output=True)
    lines = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    size, cap = int(lines[0]), int(lines[1])
    offsets = [int(x) for x in lines[2:]]
    assert size == C.sizeof(native.SbgMatch) == sb.MATCH_DTYPE.itemsize == 32
    assert cap == native.SBG_ENUM_MAX_MATCHES
    assert offsets == [getattr(native.SbgMatch, f).offset for f in fields]
    assert offsets == [sb.MATCH_DTYPE.fields[f][1] for f in fields]


def test_enum_entry_points_declared_and_bound():
    header = open(os.path.join(S.ROOT, "include", "sboxgates_b200.h")).read()
    for name in ("sbg_enum5", "sbg_enum7"):
        assert re.search(r"\bint %s\(" % name, header)
        assert name in native.SIGNATURES


def test_engine_rejects_oversized_requests():
    eng = sb.LutEngine.__new__(sb.LutEngine)   # no device needed: the check precedes the call
    with pytest.raises(ValueError):
        eng._enumerate(None, [], native.SBG_ENUM_MAX_MATCHES + 1, True, 0, 1)
