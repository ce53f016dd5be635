"""CPU: the 7-LUT chain enumeration's interface (sbg_enum7_chain) without a device -- the header and
the bindings, the chain rows, the key decode, grouping ids, depths, chain_luts and match_to_ret on
hand-built records, and the test-side chain oracle on tiny states."""
import ctypes as C
import itertools
import os
import re
import subprocess

import numpy as np
import pytest

import _enum_chain_reference as CR
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import lut, native


def test_header_declares_chain_and_native_binds_it(tmp_path):
    header = open(os.path.join(S.ROOT, "include", "sboxgates_b200.h")).read()
    for name in ("sbg_enum7_chain", "sbg_chain_row"):
        assert re.search(r"\bint %s\(" % name, header)
        assert name in native.SIGNATURES
    src = tmp_path / "shape.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "sboxgates_b200.h"\n'
                   'int main(void) {\n  printf("%zu %d %d %zu\\n", offsetof(sbg_match, shape), '
                   "SBG_SHAPE_TREE, SBG_SHAPE_CHAIN, sizeof(((sbg_match *)0)->pad));\n"
                   "  return 0;\n}\n")
    exe = tmp_path / "shape"
    subprocess.run([os.environ.get("CC", "gcc"), "-I", os.path.join(S.ROOT, "include"), str(src),
                    "-o", str(exe)], check=True, capture_output=True)
    off, tree, chain, pad = (int(x) for x in subprocess.run(
        [str(exe)], check=True, capture_output=True, text=True).stdout.split())
    assert (off, tree, chain, pad) == (27, 0, 1, 4)
    assert native.SbgMatch.shape.offset == sb.MATCH_DTYPE.fields["shape"][1] == 27
    assert (native.SBG_SHAPE_TREE, native.SBG_SHAPE_CHAIN) == (tree, chain)


def test_chain_rows_against_definition():
    rows = [sb.chain_row(k) for k in range(210)]
    expect = []
    for t in itertools.combinations(range(7), 3):
        rest = [p for p in range(7) if p not in t]
        for de in itertools.combinations(rest, 2):
            fg = [p for p in rest if p not in de]
            expect.append(list(t) + list(de) + fg)
    assert rows == expect
    assert len({(tuple(r[:3]), tuple(r[3:5])) for r in rows}) == 210
    assert rows == sorted(rows)
    assert all(sorted(r) == list(range(7)) for r in rows)
    assert [CR.oracle_row(k) for k in range(210)] == rows
    for bad in (-1, 210):
        with pytest.raises(ValueError):
            sb.chain_row(bad)


def _record(key, gates, fo, fm, fi, seen, shape=1):
    r = np.zeros(1, dtype=sb.MATCH_DTYPE)[0]
    r["key"], r["gates"], r["func_outer"], r["func_middle"] = key, gates, fo, fm
    r["func_inner"], r["inner_seen"], r["width"], r["shape"] = fi, seen, 7, shape
    return r


def test_key_decode_group_and_depth():
    key = (123456 << 24) | (209 << 16) | (17 << 8) | 250
    assert sb.decode_key7_chain(key) == (123456, 209, 17, 250)
    assert sb.match_group(key, 7, "shape", shape="chain") == key >> 16
    assert sb.match_group(key, 7, "tuple", shape="chain") == 123456
    assert sb.match_group(key, 7, None, shape="chain") == key
    assert sb.match_group(key, 7, "tuple") == key >> 23   # the default keeps the tree's ids
    with pytest.raises(ValueError):
        sb.match_group(key, 5, "tuple", shape="chain")
    with pytest.raises(ValueError):
        sb.match_group(key, 7, "tuple", shape="ring")
    depth = np.array([5, 1, 2, 3, 4, 0, 9, 7], dtype=np.uint16)
    rec = _record(key, [0, 1, 2, 3, 4, 6, 7], 0x96, 0xE8, 0, 0xFF)
    # 1 + max(1 + max(1 + max(5, 1, 2), 3, 4), 9, 7) = 1 + max(8, 9) = 10
    assert sb.match_depth(rec, depth) == 10
    rec["gates"] = [6, 7, 0, 1, 2, 3, 4]
    assert sb.match_depth(rec, depth) == 1 + max(1 + max(1 + 9, 5, 1), 2, 3)
    rec["shape"] = 0
    assert sb.match_depth(rec, depth) == 1 + max(1 + max(9, 7, 5), 1 + max(1, 2, 3), 4)


def test_chain_luts_and_match_to_ret():
    rec = _record(0, [3, 5, 8, 9, 11, 12, 14], 0x96, 0xCA, 0x28, 0x3C)
    luts = sb.chain_luts(rec, 0x28 | 0xC1)
    assert luts == [(0x96, (3, 5, 8)), (0xCA, (("new", 0), 9, 11)),
                    (0x28 | 0xC1, (("new", 1), 12, 14))]
    rng = sb.Xorshift1024(bytes(range(128)))
    ref = sb.Xorshift1024(bytes(range(128)))
    f3 = sb.chain_luts(rec, rng)[2][0]
    assert f3 == 0x28 | (~0x3C & 0xFF & (ref.next() & 0xFF)) and rng.draws == 1
    with pytest.raises(ValueError):
        sb.chain_luts(rec, 0x00)   # disagrees with the solved bits
    with pytest.raises(ValueError):
        sb.match_to_ret(rec, rng)
    rec["shape"] = 0
    with pytest.raises(ValueError):
        sb.chain_luts(rec, 0x28)
    assert len(sb.match_to_ret(rec, sb.Xorshift1024(bytes(128)))) == 10


def test_oracle_finds_planted_chain_and_its_records_rebuild():
    n = 9
    tabs = S.synthetic_state(n, seed=11)
    g = [1, 2, 4, 5, 6, 7, 8]
    f1, f2, f3 = 0x96, 0x8E, 0xB2
    x1 = S.lut_table(f1, tabs[g[0]], tabs[g[1]], tabs[g[2]])
    x2 = S.lut_table(f2, x1, tabs[g[3]], tabs[g[4]])
    tgt = S.lut_table(f3, x2, tabs[g[5]], tabs[g[6]])
    mask = S.mux_mask([(0, 1), (3, 0)])
    rs = np.random.RandomState(5)
    orders = (bytes(rs.permutation(256).astype(np.uint8)), bytes(rs.permutation(256).astype(np.uint8)))
    feas, recs = CR.chain_reference(tabs, tgt, mask, [], orders)
    assert len(recs) > 0
    k = sb.chain_row(0)  # row 0: outer (0,1,2), {d,e} = (3,4), {f,g} = (5,6)
    assert k == [0, 1, 2, 3, 4, 5, 6]
    po = bytes(orders[0]).index(f1)
    pm = bytes(orders[1]).index(f2)
    rank = sum(1 for c in itertools.combinations(range(n), 7) if list(c) < g)
    planted = (rank << 24) | (0 << 16) | (po << 8) | pm
    assert planted in set(int(x) for x in recs["key"])
    assert np.all(recs["key"][1:] > recs["key"][:-1])
    for r in recs[:: max(1, len(recs) // 200)]:
        fill = lut.allowed_fill(r["func_inner"], r["inner_seen"])
        assert CR.rebuild_ok(r, tabs, tgt, mask, fill)


def test_oracle_against_brute_force_on_a_tiny_state():
    """On n = 7 with a mask of 20 positions, every (row, L1, L2) decided by building the whole
    circuit's table and every L3: the oracle's matches are exactly those with some L3."""
    tabs = S.synthetic_state(7, seed=3)
    mask = np.zeros(4, dtype=np.uint64)
    mask[0] = np.uint64(sum(1 << int(b) for b in np.random.RandomState(2).choice(64, 20, replace=False)))
    tgt = S.synthetic_state(8, seed=4)[7]
    rs = np.random.RandomState(1)
    orders = (bytes(rs.permutation(256).astype(np.uint8)), bytes(rs.permutation(256).astype(np.uint8)))
    keys, _, _ = CR.chain_matches(tabs, tgt, mask, np.arange(7, dtype=np.uint16)[None, :],
                                         orders, cap=210 << 16)
    got = set(int(k) for k in keys)
    bits = [b for b in range(64) if (int(mask[0]) >> b) & 1]
    val = lambda t, b: (int(t[0]) >> b) & 1
    expect = set()
    for k in range(0, 210, 37):   # a spread of rows; the rest follow the same code
        row = sb.chain_row(k)
        G = [tabs[p] for p in row]
        for po in range(0, 256, 5):
            f1 = orders[0][po]
            for pm in range(256):
                f2 = orders[1][pm]
                cell = {}
                ok = True
                for b in bits:
                    x1 = (f1 >> (val(G[0], b) << 2 | val(G[1], b) << 1 | val(G[2], b))) & 1
                    x2 = (f2 >> (x1 << 2 | val(G[3], b) << 1 | val(G[4], b))) & 1
                    c = x2 << 2 | val(G[5], b) << 1 | val(G[6], b)
                    if cell.setdefault(c, val(tgt, b)) != val(tgt, b):
                        ok = False
                        break
                if ok:
                    expect.add((k << 16) | (po << 8) | pm)
    assert {x for x in got if ((x >> 16) & 0xFF) % 37 == 0 and ((x >> 8) & 0xFF) % 5 == 0} == expect
