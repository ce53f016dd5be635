"""The whole-space 7-LUT enumeration without a GPU: the C ABI symbol and its Python binding, the
header's limit, and the test-side whole-space reference against the list reference (cut at a
phase-1 cap, the whole-space matches whose combination lies in the list are the list's matches,
ranks mapped back to list indices)."""
import ctypes as C
import re
from math import comb

import numpy as np
import pytest

import _enum7_all_reference as W
import _enum_reference as R
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native


def test_abi_symbol_and_argtypes():
    restype, argtypes = native.SIGNATURES["sbg_enum7_all"]
    assert restype is C.c_int
    assert argtypes == native.SIGNATURES["sbg_enum7"][1]
    lib = native.load_library()
    assert lib.sbg_enum7_all.argtypes == argtypes
    with open(S.ROOT + "/include/sboxgates_b200.h") as f:
        header = f.read()
    assert re.search(r"#define SBG_ENUM7_ALL_MAX_GATES 64\b", header)
    assert native.SBG_ENUM7_ALL_MAX_GATES == 64
    assert re.search(r"int sbg_enum7_all\(sbg_handle \*h, int part, int nparts, const uint8_t "
                     r"\*outer_order,\s+const uint8_t \*middle_order, uint64_t max_matches, "
                     r"sbg_match \*out, uint64_t \*n_out,\s+uint64_t \*total, uint64_t \*feasible\);",
                     header)
    assert callable(sb.enumerate_7lut_all) and callable(sb.LutEngine.enumerate7_all)


def test_enumerate_7lut_all_checks_the_gate_count():
    tabs = S.synthetic_state(65, seed=3)
    with pytest.raises(ValueError):
        sb.enumerate_7lut_all(None, tabs[:6], tabs[0], S.mux_mask([]), [], b"", b"", 1)
    with pytest.raises(ValueError):
        sb.enumerate_7lut_all(None, tabs, tabs[0], S.mux_mask([]), [], b"", b"", 1)


def test_lex_ranks_are_the_oracle_ranks():
    rs = np.random.RandomState(4)
    for n in (7, 9, 16, 40, 64):
        combos = np.sort(np.array([rs.choice(n, 7, replace=False) for _ in range(50)]), axis=1)
        got = W.lex_ranks(combos, n)
        want = [S.oracle_lib().orc_combination_rank(n, 7, (C.c_uint16 * 7)(*map(int, c)))
                for c in combos]
        assert got.tolist() == list(want)
    assert W.lex_ranks(np.array([list(range(7)), list(range(57, 64))]), 64).tolist() == \
        [0, comb(64, 7) - 1]


def _states():
    """Seeded 7-LUT states, small enough for the brute-force key oracle: a planted circuit on
    random gates, a random mask of 24-40 positions, some input bits excluded."""
    rs = np.random.RandomState(77)
    out = []
    while len(out) < 4:
        n = int(rs.randint(8, 13))
        tabs = S.synthetic_state(n, seed=int(rs.randint(1 << 30)))
        inb = sorted(int(x) for x in rs.choice(8, int(rs.randint(0, 3)), replace=False))
        g = [int(x) for x in rs.choice([x for x in range(n) if x not in inb], 7, replace=False)]
        f = [int(x) for x in rs.randint(1, 255, 3)]
        tgt = S.lut_table(f[2], S.lut_table(f[0], tabs[g[0]], tabs[g[1]], tabs[g[2]]),
                          S.lut_table(f[1], tabs[g[3]], tabs[g[4]], tabs[g[5]]), tabs[g[6]])
        mask = np.zeros(4, dtype=np.uint64)
        for p in rs.choice(256, int(rs.randint(24, 41)), replace=False):
            mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
        feas = W.feasible_tuples(tabs, tgt, mask, inb)
        if 3 <= len(feas) <= 40:
            out.append((tabs, tgt, mask, inb, feas))
    return out


@pytest.mark.parametrize("cap", [2, 100000])
def test_whole_reference_cut_at_the_cap_is_the_list_reference(cap):
    """At cap 100,000 the list is every feasible combination of these states, so the two
    references must agree record for record; at cap 2 the whole space holds more than the list."""
    for i, (tabs, tgt, mask, inb, feas) in enumerate(_states()):
        rs = np.random.RandomState(i)
        orders = (bytes(rs.permutation(256).astype(np.uint8)),
                  bytes(rs.permutation(256).astype(np.uint8)))
        whole = W.WholeReference(tabs, tgt, mask, inb, orders, tuples=feas)
        lst, _ = S.oracle_filter7(tabs, tgt, mask, inb, cap=cap)
        lst = np.asarray(lst, dtype=np.uint16).reshape(-1, 7)
        assert np.array_equal(lst, feas[:cap]), i
        listed = R.Reference(7, tabs, tgt, mask, inb, orders, tuples=lst)
        # the whole-space matches of the list's combinations, ranks mapped back to list indices
        ranks = W.lex_ranks(lst, len(tabs))
        rank_of = whole.all["key"] >> np.uint64(23)
        inside = np.isin(rank_of, ranks.astype(np.uint64))
        cut = whole.all[inside].copy()
        cut["key"] = (np.searchsorted(ranks, rank_of[inside].astype(np.int64)).astype(np.uint64)
                      << np.uint64(23)) | (cut["key"] & W.LOW23)
        assert cut.tobytes() == listed.all.tobytes(), i
        assert whole.feasible == len(feas) and listed.feasible == len(lst)
        assert whole.total >= listed.total
        if cap >= len(feas):
            assert whole.total == listed.total
