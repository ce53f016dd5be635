"""Fetch and pick on the enumeration cursor, without a GPU: the closed-form rank -> record helpers
(tests/_fetch_support.py, the oracle of the GPU tests) against brute force over itertools, the C
declarations and their ctypes bindings, and sample_matches' argument checks."""
import ctypes as C
import itertools
import os
import re

import numpy as np
import pytest

import _fetch_support as F
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _brute_inner(t1, t2, t3, target, mask):
    ok, fi, seen = sb.solve_inner(t1, t2, t3, target, mask)
    assert ok
    return fi, seen


def _masks():
    return [np.zeros(4, dtype=np.uint64), F.one_position_mask(77), F.one_position_mask(200)]


def test_unrank_and_rank_are_lexicographic():
    for n, t in ((9, 3), (10, 5), (9, 7)):
        for r, combo in enumerate(itertools.combinations(range(n), t)):
            assert F.unrank(list(range(n)), t, r) == list(combo)
            assert F.rank_of(n, combo) == r


def test_record3_matches_brute_force():
    n = 9
    tabs = S.synthetic_state(n, seed=71)
    order = [int(x) for x in np.random.RandomState(5).permutation(n)]
    tgt = S.sbox_target(S.rijndael_sbox(), 2)
    for mask in _masks():
        brute = list(itertools.combinations(range(n), 3))
        assert F.total3(n) == len(brute)
        for r, (i, k, m) in enumerate(brute):
            g = [order[i], order[k], order[m]]
            fi, seen = _brute_inner(tabs[g[0]], tabs[g[1]], tabs[g[2]], tgt, mask)
            want = (i << 18 | k << 9 | m, g + [0] * 4, 0, 0, fi, seen, 3)
            assert F.record3(r, tabs, tgt, mask, order) == want, r


@pytest.mark.parametrize("inbits", [[], [0, 3], [1, 2, 6]])
def test_record5_matches_brute_force(inbits):
    n = 10
    tabs = S.synthetic_state(n, seed=72)
    order = bytes(np.random.RandomState(6).permutation(256).astype(np.uint8))
    tgt = S.sbox_target(S.rijndael_sbox(), 5)
    rows5 = S.order5_rows()
    # every key of search_5lut's enumeration order, inbits rejections skipped (lut.c:177-185)
    keys = [(c, k, pos) for c, combo in enumerate(itertools.combinations(range(n), 5))
            if not set(combo) & set(inbits) for k in range(10) for pos in range(256)]
    assert F.total5(n, inbits) == len(keys)
    combos = list(itertools.combinations(range(n), 5))
    rs = np.random.RandomState(len(inbits))
    ranks = sorted({0, len(keys) - 1, 2559, 2560} | {int(x) for x in rs.randint(0, len(keys), 150)})
    for mask in _masks():
        for r in ranks:
            c, k, pos = keys[r]
            g = [combos[c][rows5[k][i]] for i in range(5)]
            fo = order[pos]
            fi, seen = _brute_inner(sb.lut_table(fo, tabs[g[0]], tabs[g[1]], tabs[g[2]]), tabs[g[3]],
                                    tabs[g[4]], tgt, mask)
            want = (c << 12 | k << 8 | pos, g + [0, 0], fo, 0, fi, seen, 5)
            assert F.record5(r, tabs, tgt, mask, inbits, order, rows5) == want, (inbits, r)


def test_record7_matches_brute_force_on_a_capped_list():
    n, cap = 9, 3
    tabs = S.synthetic_state(n, seed=73)
    rs = np.random.RandomState(7)
    outer = bytes(rs.permutation(256).astype(np.uint8))
    middle = bytes(rs.permutation(256).astype(np.uint8))
    tgt = S.sbox_target(S.rijndael_sbox(), 1)
    rows7 = S.order7_rows()
    lst = list(itertools.combinations(range(n), 7))[:cap]
    total = F.total7(n, cap)
    assert total == cap * 70 * 65536
    # brute force: the (entry, row, outer position, middle position) product in key order
    ranks = sorted({0, total - 1, 65535, 65536, F.W7 - 1, F.W7} | {int(x) for x in
                                                                   rs.randint(0, total, 40)})
    for mask in _masks():
        for r in ranks:
            idx, k, po, pm = next(itertools.islice(
                itertools.product(range(len(lst)), range(70), range(256), range(256)), r, None))
            g = [lst[idx][rows7[k][i]] for i in range(7)]
            fo, fm = outer[po], middle[pm]
            fi, seen = _brute_inner(sb.lut_table(fo, tabs[g[0]], tabs[g[1]], tabs[g[2]]),
                                    sb.lut_table(fm, tabs[g[3]], tabs[g[4]], tabs[g[5]]),
                                    tabs[g[6]], tgt, mask)
            want = (idx << 23 | k << 16 | po << 8 | pm, g, fo, fm, fi, seen, 7)
            assert F.record7(r, tabs, tgt, mask, outer, middle, rows7, cap) == want, r
    assert F.total7(8, 100000) == 8 * F.W7   # a list shorter than the cap


def test_header_declares_fetch_and_pick():
    with open(os.path.join(ROOT, "include", "sboxgates_b200.h")) as f:
        text = re.sub(r"\s+", " ", f.read())
    assert ("int sbg_enum_fetch(sbg_handle *h, uint64_t first, uint64_t count, sbg_match *out, "
            "uint64_t *n_out);") in text
    assert ("int sbg_enum_pick(sbg_handle *h, const uint64_t *ranks, uint64_t nranks, "
            "sbg_match *out);") in text


def test_bindings_match_the_declarations():
    u64p = C.POINTER(C.c_uint64)
    assert native.SIGNATURES["sbg_enum_fetch"] == (
        C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, u64p])
    assert native.SIGNATURES["sbg_enum_pick"] == (C.c_int, [C.c_void_p, u64p, C.c_uint64, C.c_void_p])
    lib = native.load_library()
    assert lib.sbg_enum_fetch.argtypes[1] is C.c_uint64 and lib.sbg_enum_pick.restype is C.c_int


class _StandIn:
    """An engine that answers pick_matches with records whose key is the rank."""

    def __init__(self):
        self.picks = []

    def pick_matches(self, ranks):
        self.picks.append(np.array(ranks))
        out = np.zeros(len(ranks), dtype=sb.MATCH_DTYPE)
        out["key"] = ranks
        return out


def test_sample_matches_validates_and_draws():
    eng = _StandIn()
    e = sb.Enumeration(total=1000, feasible=0, matches=np.zeros(0, dtype=sb.MATCH_DTYPE))
    with pytest.raises(ValueError):
        sb.sample_matches(eng, sb.Enumeration(None, 0, e.matches), 1, 0)
    with pytest.raises(ValueError):
        sb.sample_matches(eng, e, 1001, 0)
    with pytest.raises(ValueError):
        sb.sample_matches(eng, e, -1, 0)
    assert eng.picks == []
    ranks, recs = sb.sample_matches(eng, e, 1000, 3)
    assert list(ranks) == list(range(1000))
    ranks, recs = sb.sample_matches(eng, e, 50, 3)
    assert len(set(ranks.tolist())) == 50 and list(ranks) == sorted(ranks.tolist())
    assert list(recs["key"]) == list(ranks)
    again, _ = sb.sample_matches(eng, e, 50, 3)
    assert np.array_equal(ranks, again)
    big = sb.Enumeration(total=458_752_000_000, feasible=0, matches=e.matches)
    ranks, _ = sb.sample_matches(eng, big, 10_000, 1)
    assert len(np.unique(ranks)) == 10_000 and int(ranks.max()) < big.total
    assert np.array_equal(ranks, np.sort(np.random.default_rng(1).choice(big.total, 10_000,
                                                                         replace=False)))
