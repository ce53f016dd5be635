"""CPU: the host-side search_5lut helpers of tests/_enum_support.py (search5_tuple_key, Deal5 and
the part keys, planted5, feasible5, expected_result5) against orc_search5_key over whole spaces and
against the reference's own answers in tests/golden/."""
import glob
import os
from itertools import combinations

import numpy as np
import pytest

import _enum_support as E
import _support as S
from sboxgates_b200.lut import _fill, shuffled_order
from sboxgates_b200.rng import Xorshift1024

NONE = E.NONE
ORACLE_BUDGET_NS = 1.5e9   # replay only the recorded calls the reference itself answered this fast


def _states():
    """(tables, target, mask, inbits, order): S-box targets under small and large masks, and planted
    circuits, for n = 9 ... 24."""
    sbox = S.rijndael_sbox()
    rs = np.random.RandomState(8080)
    specs = [(9, [(0, 1)], [], False), (14, [(2, 0), (5, 1)], [0, 2], True), (18, [], [3], True),
             (24, [(1, 1), (4, 0), (6, 1)], [1], False), (24, None, [], True),
             (20, [(3, 0)], [], True)]
    for i, (n, fixed, inb, plant) in enumerate(specs):
        tabs = S.synthetic_state(n, seed=8100 + i)
        if fixed is None:
            mask = np.zeros(4, dtype=np.uint64)
            for p in rs.choice(256, 100, replace=False):
                mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
        else:
            mask = S.mux_mask(fixed)
        if plant:
            gates = sorted(int(x) for x in rs.choice(np.arange(4, n), 5, replace=False))
            tgt = E.planted5(tabs, gates, i, 0xCA, 0xD8)
        else:
            tgt = S.sbox_target(sbox, i % 8)
        yield tabs, tgt, mask, inb, bytes(rs.permutation(256).astype(np.uint8))


def test_tuple_keys_give_the_whole_key():
    found = 0
    for tabs, tgt, mask, inb, order in _states():
        n = len(tabs)
        whole = S.oracle_search5_key(tabs, tgt, mask, inb, order)
        total = int(S.oracle_lib().orc_n_choose_k(n, 5))
        keys = [E.search5_tuple_key(tabs, tgt, mask, inb, order, r) for r in range(total)]
        assert min(keys) == whole
        for r, key in enumerate(keys):
            assert key == NONE or key >> 12 == r
        # a combination with an excluded gate has no key
        for r in range(0, total, 97):
            if set(E.nth_comb(n, 5, r)) & set(inb):
                assert keys[r] == NONE
        found += whole != NONE
    assert found >= 3


@pytest.mark.parametrize("head", [False, True])
def test_deal_partitions_the_allowed_combinations(head):
    """Every block of the dealt order, in each sharding, covers its ranks once; together they cover
    every combination of allowed gates; the ranks are ascending along each part; the minimum of the
    part keys is the whole key."""
    sbox = S.rijndael_sbox()
    cases = [(8, []), (12, [0]), (24, [1, 3]), (24, []), (40, [0, 2, 7]), (40, [])]
    for i, (n, inb) in enumerate(cases):
        deal = E.Deal5(n, inb, head)
        total = int(S.oracle_lib().orc_n_choose_k(n, 5))
        cover = np.zeros(total + 1, dtype=np.int64)
        spans = []
        for j in range(deal.blocks()):
            for lo, hi in deal.block_ranges(j):
                assert lo < hi
                cover[lo] += 1
                cover[hi] -= 1
                spans.append((lo, hi))
        cover = np.cumsum(cover)[:total]
        assert cover.max() == 1, n
        bad = set(inb)
        for r in np.flatnonzero(cover == 0):
            assert set(E.nth_comb(n, 5, int(r))) & bad, (n, int(r))
        if not bad:
            assert cover.min() == 1
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))   # ascending in dealt order
        if head and n == 40:
            # the head form: chunk items first, then whole prefixes from t_offset on
            assert 0 < deal.head_blocks and 0 < deal.prefix_blocks and deal.chunks > 1, vars(deal)
        for nparts in (1, 2, 3, 7, deal.blocks() + 3):
            owned = sorted(j for p in range(nparts) for j in deal.part_blocks(p, nparts, False))
            assert owned == list(range(deal.blocks()))
        if n > 24:
            continue
        tabs = S.synthetic_state(n, seed=8200 + i)
        tgt = S.sbox_target(sbox, i % 8)
        mask = S.mux_mask([(5, 1), (6, 0)])
        order = bytes(np.random.RandomState(i).permutation(256).astype(np.uint8))
        whole = S.oracle_search5_key(tabs, tgt, mask, inb, order)
        orc = E.Search5Oracle(tabs, tgt, mask, inb, order, head)
        for nparts in (1, 2, 3, 7, deal.blocks() + 3):
            keys = [orc.part_key(p, nparts) for p in range(nparts)]
            assert min(keys) == whole, (n, nparts)
            # a part's key is the minimum of its blocks' keys
            for p in (0, nparts - 1):
                assert keys[p] == min((orc.block_key(j) for j in deal.part_blocks(p, nparts)),
                                      default=NONE)
        assert E.part_keys5(tabs, tgt, mask, inb, order, 1, 3, head) == orc.part_key(1, 3)


def test_planted_rows_decompose_on_their_row():
    """planted5 on row k: the combination's own key is on row k (functions without two symmetric
    inputs under a large mask leave no other row), and expected_result5 of that key rebuilds it."""
    asym = [0xCA, 0xD8, 0xE4, 0xB4, 0xA6, 0x1B, 0x72, 0x4E, 0x2D, 0x8E]
    rs = np.random.RandomState(8300)
    n = 20
    tabs = S.synthetic_state(n, seed=8301)
    full = np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)
    rows = set()
    for k in range(10):
        for _ in range(4):
            gates = sorted(int(x) for x in rs.choice(n, 5, replace=False))
            fo, fi = (int(x) for x in rs.choice(asym, 2))
            tgt = E.planted5(tabs, gates, k, fo, fi)
            order = bytes(rs.permutation(256).astype(np.uint8))
            rank = E.comb_rank(n, 5, gates)
            key = E.search5_tuple_key(tabs, tgt, full, [], order, rank)
            assert key != NONE and (key >> 8) & 0xF <= k
            res = E.expected_result5(key, tabs, tgt, full, order)
            assert res["index"] == rank and sorted(res["gates"]) == gates
            got = S.lut_table(res["func_inner"], S.lut_table(res["func_outer"],
                              *[tabs[g] for g in res["gates"][:3]]), *[tabs[g] for g in res["gates"][3:]])
            assert np.array_equal(got, tgt)
            rows.add((key >> 8) & 0xF)
            if (key >> 8) & 0xF == k:
                row = S.order5_rows()[k]
                assert res["gates"] == [gates[row[i]] for i in range(5)]
                break
        else:
            pytest.fail("row %d never decomposed first" % k)
    assert rows == set(range(10))


def test_feasible5_counts_the_feasible_allowed_combinations():
    for tabs, tgt, mask, inb, order in _states():
        n = len(tabs)
        want = E.oracle_enum5(tabs, tgt, mask, inb, order, 0)[2]
        assert E.feasible5(tabs, tgt, mask, inb) == want
        assert E.feasible5(tabs, tgt, mask, inb, piece=777) == want
        brute = sum(S.oracle_check(5, tgt, mask, [tabs[g] for g in c])
                    for c in combinations(range(n), 5) if not set(c) & set(inb)) if n <= 14 else want
        assert brute == want


def _records5():
    out = []
    for path in [os.path.join(S.GOLDEN, "ref_cases.bin")] + sorted(
            glob.glob(os.path.join(S.GOLDEN, "run_*.bin"))):
        out += [r for r in S.read_records(path) if r.which == 5 and r.ns < ORACLE_BUDGET_NS]
    return out


def test_expected_result5_reproduces_the_recorded_calls():
    """Every 5-LUT call of ref_cases.bin and the recorded runs (answered by the reference's own
    object code): the oracle's key, expected_result5 and the don't-care fill give the recorded
    ret[10] and draw count."""
    recs = _records5()
    assert len(recs) >= 20
    found = 0
    for rec in recs:
        rng = Xorshift1024.from_state(rec.rng_s, rec.rng_p)
        order = shuffled_order(rng)
        n = rec.tables.shape[0]
        key = E.search5_range(rec.tables, rec.target, rec.mask, rec.inbits_list(), order, 0,
                              int(S.oracle_lib().orc_n_choose_k(n, 5)), 200_000)
        res = E.expected_result5(key, rec.tables, rec.target, rec.mask, order)
        assert (res is not None) == rec.found == (key != NONE)
        if res is None:
            assert rec.ret == [0] * 10
        else:
            fi = _fill(res["func_inner"], res["inner_seen"], rng)
            assert [res["func_outer"], fi] + res["gates"] + [0, 0, 0] == rec.ret
            found += 1
        assert rng.draws == rec.draws
    assert found >= 10, found
