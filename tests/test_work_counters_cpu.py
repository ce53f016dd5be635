"""CPU: the ground truth of the searches' work counters (sbg_result::tuples_swept), no device.

The GPU counter tests (test_work_counters_gpu.py) hold the library to closed forms instead of a CPU
sweep, so that they reach n = 160, where C(n,7) is far past 2^32.  Here those forms meet the
oracle's own counts (OrcStats.tuples_filtered of orc_filter_7lut / orc_search_5lut, the reference's
loops of lut.c:137-187 and 294-318):
  - 7-LUT: C(n,7) for a list below the cap; the rank of the last entry + 1 for a capped one;
  - 5-LUT: C(n,5) on a miss, the hit's rank + 1 on a hit;
and search_5lut's deal (Deal5, with and without the fused kernel's chunk head) cuts C(n,5) into
parts that cover every combination exactly once, excluded-gate prefixes included.  The chunk head
walks the allowed gates only, so the prefixes in front of its end that hold an excluded gate are in
no block; the library credits their combinations to part 0 (head_skipped5)."""
from math import comb

import numpy as np
import pytest

import _counter_support as W
import _enum_support as E
import _handle_support as H
import _support as S
from sboxgates_b200.lut import pack_tuple7

FULL = np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)


def _state(n, seed, mask, bit=0):
    return S.synthetic_state(n, seed=seed, num_inputs=min(8, n)), S.sbox_target(S.rijndael_sbox(),
                                                                                bit), mask


# (n, mask, inbits, cap): small caps make every dense state a capped one without a long walk
SWEEP7_CASES = [
    (7, FULL, [], 100000),
    (7, FULL, [0], 100000),              # the one tuple is rejected by inbits
    (8, FULL, [1, 3, 5], 100000),
    (9, S.mux_mask([(0, 1)]), [0, 2, 4, 6], 100000),
    (12, S.mux_mask([(0, 1), (5, 0)]), [0, 5], 100000),
    (14, S.mux_mask([(2, 0), (3, 1), (7, 0)]), [2, 3, 7], 100000),
    (16, S.mux_mask([(1, 1), (4, 0), (6, 1)]), [], 1),
    (16, S.mux_mask([(1, 1), (4, 0), (6, 1)]), [1, 4, 6], 37),
    (18, S.mux_mask([(0, 0), (3, 1), (7, 0)]), [0, 3, 7], 300),
    (20, S.mux_mask([(2, 1), (5, 0), (6, 1)]), [], 200),
    (20, H.random_mask(np.random.RandomState(20), 12), [0], 2500),
]


@pytest.mark.parametrize("case", range(len(SWEEP7_CASES)))
def test_sweep7_closed_form_matches_the_oracle(case):
    n, mask, inb, cap = SWEEP7_CASES[case]
    tabs, tgt, mask = _state(n, 7100 + case, mask, case % 8)
    lst, st = S.oracle_filter7(tabs, tgt, mask, inb, cap=cap)
    count = len(lst)
    assert st.tuples_feasible == count
    last = lst[-1] if count else None
    want = W.reference_sweep7_tuple(n, last, count, cap)
    assert st.tuples_filtered == want, (n, inb, cap, count, st.tuples_filtered, want)
    assert want <= comb(n, 7)
    if count:
        packed = pack_tuple7(lst[-1])
        assert W.reference_sweep7(n, packed, count, cap) == want
    if cap < 100000:
        assert count == cap, (n, cap, count)   # the case really is capped


def test_sweep7_cases_cover_both_sides_of_the_cap():
    capped = [c for c in SWEEP7_CASES if c[3] < 100000]
    assert capped and len(capped) < len(SWEEP7_CASES)


def _sweep5_cases():
    rs = np.random.RandomState(7200)
    out = []
    for i, (n, fixed) in enumerate([(5, []), (7, [(0, 1)]), (9, [(1, 0), (4, 1)]), (12, []),
                                    (14, [(2, 1)]), (16, [(0, 0), (3, 1), (6, 0)]), (20, [])]):
        tabs, tgt, mask = _state(n, 7300 + i, S.mux_mask(fixed), i % 8)
        inb = [b for b, _ in fixed if b < n]
        out.append((tabs, tgt, mask, inb))
        # the same gates with a planted 5-LUT on allowed gates: a hit
        allowed = [g for g in range(n) if g not in inb]
        gates = sorted(int(x) for x in rs.choice(allowed, 5, replace=False))
        out.append((tabs, E.planted5(tabs, gates, int(rs.randint(10)), 0x96, 0xCA), mask, inb))
    return out


def test_sweep5_closed_form_matches_the_oracle():
    hits = misses = 0
    for tabs, tgt, mask, inb in _sweep5_cases():
        n = len(tabs)
        rng = S.OrcRng.from_seed(n)
        found, ret, st = S.oracle_search(5, tabs, tgt, mask, inb, rng)
        rank = E.comb_rank(n, 5, sorted(ret[2:7])) if found else None
        assert st.tuples_filtered == W.reference_sweep5(n, rank), (n, inb, found, rank)
        hits += found
        misses += not found
    assert hits >= 5 and misses >= 2, (hits, misses)


def _covered(deal, nparts):
    """Every part's rank ranges under the deal, sorted: (lo, hi, part)."""
    out = []
    for p in range(nparts):
        for j in deal.part_blocks(p, nparts, skip_excluded=False):
            out += [(lo, hi, p) for lo, hi in deal.block_ranges(j)]
    return sorted(out)


DEAL5_CASES = [(n, inb, head) for n, head in ((5, False), (6, False), (9, False), (33, False),
                                              (64, False), (128, False), (128, True), (130, True),
                                              (200, True))
               for inb in ([], [0], [1, 4, 6], [0, 2, 5, 7])]


@pytest.mark.parametrize("n,inb,head", DEAL5_CASES)
def test_deal5_parts_add_up_to_the_whole(n, inb, head):
    """The parts' shares (Deal5, all blocks, the head's skipped prefixes on part 0) add up to C(n,5)
    for P = 1, 2, 3, 7 and P larger than the number of blocks; no combination is in two blocks, and
    the ones in none are exactly the head's skipped prefixes."""
    deal = E.Deal5(n, inb, head)
    skipped = W.head_skipped5(deal, inb)
    assert (skipped > 0) == (head and bool(inb)), (n, inb, head, skipped)
    for P in (1, 2, 3, 7, deal.blocks() + 3):
        shares = [W.deal5_part_sweep(deal, p, P, inb) for p in range(P)]
        assert sum(shares) == comb(n, 5), (n, inb, head, P, shares)
        gaps, pos = 0, 0
        for lo, hi, p in _covered(deal, P):
            assert lo >= pos and hi > lo, (n, inb, head, P, p, lo, hi, pos)
            gaps += lo - pos
            pos = hi
        assert gaps + comb(n, 5) - pos == skipped
        if P > deal.blocks():
            assert shares[-1] == 0, (n, P)


def test_search5_head_rule():
    """The head runs only in the fused kernel from n = 128 on, unless switched off, and a part that
    fell back from the two-kernel form keeps the prefix deal."""
    assert W.search5_head(True, False, 128, 3)
    assert not W.search5_head(True, False, 127, 1)
    assert not W.search5_head(False, True, 200, 1)
    assert not W.search5_head(True, True, 200, 2)
    assert W.search5_head(True, True, 200, 1)
    assert not W.search5_head(True, False, 200, 1, head_off=True)
