"""The exact work counts of the searches (sbg_result::tuples_swept), as the reference counts them
(OrcStats.tuples_filtered of the oracle's orc_filter_7lut / orc_search_5lut, lut.c:294-318) and as
search_5lut's deal (Deal5) cuts them into parts.  No device needed; tests/test_work_counters_cpu.py
checks these against the oracle, tests/test_work_counters_gpu.py checks the library against them."""
from math import comb

import _enum_support as E
from sboxgates_b200.lut import unpack_tuple7

LIST_CAP = 100000


def reference_sweep7(n, last_packed, count, cap=LIST_CAP):
    """The reference's phase-1 count: C(n,7) when the list stays below the cap, else the rank of
    its last entry + 1 (the sweep stops right after the entry that fills the list)."""
    if count < cap:
        return comb(n, 7)
    return E.comb_rank(n, 7, unpack_tuple7(last_packed)) + 1


def reference_sweep7_tuple(n, last_tuple, count, cap=LIST_CAP):
    """reference_sweep7 for a list given as gate numbers (the oracle's (count, 7) array)."""
    if count < cap:
        return comb(n, 7)
    return E.comb_rank(n, 7, [int(g) for g in last_tuple]) + 1


def reference_sweep5(n, rank=None):
    """The reference's search_5lut count: C(n,5) on a miss, the hit's rank + 1 on a hit."""
    return comb(n, 5) if rank is None else rank + 1


def head_skipped5(deal, excluded):
    """The combinations no ticket of search_5lut's head form meets: those of the 3-gate prefixes in
    front of the head's end (t_offset) that hold an excluded gate (the head walks the allowed gates
    only).  The library credits them to part 0."""
    if deal.items == 0 or not excluded:
        return 0
    n = deal.n
    out = 0
    for t in range(deal.t_offset):
        pre = E.nth_comb(n - 2, 3, t)
        if set(pre) & set(excluded):
            out += comb(n - 1 - pre[2], 2)
    return out


def deal5_part_sweep(deal, part, nparts, excluded=()):
    """The combinations in part `part` of `nparts`'s blocks under Deal5, excluded-gate prefixes
    included (a part credits every combination its prefixes span, inbits rejections too), plus on
    part 0 what the head skips (head_skipped5)."""
    own = sum(hi - lo for j in deal.part_blocks(part, nparts, skip_excluded=False)
              for lo, hi in deal.block_ranges(j))
    return own + (head_skipped5(deal, excluded) if part == 0 else 0)


def search5_head(fused, two_first, n, nparts, head_off=False):
    """Whether search_5lut's sweep of a part ran with the fused kernel's chunk head: the fused
    kernel ran (`fused`), the head is not switched off (SBG_HEAD=0), n >= 128, and the part either
    started in the fused form or is the whole (a part that falls back from the two-kernel form keeps
    the prefix deal the other parts cut their shares by)."""
    return fused and not head_off and n >= 128 and (not two_first or nparts == 1)
