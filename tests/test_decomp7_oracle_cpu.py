"""CPU: the host-side phase-2 helpers of tests/_enum_support.py (decomp7_range, decomp7_key, the
per-entry and per-part keys, expected_result7) against orc_decomp7_key of whole lists and against
the reference's own answers in tests/golden/ref_cases.bin."""
import os

import numpy as np

import _enum_support as E
import _support as S
from sboxgates_b200.lut import _fill, shuffled_orders7
from sboxgates_b200.rng import Xorshift1024

NONE = E.NONE


def _cases():
    """(tables, target, mask, list, outer, middle): dense lists with matches in many rows, stale pairs
    whose target is planted on the stale tables, and windows of a real phase-1 list."""
    rs = np.random.RandomState(77)
    for i, (n, fixed) in enumerate([(24, [(0, 1), (3, 0)]), (40, [(6, 1)])]):
        tabs = S.synthetic_state(n, seed=900 + i)
        mask = S.mux_mask(fixed)
        outer, middle = shuffled_orders7(Xorshift1024(rs.bytes(128)))
        pairs = E.stale_pairs(rs, n, 2)
        # the target runs on the stale outer tables of the second entry of pair 1, row 2
        cur, prev = pairs[3], pairs[2]
        tgt = E.planted7(tabs, cur, 2, 0x96, 0xE8, 0xCA, stale_gate=prev[1])
        lst = np.array(sorted(pairs), dtype=np.uint16)
        yield tabs, tgt, mask, lst, outer, middle
        # a window of the phase-1 list under a 3-LUT of three gates (matches in many entries)
        tgt = S.lut_table(0x6A, tabs[1], tabs[n // 2], tabs[n - 1])
        full, _ = S.oracle_filter7(tabs, tgt, mask, [], cap=200)
        assert len(full) >= 40
        start = int(rs.randint(0, len(full) - 20))
        yield tabs, tgt, mask, full[:start + 20], outer, middle


def test_ranges_entries_and_parts_agree_with_the_whole_list():
    stale_seen = 0
    for tabs, tgt, mask, lst, outer, middle in _cases():
        whole = S.oracle_decomp7_key(tabs, tgt, mask, lst, outer, middle)
        assert E.decomp7_key(tabs, tgt, mask, lst, outer, middle, piece=5) == whole
        entry = E.decomp7_entry_keys(tabs, tgt, mask, lst, outer, middle)
        assert min(entry) == whole
        for i, key in enumerate(entry):
            assert key == NONE or key >> 23 == i
        # cuts at every stale entry (its outer cache comes from the entry before the cut) and at
        # random places
        rs = np.random.RandomState(len(lst))
        stale = [i for i in range(1, len(lst)) if E.stale_source(lst, i, 0) is not None]
        stale_seen += len(stale)
        cuts = sorted(set(stale) | {int(x) for x in rs.randint(1, len(lst), 3)})
        bounds = [0] + cuts + [len(lst)]
        got = [E.decomp7_range(tabs, tgt, mask, lst, outer, middle, a, b)
               for a, b in zip(bounds, bounds[1:])]
        assert min(got) == whole
        for a, b, key in zip(bounds, bounds[1:], got):
            assert key == min(entry[a:b], default=NONE)
        for nparts in (3, len(lst) + 3):
            want = E.part_keys(entry, nparts)
            for p in range(nparts):
                assert S.oracle_decomp7_key(tabs, tgt, mask, lst, outer, middle, p, nparts) == want[p]
    assert stale_seen >= 4


def test_a_stale_entry_is_decided_on_its_predecessors_tables():
    """The planted stale-row target matches at the stale entry only with its predecessor in place:
    decided alone (no predecessor) the entry's first match is elsewhere or absent."""
    tabs, tgt, mask, lst, outer, middle = next(_cases())
    i = 3
    assert E.stale_source(lst, i, 2) is not None
    key = E.decomp7_range(tabs, tgt, mask, lst, outer, middle, i, i + 1)
    assert key != NONE and key >> 23 == i and (key >> 16) & 0x7F < 4
    alone = S.oracle_decomp7_key(tabs, tgt, mask, lst[i:i + 1], outer, middle)
    assert alone == NONE or (alone & ((1 << 23) - 1)) != (key & ((1 << 23) - 1))
    res = E.expected_result7(key, lst, tabs, tgt, mask, outer, middle)
    assert res["stale_outer"] == 1 and res["index"] == i


def test_expected_result7_reproduces_the_reference_cases():
    """Every 7-LUT call of ref_cases.bin (answered by the reference's own object code): the oracle's
    list and key, expected_result7 and the don't-care fill give the recorded ret[10] and draws."""
    recs = [r for r in S.read_records(os.path.join(S.GOLDEN, "ref_cases.bin")) if r.which == 7]
    assert recs
    stale = found = 0
    for rec in recs:
        rng = Xorshift1024.from_state(rec.rng_s, rec.rng_p)
        outer, middle = shuffled_orders7(rng)
        lst, _ = S.oracle_filter7(rec.tables, rec.target, rec.mask, rec.inbits_list())
        key = E.decomp7_key(rec.tables, rec.target, rec.mask, lst, outer, middle)
        res = E.expected_result7(key, lst, rec.tables, rec.target, rec.mask, outer, middle)
        assert (res is not None) == rec.found == (key != NONE)
        if res is None:
            assert rec.ret == [0] * 10
        else:
            fi = _fill(res["func_inner"], res["inner_seen"], rng)
            assert [res["func_outer"], res["func_middle"], fi] + res["gates"] == rec.ret
            stale += res["stale_outer"]
            found += 1
        assert rng.draws == rec.draws
    assert found > 0 and stale >= 3, (found, stale)   # answers that came from a stale-cache row
