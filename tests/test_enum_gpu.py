"""GPU: sbg_enum5 / sbg_enum7 against the CPU enumeration oracle (tests/enum_oracle.c) and against
the library's own first-match searches.  Seeded synthetic states under mux masks of depth 0-3, with
and without gate 0 among the excluded input bits; 7-LUT comparisons with the oracle run on short
installed lists so that the oracle (0.3 s per list entry) finishes in seconds."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import _enum_reference as R
import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native

pytestmark = pytest.mark.gpu

K = 300          # matches compared record for record
MUX = [[], [(3, 1)], [(0, 0), (5, 1)], [(1, 1), (4, 0), (6, 1)]]

# (n, mask, excluded input bits); mask 0-3 = mux mask of that depth, larger = a random mask of that
# many positions, whose last 32-bit word is partly padding
CASES5 = [(12, 0, []), (12, 1, [0]), (12, 3, [2]), (16, 2, [0, 5]), (16, 3, []), (20, 1, []),
          (20, 2, [0]), (24, 0, [1]), (24, 1, [0, 2]), (16, 33, [0]), (20, 65, []), (20, 129, [0]),
          (24, 200, [])]
CASES7 = [(10, 0, []), (10, 2, [0]), (12, 1, [0, 3]), (12, 3, []), (14, 2, [0]), (14, 3, [4]),
          (12, 33, [0]), (14, 65, []), (12, 129, []), (10, 200, [0])]
LIST7 = 3        # list entries the 7-LUT oracle comparisons enumerate


def _mask(spec, seed):
    if spec < len(MUX):
        return S.mux_mask(MUX[spec])
    rs = np.random.RandomState(seed)
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, spec, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def _state(n, depth, inb, seed, width):
    """A synthetic state whose target is a random 2-LUT (width 5) or 3-LUT (width 7) circuit of
    gates that inbits allows, so that there is something to enumerate."""
    tabs = S.synthetic_state(n, seed=seed)
    rs = np.random.RandomState(seed)
    g = [int(x) for x in rs.choice([x for x in range(n) if x not in inb], width, replace=False)]
    f = [int(x) for x in rs.randint(1, 255, 3)]
    outer = S.lut_table(f[0], tabs[g[0]], tabs[g[1]], tabs[g[2]])
    mid = tabs[g[3]] if width == 5 else S.lut_table(f[1], tabs[g[3]], tabs[g[4]], tabs[g[5]])
    tgt = S.lut_table(f[2], outer, mid, tabs[g[-1]])
    return tabs, tgt, _mask(depth, seed), inb


def _states5():
    return [_state(n, d, inb, 9100 + i, 5) for i, (n, d, inb) in enumerate(CASES5)]


def _states7():
    return [_state(n, d, inb, 9200 + i, 7) for i, (n, d, inb) in enumerate(CASES7)]


def _pool():
    return ThreadPoolExecutor(max_workers=max(1, min(8, os.cpu_count() or 1)))


def _keys(e):
    return [int(k) for k in e.matches["key"]]


def _check_records(which, e, tabs, tgt, mask, order, middle=None, tuples=None):
    assert R.check_realises(e.matches, tabs, tgt, mask) == len(e.matches)
    for rec in e.matches[:60]:
        key = int(rec["key"])
        t7 = tuples[key >> 23] if which == 7 else None
        want = E.expected_record(which, key, tabs, tgt, mask, order, middle, t7)
        assert want is not None and E.record_fields(rec) == want, (which, hex(key))


def test_enum5_matches_oracle(engine):
    states = _states5()
    with _pool() as pool:
        wants = list(pool.map(lambda a: E.oracle_enum5(*a[1], E.orders(a[0])[0], K),
                              enumerate(states)))
    nonzero = 0
    for i, ((tabs, tgt, mask, inb), (total, keys, feasible)) in enumerate(zip(states, wants)):
        order = E.orders(i)[0]
        e = sb.enumerate_5lut(engine, tabs, tgt, mask, inb, order, K)
        assert (e.total, e.feasible) == (total, feasible), (i, e.total, total)
        assert _keys(e) == keys, i
        _check_records(5, e, tabs, tgt, mask, order)
        nonzero += total > 0
    assert nonzero >= 4


def test_enum7_matches_oracle_on_short_lists(engine):
    states = _states7()
    lists = []
    for tabs, tgt, mask, inb in states:
        engine.load(tabs, tgt, mask, inb)
        lists.append(engine.filter7_part(0, 1)[:LIST7])
    with _pool() as pool:
        wants = list(pool.map(
            lambda a: E.oracle_enum7(a[1][0], a[1][1], a[1][2], E.unpack_list(lists[a[0]]),
                                     *E.orders(a[0])[1:], K), enumerate(states)))
    nonzero = 0
    for i, ((tabs, tgt, mask, inb), (total, keys)) in enumerate(zip(states, wants)):
        _, outer, middle = E.orders(i)
        engine.load(tabs, tgt, mask, inb)
        engine.set_list7(lists[i])
        e = engine.enumerate7(outer, middle, K)
        assert (e.total, e.feasible) == (total, len(lists[i])), (i, e.total, total)
        assert _keys(e) == keys, i
        _check_records(7, e, tabs, tgt, mask, outer, middle, E.unpack_list(lists[i]))
        nonzero += total > 0
    assert nonzero >= 3


def test_first_match_is_the_search_result(engine):
    """min of the matches = sbg_search5 / sbg_search7's key (7-LUT: gate 0 excluded, so no stale
    cache row), counted and count-free with K = 1."""
    checked7 = 0
    for i, (tabs, tgt, mask, inb) in enumerate(_states5() + _states7()):
        order, outer, middle = E.orders(50 + i)
        engine.load(tabs, tgt, mask, inb)
        want5 = int(engine.search5(order).key)
        for count in (True, False):
            e = engine.enumerate5(order, 1, count=count)
            assert (_keys(e) or [native.SBG_KEY_NONE])[0] == want5, (i, count)
        if 0 not in inb or tabs.shape[0] < 7:
            continue
        engine.load(tabs, tgt, mask, inb)
        want7 = int(engine.search7(outer, middle).key)
        for count in (True, False):
            engine.load(tabs, tgt, mask, inb)   # phase 1 inside the enumeration
            e = engine.enumerate7(outer, middle, 1, count=count)
            assert (_keys(e) or [native.SBG_KEY_NONE])[0] == want7, (i, count)
        checked7 += 1
    assert checked7 >= 3


def test_shards_add_up(engine):
    for which, (tabs, tgt, mask, inb) in [(5, _states5()[6]), (5, _states5()[8]), (7, _states7()[3]),
                                          (7, _states7()[4])]:
        order, outer, middle = E.orders(7)
        engine.load(tabs, tgt, mask, inb)
        run = ((lambda p, q: engine.enumerate5(order, K, part=p, nparts=q)) if which == 5 else
               (lambda p, q: engine.enumerate7(outer, middle, K, part=p, nparts=q)))
        whole = run(0, 1)
        assert whole.total > 0, which
        for nparts in (2, 3):
            parts = [run(p, nparts) for p in range(nparts)]
            assert sum(p.total for p in parts) == whole.total, (which, nparts)
            merged = np.sort(np.concatenate([p.matches for p in parts]), order="key")[:K]
            assert np.array_equal(merged, whole.matches), (which, nparts)


def test_totals_do_not_depend_on_orders(engine):
    for i, (tabs, tgt, mask, inb) in enumerate(_states5()[3:7]):
        engine.load(tabs, tgt, mask, inb)
        t5 = {engine.enumerate5(E.orders(s)[0], 0).total for s in (1, 2, 3)}
        t7 = {engine.enumerate7(*E.orders(s)[1:], 0).total for s in (1, 2)}
        assert len(t5) == 1 and len(t7) == 1, (i, t5, t7)


@pytest.mark.parametrize("n", [64, 128])
def test_planted_circuits_larger_n(engine, n):
    """A planted 2-LUT (5 inputs) and 3-LUT (7 inputs) circuit is among the matches; every emitted
    match is rebuilt on the host with lut_table and checked with solve_inner under the mask."""
    tabs = S.synthetic_state(n, seed=640 + n)
    rs = np.random.RandomState(n)
    full = np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)
    g = [int(x) for x in rs.choice(n, 7, replace=False)]
    tgt5 = S.lut_table(0xCA, S.lut_table(0x96, tabs[g[0]], tabs[g[1]], tabs[g[2]]), tabs[g[3]],
                       tabs[g[4]])
    tgt7 = S.lut_table(0xE8, S.lut_table(0x96, tabs[g[0]], tabs[g[1]], tabs[g[2]]),
                       S.lut_table(0x6B, tabs[g[3]], tabs[g[4]], tabs[g[5]]), tabs[g[6]])
    order, outer, middle = E.orders(n)
    for which, tgt in ((5, tgt5), (7, tgt7)):
        for mask in (full, S.mux_mask([(2, 1)])):
            if which == 5:
                e = sb.enumerate_5lut(engine, tabs, tgt, mask, [], order, 500)
            else:
                e = sb.enumerate_7lut(engine, tabs, tgt, mask, [], outer, middle, 500)
            assert e.total >= 1 and len(e.matches) == min(e.total, 500), (which, n)
            keys = _keys(e)
            assert keys == sorted(set(keys))
            for rec in e.matches:
                gates, fo, fm, fi, seen = E.record_fields(rec)
                t1 = sb.lut_table(fo, tabs[gates[0]], tabs[gates[1]], tabs[gates[2]])
                t2 = tabs[gates[3]] if which == 5 else sb.lut_table(fm, *[tabs[x] for x in gates[3:6]])
                ok, f2, s2 = sb.solve_inner(t1, t2, tabs[gates[-1]], tgt, mask)
                assert ok and (f2, s2) == (fi, seen), (which, n, hex(int(rec["key"])))
                if which == 5:
                    assert order[(int(rec["key"]) >> 0) & 0xFF] == fo
                else:
                    assert (outer[(int(rec["key"]) >> 8) & 0xFF], middle[int(rec["key"]) & 0xFF]) \
                        == (fo, fm)


def test_small_ticket_table_gives_the_same_result(engine, monkeypatch):
    """SBG_TICKET_TABLE (read at handle creation) forces phase 1 into several segments; the list
    the enumeration runs on, and so its result, do not change."""
    tabs, tgt, mask, inb = _state(26, 2, [1], 9300, 7)
    _, outer, middle = E.orders(3)
    order = E.orders(3)[0]
    engine.load(tabs, tgt, mask, inb)
    want7 = engine.enumerate7(outer, middle, K)
    want5 = engine.enumerate5(order, K)
    monkeypatch.setenv("SBG_TICKET_TABLE", "4096")
    small = sb.LutEngine(0)
    try:
        small.load(tabs, tgt, mask, inb)
        got7 = small.enumerate7(outer, middle, K)
        got5 = small.enumerate5(order, K)
    finally:
        small.close()
    assert want7.total > 0
    assert (got7.total, got7.feasible) == (want7.total, want7.feasible)
    assert np.array_equal(got7.matches, want7.matches)
    assert got5.total == want5.total and np.array_equal(got5.matches, want5.matches)


def test_search_after_enumeration_is_unchanged(engine):
    fields = ("found", "key", "func_inner", "inner_seen", "tuples_feasible")
    fresh = sb.LutEngine(0)
    try:
        for tabs, tgt, mask, inb in (_states5()[4], _states7()[2]):
            order, outer, middle = E.orders(11)
            for eng in (fresh, engine):
                eng.load(tabs, tgt, mask, inb)
            engine.enumerate5(order, 10)
            engine.enumerate7(outer, middle, 10)
            for search in (lambda e: e.search5(order), lambda e: e.search7(outer, middle)):
                a, b = search(fresh), search(engine)
                assert [getattr(a, f) for f in fields] == [getattr(b, f) for f in fields]
                assert list(a.gates) == list(b.gates)
    finally:
        fresh.close()
