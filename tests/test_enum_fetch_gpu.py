"""GPU: sbg_enum_fetch / sbg_enum_pick, the matches at any rank of the last counted enumeration.
Fetches and picks are compared with the records the counted call emits (K = total) on planted and
mux / random-mask states, and with closed forms (tests/_fetch_support.py) on states in which every
candidate matches, whose totals pass SBG_ENUM_MAX_MATCHES.  Also: the cursor's lifetime, shards,
the error codes and sample_matches."""
import ctypes as C

import numpy as np
import pytest

import _enum_reference as R
import _enum_support as E
import _fetch_support as F
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = -1, -4
MUX = [[], [(3, 1)], [(0, 0), (5, 1)], [(1, 1), (4, 0), (6, 1)]]


def _mask(spec, seed):
    if spec < len(MUX):
        return S.mux_mask(MUX[spec])
    rs = np.random.RandomState(seed)
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, spec, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def _planted(n, spec, inb, seed, width):
    """A synthetic state whose target is a planted circuit of `width` gates inbits allows."""
    tabs = S.synthetic_state(n, seed=seed)
    rs = np.random.RandomState(seed)
    g = [int(x) for x in rs.choice([x for x in range(n) if x not in inb], width, replace=False)]
    f = [int(x) for x in rs.randint(1, 255, 3)]
    if width == 3:
        tgt = S.lut_table(f[0], tabs[g[0]], tabs[g[1]], tabs[g[2]])
    else:
        outer = S.lut_table(f[0], tabs[g[0]], tabs[g[1]], tabs[g[2]])
        mid = tabs[g[3]] if width == 5 else S.lut_table(f[1], tabs[g[3]], tabs[g[4]], tabs[g[5]])
        tgt = S.lut_table(f[2], outer, mid, tabs[g[-1]])
    return tabs, tgt, _mask(spec, seed), inb


def _n40_state():
    """bench.py's n = 40 state under 32 positions (seed 1), rebuilt with the same draws: 251,784
    7-LUT matches over a 71,023-entry list."""
    rs = np.random.RandomState(1)
    for i in range(4):
        bits = rs.choice(8, i, replace=False)
        fixed = [(int(b), int(rs.randint(0, 2))) for b in bits]
        _, outer, middle = [bytes(rs.permutation(256).astype(np.uint8)) for _ in range(3)]
        seed = int(rs.randint(1 << 30))
    return (S.synthetic_state(40, seed), S.sbox_target(S.rijndael_sbox(), 0), S.mux_mask(fixed),
            [b for b, _ in fixed], outer, middle)


def _run(engine, width, orders, k, count=True, part=0, nparts=1):
    if width == 3:
        return engine.enumerate3(orders[0], k, count, part, nparts)
    if width == 5:
        return engine.enumerate5(orders[1], k, count, part, nparts)
    return engine.enumerate7(orders[2], orders[3], k, count, part, nparts)


def _orders(seed, n):
    o5, outer, middle = E.orders(seed)
    return [int(x) for x in np.random.RandomState(seed).permutation(n)], o5, outer, middle


def _tickets(width, keys, n):
    """Ticket of each key (nparts = 1): position pair, 3-gate prefix or list entry."""
    keys = np.asarray(keys, dtype=np.uint64)
    if width == 3:
        return (keys >> np.uint64(9)).astype(np.int64)
    if width == 7:
        return (keys >> np.uint64(23)).astype(np.int64)
    return [tuple(E.nth_comb(n, 5, int(k) >> 12)[:3]) for k in keys]


def _seams(tk):
    """Ranks at which a new ticket starts (after the first)."""
    return [i for i in range(1, len(tk)) if tk[i] != tk[i - 1]]


# (width, n, mask spec, inbits); mask spec 0-3 = mux depth, larger = random positions
CASES = [(3, 12, 0, []), (3, 20, 2, []), (3, 40, 65, []), (3, 64, 3, []),
         (5, 12, 1, [0]), (5, 16, 3, []), (5, 20, 33, [0]), (5, 24, 1, [0, 2]),
         (7, 10, 0, []), (7, 12, 1, [0, 3]), (7, 14, 2, [0]), (7, 12, 129, [])]


def _case_state(i):
    width, n, spec, inb = CASES[i]
    return width, _planted(n, spec, inb, 9500 + i, width), _orders(9600 + i, n)


def _check_against_whole(engine, width, n, whole, rs):
    total = len(whole)
    # pages at random (first, count)
    for _ in range(12):
        first = int(rs.randint(0, total))
        count = int(rs.randint(1, max(2, total // 3)))
        got = engine.fetch_matches(first, count)
        assert np.array_equal(got, whole[first:first + count]), (first, count)
    # pages starting and ending on ticket seams
    seams = _seams(_tickets(width, whole["key"], n))
    for a, b in zip([0] + seams[:6], seams[:6] + [total]):
        assert np.array_equal(engine.fetch_matches(a, b - a), whole[a:b]), (a, b)
        if b < total:
            assert np.array_equal(engine.fetch_matches(a, b - a + 1), whole[a:b + 1]), (a, b)
    # count = 0, first = total, first + count > total (n_out cut short)
    assert len(engine.fetch_matches(0, 0)) == 0
    assert len(engine.fetch_matches(total, 5)) == 0
    assert len(engine.fetch_matches(total + 1000, 5)) == 0
    tail = engine.fetch_matches(max(0, total - 3), 100)
    assert np.array_equal(tail, whole[max(0, total - 3):])
    # picks: unsorted, with duplicates, including 0 and total - 1
    ranks = np.concatenate([[total - 1, 0], rs.randint(0, total, 300), [0, total - 1],
                            rs.randint(0, total, 5).repeat(3)]).astype(np.int64)
    rs.shuffle(ranks)
    assert np.array_equal(engine.pick_matches(ranks), whole[ranks])


@pytest.mark.parametrize("case", range(len(CASES)))
def test_fetch_and_pick_agree_with_first_k(engine, case):
    width, (tabs, tgt, mask, inb), orders = _case_state(case)
    n = len(tabs)
    engine.load(tabs, tgt, mask, inb)
    total = _run(engine, width, orders, 0).total
    assert 1 <= total <= sb.native.SBG_ENUM_MAX_MATCHES, (case, total)
    whole = _run(engine, width, orders, total).matches
    assert len(whole) == total
    _check_against_whole(engine, width, n, whole, np.random.RandomState(case))
    # a count with K = 0 is as good a cursor
    assert _run(engine, width, orders, 0).total == total
    step = max(997, -(-total // 40))
    pages = [engine.fetch_matches(a, step) for a in range(0, total, step)]
    assert np.array_equal(np.concatenate(pages), whole)


def test_fetch_and_pick_on_the_long_7lut_list(engine):
    tabs, tgt, mask, inb, outer, middle = _n40_state()
    engine.load(tabs, tgt, mask, inb)
    e = engine.enumerate7(outer, middle, 0)
    assert (e.total, e.feasible) == (251_784, 71_023)
    whole = engine.enumerate7(outer, middle, e.total).matches
    assert R.check_realises(whole, tabs, tgt, mask) == e.total
    _check_against_whole(engine, 7, 40, whole, np.random.RandomState(40))
    engine.enumerate7(outer, middle, 0)
    assert np.array_equal(engine.fetch_matches(0, e.total), whole)


def _check_closed(engine, total, record, rs, picks, state):
    """First page, pages across rank 2**24, the last page, deep random pages, seeded picks; every
    record fetched or picked realises the target of `state` (tables, target, mask)."""
    firsts = [0, (1 << 24) - 2048, (1 << 24) - 1, 1 << 24, total - 4096] + \
        [int(x) for x in rs.randint(0, total - 600, 4)]
    for first in firsts:
        count = 4096 if first in (0, total - 4096) else 600
        got = engine.fetch_matches(first, count)
        assert len(got) == min(count, total - first)
        assert R.check_realises(got, *state, what=first) == len(got)
        for j in sorted({0, len(got) - 1} | {int(x) for x in rs.randint(0, len(got), 40)}):
            assert F.as_tuple(got[j]) == record(first + j), (first, j)
    ranks = np.random.default_rng(int(rs.randint(1 << 30))).choice(total, picks, replace=False)
    got = engine.pick_matches(ranks)
    assert R.check_realises(got, *state, what="picks") == len(got)
    for r, rec in zip(ranks, got):
        assert F.as_tuple(rec) == record(int(r)), int(r)


@pytest.mark.parametrize("p", [None, 150])
def test_3lut_n500_closed_form(engine, p):
    n = 500
    tabs = S.synthetic_state(n, seed=5000)
    tgt = S.sbox_target(S.rijndael_sbox(), 3)
    mask = np.zeros(4, dtype=np.uint64) if p is None else F.one_position_mask(p)
    order = [int(x) for x in np.random.RandomState(5001).permutation(n)]
    engine.load(tabs, tgt, mask, [])
    e = engine.enumerate3(order, 0)
    assert e.total == F.total3(n) == 20_708_500
    _check_closed(engine, e.total, lambda r: F.record3(r, tabs, tgt, mask, order),
                  np.random.RandomState(3), 10_000, (tabs, tgt, mask))


@pytest.mark.parametrize("n,inb,p", [(40, [], None), (40, [0, 2, 5], None), (64, [], None),
                                     (64, [1, 3, 4, 7], None), (40, [2], 9)])
def test_5lut_closed_form(engine, n, inb, p):
    tabs = S.synthetic_state(n, seed=5100 + n)
    tgt = S.sbox_target(S.rijndael_sbox(), 6)
    mask = np.zeros(4, dtype=np.uint64) if p is None else F.one_position_mask(p)
    order = E.orders(n + len(inb))[0]
    rows5 = S.order5_rows()
    engine.load(tabs, tgt, mask, inb)
    e = engine.enumerate5(order, 0)
    assert e.total == F.total5(n, inb) > (1 << 24)
    _check_closed(engine, e.total, lambda r: F.record5(r, tabs, tgt, mask, inb, order, rows5),
                  np.random.RandomState(n), 10_000, (tabs, tgt, mask))


@pytest.mark.parametrize("p", [None, 33])
def test_7lut_n40_closed_form(engine, p):
    n = 40
    tabs = S.synthetic_state(n, seed=5200)
    tgt = S.sbox_target(S.rijndael_sbox(), 4)
    mask = np.zeros(4, dtype=np.uint64) if p is None else F.one_position_mask(p)
    _, outer, middle = E.orders(77)
    rows7 = S.order7_rows()
    engine.load(tabs, tgt, mask, [])
    e = engine.enumerate7(outer, middle, 0)
    assert (e.total, e.feasible) == (F.total7(n, 100_000), 100_000)
    assert e.total == 458_752_000_000
    _check_closed(engine, e.total,
                  lambda r: F.record7(r, tabs, tgt, mask, outer, middle, rows7, 100_000),
                  np.random.RandomState(7), 10_000 if p is None else 2_000, (tabs, tgt, mask))


def _raw_fetch(engine, first, count, out=True, n_out=True):
    buf = np.zeros(max(count, 1), dtype=sb.MATCH_DTYPE)
    n = C.c_uint64(12345)
    rc = engine.lib.sbg_enum_fetch(engine._h, first, count,
                                   buf.ctypes.data_as(C.c_void_p) if out else None,
                                   C.byref(n) if n_out else None)
    return rc, n.value, buf


def _raw_pick(engine, ranks, nranks=None):
    r = np.ascontiguousarray(ranks, dtype=np.uint64)
    buf = np.full(max(len(r), 1) * 32, 0xAB, dtype=np.uint8)
    rc = engine.lib.sbg_enum_pick(engine._h, r.ctypes.data_as(native.u64p),
                                  len(r) if nranks is None else nranks,
                                  buf.ctypes.data_as(C.c_void_p))
    return rc, buf


def test_cursor_lifetime():
    width, (tabs, tgt, mask, inb), orders = _case_state(5)
    _, (tabs7, tgt7, mask7, inb7), orders7 = _case_state(10)
    eng = sb.LutEngine(0)
    try:
        assert _raw_fetch(eng, 0, 1)[0] == ERR_STATE
        assert _raw_pick(eng, [0])[0] == ERR_STATE
        eng.load(tabs, tgt, mask, inb)
        assert _raw_fetch(eng, 0, 1)[0] == ERR_STATE
        total = _run(eng, 5, orders, 0).total
        whole = _run(eng, 5, orders, total).matches
        # queries and settings keep the cursor
        eng.launches, eng.transfer_stats(), eng.kernel_ms(0)
        eng.set_timing(True)
        eng.set_timing(False)
        eng.set_stream(None)
        eng.lib.sbg_last_error(eng._h)
        hs = (C.c_double * 5)()
        assert eng.lib.sbg_host_seconds(eng._h, hs) == 0
        first = eng.fetch_matches(3, 50)
        for _ in range(5):
            assert np.array_equal(eng.fetch_matches(3, 50), first)
            assert np.array_equal(eng.pick_matches([7, 3, 7]), whole[[7, 3, 7]])
        assert np.array_equal(first, whole[3:53])
        # what ends it
        enders = [
            lambda: eng.load(tabs, tgt, mask, inb),
            lambda: eng.search5(orders[1]),
            lambda: eng.search_node(0, gate_order=orders[0]),
            lambda: eng.filter7_part(0, 1),
            lambda: eng.list7_device(),
            lambda: eng.use(0),
            lambda: _run(eng, 5, orders, 10, count=False),
            lambda: _run(eng, 3, orders, 10, count=False),
            lambda: _run(eng, 7, orders, 10, count=False),
            lambda: eng.alu_peak(),
        ]
        for i, end in enumerate(enders):
            eng.load(tabs, tgt, mask, inb)
            _run(eng, 5, orders, 0)
            assert _raw_fetch(eng, 0, 1)[0] == 0, i
            end()
            assert _raw_fetch(eng, 0, 1)[0] == ERR_STATE, i
            assert _raw_pick(eng, [0])[0] == ERR_STATE, i
        # a counted enumeration of another width replaces it
        eng.load(tabs, tgt, mask, inb)
        _run(eng, 5, orders, 0)
        e3 = _run(eng, 3, orders, 100)
        assert np.array_equal(eng.fetch_matches(0, 100), e3.matches)
        # a failing enumeration call ends it too
        _run(eng, 5, orders, 0)
        with pytest.raises(RuntimeError):
            eng.enumerate5(b"\0" * 256, 1)
        assert _raw_fetch(eng, 0, 1)[0] == ERR_STATE
    finally:
        eng.close()
    # after fetches and picks, search7 / enum7 on the same slot give what they give without them
    fresh, used = sb.LutEngine(0), sb.LutEngine(0)
    try:
        fields = ("found", "key", "func_inner", "inner_seen", "tuples_feasible")
        res = []
        for eng, fetch in ((fresh, False), (used, True)):
            eng.load(tabs7, tgt7, mask7, inb7)
            total = _run(eng, 7, orders7, 0).total
            if fetch:
                eng.fetch_matches(0, total)
                eng.pick_matches(np.arange(total)[::-1])
            r7 = eng.search7(orders7[2], orders7[3])
            e7 = _run(eng, 7, orders7, total)
            res.append(([getattr(r7, f) for f in fields], list(r7.gates), e7.total, e7.matches))
        assert res[0][:3] == res[1][:3]
        assert np.array_equal(res[0][3], res[1][3])
    finally:
        fresh.close()
        used.close()


@pytest.mark.parametrize("width", [3, 5, 7])
def test_shards_serve_their_own_ranks(engine, width):
    case = {3: 1, 5: 7, 7: 9}[width]
    _, (tabs, tgt, mask, inb), orders = _case_state(case)
    engine.load(tabs, tgt, mask, inb)
    total = _run(engine, width, orders, 0).total
    whole = _run(engine, width, orders, total).matches
    for nparts in (2, 3, 7):
        got = []
        for part in range(nparts):
            ref = _run(engine, width, orders, total, part=part, nparts=nparts)
            _run(engine, width, orders, 0, part=part, nparts=nparts)
            mine = engine.fetch_matches(0, ref.total)
            assert np.array_equal(mine, ref.matches), (nparts, part)
            if ref.total:
                r = np.random.RandomState(part).randint(0, ref.total, 20)
                assert np.array_equal(engine.pick_matches(r), ref.matches[r]), (nparts, part)
            got.append(mine)
        merged = np.sort(np.concatenate(got), order="key")
        assert np.array_equal(merged, whole), nparts


def test_errors(engine):
    _, (tabs, tgt, mask, inb), orders = _case_state(4)
    engine.load(tabs, tgt, mask, inb)
    total = _run(engine, 5, orders, 0).total
    big = sb.native.SBG_ENUM_MAX_MATCHES
    buf = np.zeros(1, dtype=sb.MATCH_DTYPE)
    n = C.c_uint64()
    assert engine.lib.sbg_enum_fetch(engine._h, 0, big + 1, buf.ctypes.data_as(C.c_void_p),
                                     C.byref(n)) == ERR_ARG
    assert _raw_fetch(engine, 0, 5, out=False)[0] == ERR_ARG
    assert _raw_fetch(engine, 0, 5, n_out=False)[0] == ERR_ARG
    rc, n_out, _ = _raw_fetch(engine, 0, 0, out=False)
    assert (rc, n_out) == (0, 0)
    assert _raw_pick(engine, [0], nranks=big + 1)[0] == ERR_ARG
    assert engine.lib.sbg_enum_pick(engine._h, None, 3, buf.ctypes.data_as(C.c_void_p)) == ERR_ARG
    rc, out = _raw_pick(engine, [0, 1, total, 2])
    assert rc == ERR_ARG and np.all(out == 0xAB)
    rc, out = _raw_pick(engine, [total - 1, 2**64 - 1])
    assert rc == ERR_ARG and np.all(out == 0xAB)
    # the cursor survives the refused calls
    assert np.array_equal(engine.pick_matches([total - 1]), engine.fetch_matches(total - 1, 1))
    with pytest.raises(ValueError):
        engine.fetch_matches(0, big + 1)
    with pytest.raises(ValueError):
        engine.pick_matches(np.zeros((2, 2), dtype=np.int64))
    with pytest.raises(ValueError):
        engine.pick_matches([0.5])
    with pytest.raises(ValueError):
        engine.pick_matches([-1])
    with pytest.raises(RuntimeError):
        engine.pick_matches([total])


def test_sample_matches(engine):
    _, (tabs, tgt, mask, inb), orders = _case_state(6)
    engine.load(tabs, tgt, mask, inb)
    e = _run(engine, 5, orders, 0)
    whole = _run(engine, 5, orders, e.total).matches
    ranks, recs = sb.sample_matches(engine, e, 500, seed=11)
    assert len(np.unique(ranks)) == 500 and np.all(np.diff(ranks.astype(np.int64)) > 0)
    assert int(ranks.max()) < e.total
    assert np.array_equal(recs, whole[ranks.astype(np.int64)])
    assert np.array_equal(recs, engine.pick_matches(ranks))
    again, recs2 = sb.sample_matches(engine, e, 500, seed=11)
    assert np.array_equal(ranks, again) and np.array_equal(recs, recs2)
    with pytest.raises(ValueError):
        sb.sample_matches(engine, e, e.total + 1, seed=1)
    with pytest.raises(ValueError):
        sb.sample_matches(engine, _run(engine, 5, orders, 1, count=False), 1, seed=1)
