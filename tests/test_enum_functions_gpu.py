"""GPU: the function filter of the enumerations (sbg_enum_set_functions).  Under a filter,
sbg_enum3/5/7 must enumerate exactly the unfiltered matches whose LUTs pass match_functions_allowed,
in the same order with the same records: checked against a full unfiltered fetch filtered on the
host, against the CPU oracle's keys, with the depth filter, across shares, and on a planted circuit
at n = 128.  The depth tests' CASES run every function-filtered kernel form (width 3, 5, 7 at
NW = 1, 2, 4, 8 words per table)."""
import numpy as np
import pytest

import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native
from test_enum_depth_gpu import CASES, FULL_CAP, _all, _hist, _load, _mask, _nw, _random_depth, \
    _run
from test_oracle_large_gpu import _n40_state

pytestmark = pytest.mark.gpu

ERR_STATE = -4
AFF = sorted(sb.AFFINE_FUNCTIONS)
G194 = sorted(sb.gate_functions(194))


@pytest.fixture(autouse=True)
def _clear_filters(engine):
    """The session's engine leaves every test of this module without a filter."""
    yield
    engine.clear_function_filter()
    engine.clear_depth_filter()


def _allowed(recs, outer=None, middle=None, inner=None):
    """match_functions_allowed over an array of records, vectorised: the host reference."""
    width = recs["width"].astype(np.int64)
    ok = np.ones(len(recs), dtype=bool)
    if outer is not None:
        ok &= (width == 3) | np.isin(recs["func_outer"], list(outer))
    if middle is not None:
        ok &= (width != 7) | np.isin(recs["func_middle"], list(middle))
    if inner is not None:
        comp = np.zeros((256, 256), dtype=bool)    # [seen, ones]
        s = np.arange(256)
        for f in inner:
            comp[s, int(f) & s] = True
        ok &= comp[recs["inner_seen"].astype(np.int64), recs["func_inner"].astype(np.int64)]
    return ok


def _filters(full, width, seed):
    """The filters each case runs: one role at a time, affine, AND/OR/XOR, a single function in
    every role (taken from a match, so the set is not empty) and an empty set in one role."""
    rs = np.random.RandomState(seed)
    half = lambda: sorted(int(x) for x in rs.choice(256, 128, replace=False))  # noqa: E731
    mid = full[len(full) // 2]
    single = ([int(mid["func_outer"])], [int(mid["func_middle"])],
              [sb.allowed_fill(mid["func_inner"], mid["inner_seen"])])
    out = {"outer": (half(), None, None), "middle": (None, half(), None),
           "inner": (None, None, sorted(int(x) for x in rs.choice(256, 40, replace=False))),
           "affine": (AFF, AFF, AFF), "gates194": (G194, G194, G194), "single": single,
           "empty": (None, None, []) if width == 3 else ([], None, None)}
    return out


def _check(engine, width, orders, want, unf, k=200, seed=0):
    """The installed filter's count, first K, pages, picks and samples against `want`."""
    e = _run(engine, width, orders, k)
    assert e.total == len(want)
    assert e.feasible == unf.feasible
    assert e.matches.tobytes() == want[:k].tobytes()
    t = e.total
    for first in sorted({0, t // 3, max(t - 7, 0), t}):
        assert engine.fetch_matches(first, 64).tobytes() == want[first:first + 64].tobytes()
    if t:
        ranks = np.random.RandomState(seed).randint(0, t, 300)
        assert engine.pick_matches(ranks).tobytes() == want[ranks].tobytes()
        r, m = sb.sample_matches(engine, e, min(t, 100), seed=5)
        assert m.tobytes() == want[r.astype(np.int64)].tobytes()
    kk = min(t, 25) or 1
    free = _run(engine, width, orders, kk, count=False)
    assert free.matches.tobytes() == want[:kk].tobytes()
    return e


def test_cases_cover_every_function_form():
    forms = {(c[0], _nw(_mask(c[2], c[4]))) for c in CASES}
    assert forms == {(w, nw) for w in (3, 5, 7) for nw in (1, 2, 4, 8)}


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_filter_equals_post_filter(engine, case):
    width = case[0]
    _, orders = _load(engine, case)
    unf = _run(engine, width, orders, 0)
    full = _all(engine, width, orders)
    assert len(full) > 0
    for name, (o, m, i) in _filters(full, width, case[4]).items():
        ok = _allowed(full, o, m, i)
        for rec, v in zip(full[:40], ok[:40]):
            assert sb.match_functions_allowed(rec, o, m, i) == v
        engine.set_function_filter(o, m, i)
        _check(engine, width, orders, full[ok], unf, seed=case[4])
        if name == "single":
            assert ok.any()
        if name == "empty":
            assert not ok.any()


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_filtered_keys_match_oracle(engine, case):
    width, n = case[0], case[1]
    (tabs, tgt, mask, inb), orders = _load(engine, case)
    tuples = None
    if width == 3:
        total, keys = E.enum3_range(tabs, tgt, mask, orders[0], n * (n - 1) * (n - 2) // 6)
    elif width == 5:
        total, keys, _ = E.oracle_enum5(tabs, tgt, mask, inb, orders[0], FULL_CAP)
    else:
        tuples = E.unpack_list(engine.filter7_part(0, 1)[:3])
        engine.set_list7(engine.filter7_part(0, 1)[:3])
        total, keys = E.oracle_enum7(tabs, tgt, mask, tuples, *orders, FULL_CAP)
    assert len(keys) == total > 0
    arr = np.zeros(len(keys), dtype=sb.MATCH_DTYPE)
    arr["width"] = width
    for j, key in enumerate(keys):
        if width == 3:
            i3, k3, m3 = sb.decode_key3(key)
            g3 = [int(orders[0][x]) for x in (i3, k3, m3)]
            ok, fi, seen = sb.solve_inner(*[tabs[x] for x in g3], tgt, mask)
            assert ok
            fo = fm = 0
        else:
            rec = E.expected_record(width, int(key), tabs, tgt, mask, orders[0],
                                    orders[1] if width == 7 else None,
                                    tuples[int(key) >> 23] if width == 7 else None)
            _, fo, fm, fi, seen = rec
        arr[j]["func_outer"], arr[j]["func_middle"] = fo, fm
        arr[j]["func_inner"], arr[j]["inner_seen"] = fi, seen
    for o, m, i in ((AFF, AFF, None), (None, None, AFF), (G194, G194, G194)):
        engine.set_function_filter(o, m, i)
        e = _run(engine, width, orders, 0)
        got = engine.fetch_matches(0, e.total)
        want = [int(k) for k, v in zip(keys, _allowed(arr, o, m, i)) if v]
        assert [int(k) for k in got["key"]] == want


@pytest.mark.parametrize("case", CASES[::2], ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_neutral_and_ignored_roles(engine, case):
    width = case[0]
    _, orders = _load(engine, case)
    plain = _run(engine, width, orders, 300)
    everything = list(range(256))
    engine.set_function_filter(everything, everything, everything)
    e = _run(engine, width, orders, 300)
    assert (e.total, e.feasible) == (plain.total, plain.feasible)
    assert e.matches.tobytes() == plain.matches.tobytes()
    # roles the width does not have
    ignored = {3: ([], []), 5: (None, []), 7: None}[width]
    if ignored is not None:
        engine.set_function_filter(ignored[0], ignored[1], None)
        e = _run(engine, width, orders, 300)
        assert (e.total, e.matches.tobytes()) == (plain.total, plain.matches.tobytes())


@pytest.mark.parametrize("case", CASES[::3], ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_with_the_depth_filter(engine, case):
    width, n = case[0], case[1]
    _, orders = _load(engine, case)
    unf = _run(engine, width, orders, 0)
    full = _all(engine, width, orders)
    depth = _random_depth(n, case[4])
    dep = E.record_depths(full, depth)
    bound = int(np.median(dep))
    engine.set_depth_filter(depth, bound)
    unf_d = _run(engine, width, orders, 0)
    for o, m, i in ((AFF, AFF, None), (None, None, G194)):
        ok = _allowed(full, o, m, i)
        engine.set_function_filter(o, m, i)
        engine.set_depth_filter(depth, sb.SBG_DEPTH_BINS - 1)
        _run(engine, width, orders, 0)
        assert np.array_equal(engine.depth_counts(), _hist(dep[ok]))
        engine.set_depth_filter(depth, bound)
        want = full[ok & (dep <= bound)]
        _run(engine, width, orders, 0)
        assert np.array_equal(engine.depth_counts(), _hist(dep[ok & (dep <= bound)]))
        _check(engine, width, orders, want, unf_d, seed=bound)
        # shallowest_matches keeps the function filter
        dmin, count, recs = sb.shallowest_matches(engine, width, orders, depth, 50)
        if ok.any():
            assert dmin == int(dep[ok].min())
            sel = full[ok & (dep == dmin)]
            assert count == len(sel) and recs.tobytes() == sel[:50].tobytes()
        else:
            assert (dmin, count) == (None, 0)
        engine.clear_depth_filter()
    assert unf.total == len(full)


@pytest.mark.parametrize("nparts", [2, 3])
@pytest.mark.parametrize("case", [CASES[1], CASES[3], CASES[6]], ids=lambda c: "w%d" % c[0])
def test_shares_add_up(engine, case, nparts):
    width = case[0]
    engs = [sb.LutEngine(0) for _ in range(nparts)]
    try:
        _, orders = _load(engine, case)
        full = _all(engine, width, orders)
        mid = full[len(full) // 2]
        inner = sorted(set(range(128)) | {sb.allowed_fill(mid["func_inner"], mid["inner_seen"])})
        outer = sorted(set(AFF) | {int(mid["func_outer"])})
        engine.set_function_filter(outer, None, inner)
        whole_e = _run(engine, width, orders, 0)
        whole = engine.fetch_matches(0, whole_e.total)
        totals = []
        for q, e in enumerate(engs):
            _load(e, case)
            e.set_function_filter(outer, None, inner)
            fn = {3: e.enumerate3, 5: e.enumerate5, 7: e.enumerate7}[width]
            totals.append(fn(*orders, 0, True, q, nparts).total)
        assert sum(totals) == whole_e.total > 0
        counts = [e.enum_block_count() for e in engs]
        sums = np.zeros((nparts, max(max(counts), 1)), dtype=np.uint64)
        for q, e in enumerate(engs):
            sums[q, :counts[q]] = e.enum_block_sums()
        assert {e.enum_set_global(sums, counts) for e in engs} == {whole_e.total}
        t = whole_e.total
        for first in (0, t // 2):
            got = sum(e.fetch_matches(first, 100).view(np.uint64) for e in engs)
            assert got.tobytes() == whole[first:first + 100].tobytes()
        ranks = np.random.RandomState(1).randint(0, t, 200)
        got = sum(e.pick_matches(ranks).view(np.uint64) for e in engs)
        assert got.tobytes() == whole[ranks].tobytes()
    finally:
        for e in engs:
            e.close()


def test_searches_ignore_the_filter(engine):
    (tabs, tgt, mask, inb), (order,) = _load(engine, CASES[3])
    _, outer, middle = E.orders(CASES[3][4])
    go = [int(x) for x in np.random.RandomState(3).permutation(tabs.shape[0])]

    def res(r):
        return (r.found, r.key, r.ordering, list(r.gates), r.func_outer, r.func_middle,
                r.func_inner, r.inner_seen)

    def results():
        engine.load(tabs, tgt, mask, inb)
        r5, r7 = engine.search5(order), engine.search7(outer, middle)
        node = engine.search_node(0, order, outer, middle, go)
        batch = engine.search_batch([{"order5": order, "gate_order": go},
                                     {"outer": outer, "middle": middle, "order5": order}])
        return [res(r5), res(r7)] + [(x.found_stage, x.key3, list(x.gates3), res(x.r5), res(x.r7))
                                     for x in [node] + batch]

    want = results()
    engine.set_function_filter([], [], [])
    assert results() == want


def test_lifetime_and_errors(engine):
    _, (order,) = _load(engine, CASES[3])
    e = engine.enumerate5(order, 0)
    engine.fetch_matches(0, 1)
    engine.set_function_filter(AFF)
    with pytest.raises(RuntimeError):
        engine.fetch_matches(0, 1)       # set_function_filter ended the cursor
    f = engine.enumerate5(order, 0)
    assert f.total <= e.total
    if f.total:
        engine.fetch_matches(0, 1)
    # a function filter alone has no histogram
    out = np.zeros(4, dtype=np.uint64)
    assert engine.lib.sbg_enum_depth_counts(engine._h, out.ctypes.data_as(native.u64p), 4) \
        == ERR_STATE
    # all three NULL clears it, and ends the cursor even so
    assert engine.lib.sbg_enum_set_functions(engine._h, None, None, None) == 0
    with pytest.raises(RuntimeError):
        engine.fetch_matches(0, 1)
    assert engine.enumerate5(order, 0).total == e.total
    # an empty set is valid and leaves nothing; a NULL handle is refused
    empty = np.zeros(4, dtype=np.uint64)
    assert engine.lib.sbg_enum_set_functions(engine._h, None, None,
                                             empty.ctypes.data_as(native.u64p)) == 0
    assert engine.enumerate5(order, 0).total == 0
    assert engine.lib.sbg_enum_set_functions(None, None, None, None) != 0
    engine.clear_function_filter()
    assert engine.enumerate5(order, 0).total == e.total


def test_long_7lut_list(engine):
    """bench.py's n = 40 32-position state: 251,784 7-LUT matches, fetched whole and filtered."""
    tabs, tgt, mask, inb, outer, middle = _n40_state()
    engine.load(tabs, tgt, mask, inb)
    orders = (outer, middle)
    unf = _run(engine, 7, orders, 0)
    full = engine.fetch_matches(0, unf.total)
    assert len(full) == 251_784
    for o, m, i in ((AFF, AFF, None), (None, None, AFF), (G194, G194, G194)):
        ok = _allowed(full, o, m, i)
        engine.set_function_filter(o, m, i)
        _check(engine, 7, orders, full[ok], unf, k=1000, seed=7)


def test_planted_affine_circuit_at_n128(engine):
    """A 7-LUT circuit with affine outer and middle LUTs planted at n = 128: under that filter its
    key is found, and every record, completed by allowed_fill, computes the target under the mask."""
    n = 128
    tabs = S.synthetic_state(n, seed=640 + n)
    rs = np.random.RandomState(n + 1)
    g = [int(x) for x in rs.choice(n, 7, replace=False)]
    outer_t = S.lut_table(0x96, tabs[g[0]], tabs[g[1]], tabs[g[2]])
    middle_t = S.lut_table(0x3C, tabs[g[3]], tabs[g[4]], tabs[g[5]])
    tgt = S.lut_table(0xE8, outer_t, middle_t, tabs[g[6]])
    mask = np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)
    _, outer, middle = E.orders(n)
    engine.load(tabs, tgt, mask, [])
    engine.set_function_filter(AFF, AFF, None)
    e = _run(engine, 7, (outer, middle), 0)
    recs = engine.fetch_matches(0, min(e.total, 20000))
    assert e.total >= 1

    def planted(rec):
        gs = [int(x) for x in rec["gates"]]
        return {frozenset(gs[:3]), frozenset(gs[3:6])} == {frozenset(g[:3]), frozenset(g[3:6])} \
            and gs[6] == g[6]
    assert any(planted(r) for r in recs)
    for rec in recs[:2000]:
        assert int(rec["func_outer"]) in sb.AFFINE_FUNCTIONS
        assert int(rec["func_middle"]) in sb.AFFINE_FUNCTIONS
        gs = [int(x) for x in rec["gates"]]
        o = sb.lut_table(int(rec["func_outer"]), *[tabs[x] for x in gs[:3]])
        m = sb.lut_table(int(rec["func_middle"]), *[tabs[x] for x in gs[3:6]])
        fi = sb.allowed_fill(rec["func_inner"], rec["inner_seen"])
        out = sb.lut_table(fi, o, m, tabs[gs[6]])
        assert not np.any((out ^ tgt) & mask)
    # with the inner LUT restricted too, every record completes inside it
    engine.set_function_filter(AFF, AFF, G194)
    e2 = _run(engine, 7, (outer, middle), 0)
    for rec in engine.fetch_matches(0, min(e2.total, 2000)):
        fi = sb.allowed_fill(rec["func_inner"], rec["inner_seen"], G194)
        assert fi is not None and fi in G194
        gs = [int(x) for x in rec["gates"]]
        o = sb.lut_table(int(rec["func_outer"]), *[tabs[x] for x in gs[:3]])
        m = sb.lut_table(int(rec["func_middle"]), *[tabs[x] for x in gs[3:6]])
        assert not np.any((sb.lut_table(fi, o, m, tabs[gs[6]]) ^ tgt) & mask)
