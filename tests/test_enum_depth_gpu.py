"""GPU: the depth filter of the enumerations (sbg_enum_set_depth / sbg_enum_depth_counts).  Under a
filter, sbg_enum3/5/7 must enumerate exactly the unfiltered matches of depth <= max_depth, in the
same order with the same records: checked against a full unfiltered fetch filtered on the host,
against the CPU oracle's keys, across shares, and on planted circuits at n = 128.  CASES run every
filtered kernel form (width 3, 5, 7 at NW = 1, 2, 4, 8 words per table); the edges of the filter
are in test_enum_depth_edges_gpu.py."""
import ctypes as C

import numpy as np
import pytest

import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = -1, -4
MUX = [[], [(3, 1)], [(0, 0), (5, 1)], [(1, 1), (4, 0), (6, 1)]]
LIST7 = 20       # list entries of the 7-LUT states (installed with set_list7)
FULL_CAP = 1 << 21


@pytest.fixture(autouse=True)
def _clear_filter(engine):
    """The session's engine leaves every test of this module without a filter."""
    yield
    engine.clear_depth_filter()


def _state(n, mask_spec, inb, seed, width):
    """A seeded state whose target is a random LUT circuit of allowed gates (as test_enum_gpu)."""
    tabs = S.synthetic_state(n, seed=seed)
    rs = np.random.RandomState(seed)
    k = max(width, 3)
    g = [int(x) for x in rs.choice([x for x in range(n) if x not in inb], k, replace=False)]
    f = [int(x) for x in rs.randint(1, 255, 3)]
    if width == 3:
        tgt = S.lut_table(f[0], tabs[g[0]], tabs[g[1]], tabs[g[2]])
    else:
        outer = S.lut_table(f[0], tabs[g[0]], tabs[g[1]], tabs[g[2]])
        mid = tabs[g[3]] if width == 5 else S.lut_table(f[1], tabs[g[3]], tabs[g[4]], tabs[g[5]])
        tgt = S.lut_table(f[2], outer, mid, tabs[g[-1]])
    return tabs, tgt, _mask(mask_spec, seed), inb


def _mask(spec, seed):
    """A mux mask of depth `spec` (0 - 3: 256 >> spec positions), or "r<count>": a seeded random mask
    of that many positions, whose last 32-bit word is partly padding."""
    if not isinstance(spec, str):
        return S.mux_mask(MUX[spec])
    rs = np.random.RandomState(1000 + seed)
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, int(spec[1:]), replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def _nw(mask):
    """The library's 32-bit words per compressed table for a mask: 1, 2, 4 or 8."""
    m = sum(bin(int(w)).count("1") for w in mask)
    return 1 if m <= 32 else 2 if m <= 64 else 4 if m <= 128 else 8


# (width, n, mask: mux depth or random "r<positions>", excluded inputs, seed).  Every width meets
# every word count NW (mux depth 3, 2, 1, 0 -> NW 1, 2, 4, 8) and one padded random mask.
CASES = [(3, 24, 2, [], 11), (3, 40, 3, [], 12), (5, 12, 2, [0], 13), (5, 16, 3, [], 14),
         (5, 20, 1, [2], 15), (7, 10, 2, [0], 16), (7, 12, 1, [], 17), (7, 14, 2, [1], 18),
         (3, 32, 1, [], 19), (3, 20, 0, [], 20), (3, 28, "r65", [1], 21), (5, 14, 0, [], 22),
         (5, 16, "r200", [0], 23), (7, 12, 3, [1], 36), (7, 12, 0, [0], 33), (7, 12, "r33", [], 30)]


def _load(engine, case):
    width, n, ms, inb, seed = case
    tabs, tgt, mask, inb = _state(n, ms, inb, seed, width)
    engine.load(tabs, tgt, mask, inb)
    rs = np.random.RandomState(seed)
    go = rs.permutation(n).astype(np.uint16)
    order, outer, middle = E.orders(seed)
    if width == 7:
        engine.set_list7(engine.filter7_part(0, 1)[:LIST7])
    orders = {3: (go,), 5: (order,), 7: (outer, middle)}[width]
    return (tabs, tgt, mask, inb), orders


def _run(engine, width, orders, k, count=True):
    fn = {3: engine.enumerate3, 5: engine.enumerate5, 7: engine.enumerate7}[width]
    return fn(*orders, k, count)


def _all(engine, width, orders):
    e = _run(engine, width, orders, 0)
    assert e.total <= FULL_CAP
    return engine.fetch_matches(0, e.total) if e.total else np.zeros(0, dtype=sb.MATCH_DTYPE)


def _hist(depths):
    return np.bincount(depths, minlength=1).astype(np.uint64)[:int(depths.max()) + 1] \
        if depths.size else np.zeros(0, dtype=np.uint64)


def _random_depth(n, seed):
    return np.random.RandomState(seed).randint(0, 7, n).astype(np.uint16)


def test_cases_cover_every_filtered_form():
    """Each of the 12 (width, NW) forms of the filtered kernels meets the host reference in CASES,
    and each width also runs a random mask whose last 32-bit word is partly padding."""
    forms = {(c[0], _nw(_mask(c[2], c[4]))) for c in CASES}
    assert forms == {(w, nw) for w in (3, 5, 7) for nw in (1, 2, 4, 8)}
    padded = {c[0] for c in CASES if isinstance(c[2], str)
              and sum(bin(int(x)).count("1") for x in _mask(c[2], c[4])) % 32 != 0}
    assert padded == {3, 5, 7}


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_filter_equals_post_filter(engine, case):
    width = case[0]
    _, orders = _load(engine, case)
    engine.clear_depth_filter()
    full = _all(engine, width, orders)
    assert len(full) > 0
    depth = _random_depth(case[1], case[4])
    dep = E.record_depths(full, depth)
    engine.set_depth_filter(depth, sb.SBG_DEPTH_BINS - 1)
    e = _run(engine, width, orders, 50)
    assert e.total == len(full)
    assert np.array_equal(engine.depth_counts(), _hist(dep))
    lo = int(dep.min())
    for bound in sorted({lo - 1, lo, int(np.median(dep)), int(dep.max()) - 1, int(dep.max())}):
        want = full[dep <= bound]
        engine.set_depth_filter(depth, bound)
        e = _run(engine, width, orders, 200)
        assert e.total == len(want), (case, bound)
        assert e.matches.tobytes() == want[:200].tobytes(), (case, bound)
        assert np.array_equal(engine.depth_counts(), _hist(dep[dep <= bound]))
        t = e.total
        for first in sorted({0, t // 3, max(t - 7, 0), t}):
            assert engine.fetch_matches(first, 64).tobytes() == want[first:first + 64].tobytes()
        if t:
            ranks = np.random.RandomState(bound + 1).randint(0, t, 300)
            assert engine.pick_matches(ranks).tobytes() == want[ranks].tobytes()
            r, m = sb.sample_matches(engine, e, min(t, 100), seed=5)
            assert m.tobytes() == want[r.astype(np.int64)].tobytes()


def _key_depth(width, key, depth, n, orders, tuples):
    if width == 3:
        i, k, m = sb.decode_key3(key)
        g = [int(orders[0][x]) for x in (i, k, m)]
        return 1 + max(int(depth[x]) for x in g)
    if width == 5:
        rank, k, _ = sb.decode_key5(key)
        comb = E.nth_comb(n, 5, rank)
        d = [int(depth[comb[i]]) for i in S.order5_rows()[k]]
        return 1 + max(1 + max(d[:3]), d[3], d[4])
    idx, k, _, _ = sb.decode_key7(key)
    d = [int(depth[int(tuples[idx][i])]) for i in S.order7_rows()[k]]
    return 1 + max(1 + max(d[:3]), 1 + max(d[3:6]), d[6])


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
    depth = _random_depth(n, case[4] + 100)
    kd = np.array([_key_depth(width, k, depth, n, orders, tuples) for k in keys], dtype=np.int64)
    for bound in sorted({int(np.median(kd)), int(kd.min())}):
        engine.set_depth_filter(depth, bound)
        e = _run(engine, width, orders, 0)
        got = engine.fetch_matches(0, e.total)
        assert [int(k) for k in got["key"]] == [k for k, d in zip(keys, kd) if d <= bound]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_neutral_filter_changes_nothing(engine, case):
    width, n = case[0], case[1]
    _, orders = _load(engine, case)
    engine.clear_depth_filter()
    plain = _run(engine, width, orders, 300)
    engine.set_depth_filter(np.zeros(n, dtype=np.uint16), 3)
    filt = _run(engine, width, orders, 300)
    assert (filt.total, filt.feasible) == (plain.total, plain.feasible)
    assert filt.matches.tobytes() == plain.matches.tobytes()
    first = _run(engine, width, orders, 1, count=False)
    assert first.matches.tobytes() == plain.matches[:1].tobytes()
    if not plain.total:
        return
    key = int(plain.matches["key"][0])
    if width == 3:
        assert engine.search_node(0, gate_order=[int(x) for x in orders[0]]).key3 == key
    elif width == 5:
        assert engine.search5(orders[0]).key == key
    elif 0 in case[3]:
        assert engine.search7(*orders).key == key


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_excluded_gate_and_count_free(engine, case):
    width, n = case[0], case[1]
    _, orders = _load(engine, case)
    engine.clear_depth_filter()
    full = _all(engine, width, orders)
    used = np.unique(full["gates"][:, :width]) if len(full) else np.zeros(0, dtype=np.uint16)
    for g in used[:3]:
        depth = _random_depth(n, case[4] + 7)
        depth[g] = native.SBG_MAX_DEPTH
        engine.set_depth_filter(depth, 20)
        e = _run(engine, width, orders, 0)
        got = engine.fetch_matches(0, e.total)
        assert not np.any(got["gates"][:, :width] == g)
        want = full[~np.any(full["gates"][:, :width] == g, axis=1)]
        assert got.tobytes() == want.tobytes()
        k = min(e.total, 25) or 1
        assert _run(engine, width, orders, k, count=False).matches.tobytes() == want[:k].tobytes()


@pytest.mark.parametrize("nparts", [2, 3])
@pytest.mark.parametrize("case", [CASES[1], CASES[3], CASES[6]], ids=lambda c: "w%d" % c[0])
def test_shares_add_up(engine, case, nparts):
    width, n = case[0], case[1]
    depth = _random_depth(n, case[4] + 3)
    engs = [sb.LutEngine(0) for _ in range(nparts)]
    try:
        _, orders = _load(engine, case)
        engine.set_depth_filter(depth, sb.SBG_DEPTH_BINS - 1)
        _run(engine, width, orders, 0)
        hist_all = engine.depth_counts()
        bound = int(np.flatnonzero(hist_all)[len(np.flatnonzero(hist_all)) // 2])
        engine.set_depth_filter(depth, bound)
        whole_e = _run(engine, width, orders, 0)
        whole = engine.fetch_matches(0, whole_e.total)
        whole_hist = engine.depth_counts()
        hists, totals = [], []
        for q, e in enumerate(engs):
            _load(e, case)
            e.set_depth_filter(depth, bound)
            fn = {3: e.enumerate3, 5: e.enumerate5, 7: e.enumerate7}[width]
            totals.append(fn(*orders, 0, True, q, nparts).total)
            h = np.zeros(sb.SBG_DEPTH_BINS, dtype=np.uint64)
            hq = e.depth_counts()
            h[:len(hq)] = hq
            hists.append(h)
        assert sum(totals) == whole_e.total
        summed = np.sum(hists, axis=0)
        assert np.array_equal(summed[:len(whole_hist)], whole_hist)
        assert not summed[len(whole_hist):].any()
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

    engine.clear_depth_filter()
    want = results()
    depth = np.full(tabs.shape[0], native.SBG_MAX_DEPTH, dtype=np.uint16)
    engine.set_depth_filter(depth, 0)
    assert results() == want


def test_lifetime_and_errors(engine):
    (tabs, tgt, mask, inb), (order,) = _load(engine, CASES[3])
    n = tabs.shape[0]
    # a cursor counted without a filter has no histogram; no cursor at all: the same code
    engine.clear_depth_filter()
    engine.enumerate5(order, 0)
    out = np.zeros(4, dtype=np.uint64)
    assert engine.lib.sbg_enum_depth_counts(engine._h, out.ctypes.data_as(native.u64p), 4) \
        == ERR_STATE
    engine.fetch_matches(0, 1)   # the refused call kept the cursor
    engine.set_depth_filter(np.zeros(n, dtype=np.uint16), 5)
    with pytest.raises(RuntimeError):
        engine.fetch_matches(0, 1)       # set_depth_filter ended the cursor
    assert engine.lib.sbg_enum_depth_counts(engine._h, out.ctypes.data_as(native.u64p), 4) \
        == ERR_STATE
    e = engine.enumerate5(order, 0)
    assert int(engine.depth_counts().sum()) == e.total
    assert engine.lib.sbg_enum_depth_counts(engine._h, out.ctypes.data_as(native.u64p),
                                            sb.SBG_DEPTH_BINS + 1) == ERR_ARG
    # a filter of the wrong length is refused by the enumeration, not by the installation
    engine.set_depth_filter(np.zeros(n + 1, dtype=np.uint16), 5)
    with pytest.raises(RuntimeError, match=r"code -1"):
        engine.enumerate5(order, 0)
    # a depth above SBG_MAX_DEPTH: the library refuses it and keeps the filter it had
    bad = (C.c_uint16 * n)(*([0] * (n - 1) + [native.SBG_MAX_DEPTH + 1]))
    assert engine.lib.sbg_enum_set_depth(engine._h, bad, n, 5) == ERR_ARG
    with pytest.raises(ValueError):
        engine.set_depth_filter(np.full(n, native.SBG_MAX_DEPTH + 1), 5)
    with pytest.raises(RuntimeError, match=r"code -1"):
        engine.enumerate5(order, 0)
    engine.clear_depth_filter()
    assert engine.enumerate5(order, 0).total == e.total


def test_shallowest_planted_circuits_at_n128(engine):
    """A planted 5-LUT and 7-LUT circuit at n = 128 (as test_planted_circuits_larger_n), the planted
    gates at depth 0 and every other gate at depth 5: the shallowest matches are the planted gates'."""
    n = 128
    tabs = S.synthetic_state(n, seed=640 + n)
    rs = np.random.RandomState(n)
    full = np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)
    g = [int(x) for x in rs.choice(n, 7, replace=False)]
    tgt5 = S.lut_table(0xCA, S.lut_table(0x96, tabs[g[0]], tabs[g[1]], tabs[g[2]]), tabs[g[3]],
                       tabs[g[4]])
    tgt7 = S.lut_table(0xE8, S.lut_table(0x96, tabs[g[0]], tabs[g[1]], tabs[g[2]]),
                       S.lut_table(0x6B, tabs[g[3]], tabs[g[4]], tabs[g[5]]), tabs[g[6]])
    order, outer, middle = E.orders(n)
    for width, tgt, orders in ((5, tgt5, (order,)), (7, tgt7, (outer, middle))):
        depth = np.full(n, 5, dtype=np.uint16)
        depth[g[:width]] = 0
        engine.load(tabs, tgt, full, [])
        dmin, count, recs = sb.shallowest_matches(engine, width, orders, depth, 1000)
        assert dmin == 2 and count == len(recs) >= 1, (width, dmin, count)
        for rec in recs:
            assert sorted(int(x) for x in rec["gates"][:width]) == sorted(g[:width])
            assert sb.match_depth(rec, depth) == 2
        # the planted decomposition: outer LUT 0x96 (symmetric) over g0..g2; reference order lists
        # each LUT's inputs ascending, and for width 7 the LUT with the smaller first input first
        def planted(rec):
            gs = [int(x) for x in rec["gates"][:width]]
            if width == 5:
                return sorted(gs[:3]) == sorted(g[:3]) and int(rec["func_outer"]) == 0x96
            groups = {frozenset(gs[:3]), frozenset(gs[3:6])}
            return groups == {frozenset(g[:3]), frozenset(g[3:6])} and gs[6] == g[6] \
                and 0x96 in (int(rec["func_outer"]), int(rec["func_middle"]))
        assert any(planted(rec) for rec in recs), width
        # the cursor holds the shallowest set
        assert engine.fetch_matches(0, count).tobytes() == recs.tobytes()
