"""GPU: grouped enumeration (sbg_enum_set_grouping).  Under a grouping, sbg_enum5/7 must enumerate
exactly the first match of each group (the matches sharing match_group's id), with the ungrouped
records, in key order: checked against a full ungrouped fetch grouped on the host, on every kernel
form (the depth tests' CASES: widths 3, 5, 7 at NW = 1, 2, 4, 8), under the function and depth
filters, against the CPU oracle's keys, across shares and over gloo, against the closed forms of
the empty mask at n = 40, and on bench.py's n = 40 state.  Width 3 must be unchanged."""
import ctypes as C
import os
import socket

import numpy as np
import pytest

import _enum_reference as R
import _enum_support as E
import _fetch_support as F
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native
from test_enum_depth_gpu import CASES, FULL_CAP, _all, _hist, _load, _random_depth, _run, _state
from test_enum_functions_gpu import _allowed, _filters
from test_oracle_large_gpu import _n40_state

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = -1, -4
GROUPINGS = ("shape", "tuple")
SHIFT = {("shape", 5): 8, ("shape", 7): 16, ("tuple", 5): 12, ("tuple", 7): 23}


@pytest.fixture(autouse=True)
def _reset(engine):
    """The session's engine leaves every test of this module ungrouped and unfiltered."""
    yield
    engine.set_grouping(None)
    engine.clear_function_filter()
    engine.clear_depth_filter()


def _group_ids(keys, width, grouping):
    keys = np.asarray(keys, dtype=np.uint64)
    if grouping is None or width == 3:
        return keys
    return keys >> np.uint64(SHIFT[(grouping, width)])


def _grouped(recs, width, grouping):
    """The host reference: the first record of each run of equal group ids (records in key order)."""
    if len(recs) == 0:
        return recs
    ids = _group_ids(recs["key"], width, grouping)
    for r, i in zip(recs[::max(1, len(recs) // 50)], ids[::max(1, len(recs) // 50)]):
        assert sb.match_group(int(r["key"]), width, grouping) == int(i)
    keep = np.ones(len(recs), dtype=bool)
    keep[1:] = ids[1:] != ids[:-1]
    return recs[keep]


def _check(engine, width, orders, want, feasible, k=200, seed=0):
    """The installed grouping's count, first K, pages, picks, sample and count-free first K."""
    e = _run(engine, width, orders, k)
    assert e.total == len(want)
    assert e.feasible == feasible
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


def _each_grouping(engine, width, orders, recs, feasible, seed):
    """Both groupings against the host grouping of `recs` (the ungrouped set under the installed
    filters); returns the grouped sets."""
    out = {}
    for g in GROUPINGS:
        want = _grouped(recs, width, g)
        if width == 3:
            assert want.tobytes() == recs.tobytes()
        engine.set_grouping(g)
        _check(engine, width, orders, want, feasible, seed=seed)
        engine.set_grouping(None)
        out[g] = want
    return out


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_grouped_equals_post_grouped(engine, case):
    width = case[0]
    _, orders = _load(engine, case)
    unf = _run(engine, width, orders, 0)
    full = _all(engine, width, orders)
    assert len(full) > 0
    got = _each_grouping(engine, width, orders, full, unf.feasible, case[4])
    if width != 3:
        # a gate set holds at least one wiring, and every tuple group is the first of its shapes
        assert 0 < len(got["tuple"]) <= len(got["shape"]) <= len(full)
        assert set(got["tuple"]["key"].tolist()) <= set(got["shape"]["key"].tolist())


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_grouped_under_the_function_filters(engine, case):
    width = case[0]
    _, orders = _load(engine, case)
    full = _all(engine, width, orders)
    for name, (o, m, i) in _filters(full, width, case[4]).items():
        engine.set_function_filter(o, m, i)
        feasible = _run(engine, width, orders, 0).feasible
        _each_grouping(engine, width, orders, full[_allowed(full, o, m, i)], feasible, case[4])


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_grouped_under_the_depth_filter(engine, case):
    width, n = case[0], case[1]
    _, orders = _load(engine, case)
    full = _all(engine, width, orders)
    depth = _random_depth(n, case[4] + 50)
    dep = E.record_depths(full, depth)
    med = int(np.median(dep))
    for bound in sorted({sb.SBG_DEPTH_BINS - 1, med}):
        engine.set_depth_filter(depth, bound)
        feasible = _run(engine, width, orders, 0).feasible
        got = _each_grouping(engine, width, orders, full[dep <= bound], feasible, bound)
        for g, want in got.items():
            engine.set_grouping(g)
            _run(engine, width, orders, 0)
            # one count per group, at the depth of its record
            assert np.array_equal(engine.depth_counts(), _hist(E.record_depths(want, depth)))
            engine.set_grouping(None)
    # with the function filter too
    outer = sorted(sb.AFFINE_FUNCTIONS | set(range(100)))
    engine.set_depth_filter(depth, med)
    engine.set_function_filter(outer, None, None)
    ok = _allowed(full, outer, None, None)
    feasible = _run(engine, width, orders, 0).feasible
    _each_grouping(engine, width, orders, full[ok & (dep <= med)], feasible, 3)


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_grouped_keys_match_oracle(engine, case):
    width, n = case[0], case[1]
    (tabs, tgt, mask, inb), orders = _load(engine, case)
    if width == 3:
        total, keys = E.enum3_range(tabs, tgt, mask, orders[0], n * (n - 1) * (n - 2) // 6)
    elif width == 5:
        total, keys, _ = E.oracle_enum5(tabs, tgt, mask, inb, orders[0], FULL_CAP)
    else:
        tuples = E.unpack_list(engine.filter7_part(0, 1)[:3])
        engine.set_list7(engine.filter7_part(0, 1)[:3])
        total, keys = E.oracle_enum7(tabs, tgt, mask, tuples, *orders, FULL_CAP)
    assert len(keys) == total > 0
    for g in GROUPINGS:
        ids = [sb.match_group(int(k), width, g) for k in keys]
        want = [int(k) for j, k in enumerate(keys) if j == 0 or ids[j] != ids[j - 1]]
        engine.set_grouping(g)
        e = _run(engine, width, orders, 0)
        assert [int(k) for k in engine.fetch_matches(0, e.total)["key"]] == want


@pytest.mark.parametrize("grouping", GROUPINGS)
@pytest.mark.parametrize("nparts", [2, 3, 7])
@pytest.mark.parametrize("case", [CASES[1], CASES[3], CASES[6]], ids=lambda c: "w%d" % c[0])
def test_shares_add_up(engine, case, nparts, grouping):
    width = case[0]
    engs = [sb.LutEngine(0) for _ in range(nparts)]
    try:
        _, orders = _load(engine, case)
        engine.set_grouping(grouping)
        whole_e = _run(engine, width, orders, 0)
        whole = engine.fetch_matches(0, whole_e.total)
        totals = []
        for q, e in enumerate(engs):
            _load(e, case)
            e.set_grouping(grouping)
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


# -- closed forms: under the empty mask every candidate matches -----------------------------------

def _check_closed(engine, total, record, rs, picks=500):
    for first in (0, total // 2 - 300, total - 600):
        got = engine.fetch_matches(first, 600)
        assert len(got) == min(600, total - first)
        for j in sorted({0, len(got) - 1} | {int(x) for x in rs.randint(0, len(got), 20)}):
            assert F.as_tuple(got[j]) == record(first + j), (first, j)
    ranks = np.random.default_rng(int(rs.randint(1 << 30))).choice(total, picks, replace=False)
    for r, rec in zip(ranks, engine.pick_matches(ranks)):
        assert F.as_tuple(rec) == record(int(r)), int(r)


def test_5lut_empty_mask_closed_form(engine):
    n = 40
    tabs = S.synthetic_state(n, seed=5100 + n)
    tgt = S.sbox_target(S.rijndael_sbox(), 6)
    mask = np.zeros(4, dtype=np.uint64)
    order = E.orders(n)[0]
    engine.load(tabs, tgt, mask, [])
    rows5 = S.order5_rows()
    combos = F.total5(n, []) // F.W5
    assert combos == 658_008
    for g, per, want in (("tuple", F.W5, combos), ("shape", 256, 10 * combos)):
        engine.set_grouping(g)
        e = engine.enumerate5(order, 10)
        assert (e.total, e.feasible) == (want, combos)
        _check_closed(engine, e.total,
                      lambda r: F.record5(r * per, tabs, tgt, mask, [], order, rows5),
                      np.random.RandomState(len(g)))


def test_7lut_n40_empty_mask_closed_form(engine):
    n = 40
    tabs = S.synthetic_state(n, seed=5200)
    tgt = S.sbox_target(S.rijndael_sbox(), 4)
    mask = np.zeros(4, dtype=np.uint64)
    _, outer, middle = E.orders(77)
    engine.load(tabs, tgt, mask, [])
    rows7 = S.order7_rows()
    for g, per, want in (("tuple", F.W7, 100_000), ("shape", 65536, 7_000_000)):
        engine.set_grouping(g)
        e = engine.enumerate7(outer, middle, 10)
        assert (e.total, e.feasible) == (want, 100_000)
        _check_closed(engine, e.total,
                      lambda r: F.record7(r * per, tabs, tgt, mask, outer, middle, rows7, 100_000),
                      np.random.RandomState(len(g) + 7))


def test_long_7lut_list(engine):
    """bench.py's n = 40 32-position state: its 251,784 7-LUT matches, grouped on the host."""
    tabs, tgt, mask, inb, outer, middle = _n40_state()
    engine.load(tabs, tgt, mask, inb)
    orders = (outer, middle)
    unf = _run(engine, 7, orders, 0)
    full = engine.fetch_matches(0, unf.total)
    assert len(full) == 251_784
    assert R.check_realises(full, tabs, tgt, mask) == len(full)
    for g in GROUPINGS:
        want = _grouped(full, 7, g)
        assert len(want) == len(np.unique(_group_ids(full["key"], 7, g)))
        engine.set_grouping(g)
        _check(engine, 7, orders, want, unf.feasible, k=1000, seed=7)


@pytest.mark.parametrize("case", [c for c in CASES if c[0] != 3], ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_first_group_is_the_search_match(engine, case):
    width = case[0]
    _, orders = _load(engine, case)
    for g in GROUPINGS:
        engine.set_grouping(g)
        first = _run(engine, width, orders, 1, count=False)
        if not len(first.matches):
            continue
        key = int(first.matches["key"][0])
        if width == 5:
            assert engine.search5(orders[0]).key == key
        elif 0 in case[3]:
            assert engine.search7(*orders).key == key


def test_searches_ignore_the_grouping(engine):
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
    for g in GROUPINGS:
        engine.set_grouping(g)
        assert results() == want


def test_lifetime_and_errors(engine):
    _, (order,) = _load(engine, CASES[3])
    e = engine.enumerate5(order, 0)
    engine.set_grouping("tuple")
    with pytest.raises(RuntimeError):
        engine.fetch_matches(0, 1)       # set_grouping ended the cursor
    out = np.zeros(1, dtype=sb.MATCH_DTYPE)
    n_out = C.c_uint64()
    assert engine.lib.sbg_enum_fetch(engine._h, 0, 1, out.ctypes.data_as(C.c_void_p),
                                     C.byref(n_out)) == ERR_STATE
    r = np.zeros(1, dtype=np.uint64)
    assert engine.lib.sbg_enum_pick(engine._h, r.ctypes.data_as(native.u64p), 1,
                                    out.ctypes.data_as(C.c_void_p)) == ERR_STATE
    t = engine.enumerate5(order, 0)
    assert 0 < t.total <= e.total
    # fetch and pick keep the cursor
    a = engine.fetch_matches(0, 5)
    engine.pick_matches([0, t.total - 1])
    assert engine.fetch_matches(0, 5).tobytes() == a.tobytes()
    # without a depth filter there is no histogram, grouped or not
    hist = np.zeros(4, dtype=np.uint64)
    assert engine.lib.sbg_enum_depth_counts(engine._h, hist.ctypes.data_as(native.u64p), 4) \
        == ERR_STATE
    # a bad value: SBG_ERR_ARG, the setting kept (and the cursor ended all the same)
    for bad in (3, -1, 1 << 20):
        assert engine.lib.sbg_enum_set_grouping(engine._h, bad) == ERR_ARG
    with pytest.raises(RuntimeError):
        engine.fetch_matches(0, 1)
    assert engine.enumerate5(order, 0).total == t.total
    with pytest.raises(ValueError):
        engine.set_grouping("wiring")
    assert engine.lib.sbg_enum_set_grouping(None, 1) == ERR_ARG
    assert engine.lib.sbg_enum_set_grouping(engine._h, native.SBG_GROUP_NONE) == 0
    assert engine.enumerate5(order, 0).total == e.total


# -- DistributedLutSearch over gloo ----------------------------------------------------------------

DIST_CASES = [CASES[3], CASES[6]]   # widths 5 and 7


def _dist_run(drv_or_engine, engine, case, grouping, dist_api):
    """One grouped enumeration, page and pick of `case` over the whole phase-1 list."""
    width, n, ms, inb, seed = case
    engine.load(*_state(n, ms, inb, seed, width))
    order, outer, middle = E.orders(seed)
    orders = (order,) if width == 5 else (outer, middle)
    drv_or_engine.set_grouping(grouping)
    if dist_api:
        e = drv_or_engine.enumerate5(orders[0], 7) if width == 5 else \
            drv_or_engine.enumerate7(*orders, 7)
    else:
        e = _run(engine, width, orders, 7)
    t = e.total
    page = drv_or_engine.fetch_matches(t // 3, 40)
    pick = drv_or_engine.pick_matches(np.random.RandomState(case[4]).randint(0, t, 60))
    return (e.total, e.matches.tobytes(), page.tobytes(), pick.tobytes())


def _dist_worker(rank, world, port, q):
    import torch.distributed as dist
    from sboxgates_b200.distributed import DistributedLutSearch
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    eng = sb.LutEngine(0)
    try:
        drv = DistributedLutSearch(eng)
        out = [_dist_run(drv, eng, case, g, True) for case in DIST_CASES for g in GROUPINGS]
        q.put((rank, out))
    finally:
        eng.close()
        dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


@pytest.mark.parametrize("world", [2, 3])
def test_distributed_grouping_gloo(engine, world):
    import torch.multiprocessing as mp
    want = [_dist_run(engine, engine, case, g, False) for case in DIST_CASES for g in GROUPINGS]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dist_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = [q.get(timeout=600) for _ in range(world)]
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    for rank, out in got:
        assert out == want, rank
