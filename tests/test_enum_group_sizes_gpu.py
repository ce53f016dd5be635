"""GPU: group sizes (sbg_enum_group_sizes).  The size of the group at a rank must be the number of
matches the ungrouped enumeration, under the same filters, counts with that group's id: checked
against a full ungrouped fetch counted on the host, on every kernel form (the depth tests' CASES:
widths 3, 5, 7 at NW = 1, 2, 4, 8), under the function and depth filters, against the CPU oracle's
keys, against the closed forms of the empty mask at n = 40, on bench.py's n = 40 state, across
shares and over gloo.  The call must keep the cursor and change nothing a later call reads."""
import ctypes as C
import os
import socket
from collections import Counter

import numpy as np
import pytest

import _enum_reference as R
import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native
from test_enum_depth_gpu import CASES, FULL_CAP, _all, _load, _random_depth, _run, _state
from test_enum_functions_gpu import _allowed, _filters
from test_oracle_large_gpu import _n40_state

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = -1, -4
GROUPINGS = ("shape", "tuple")


@pytest.fixture(autouse=True)
def _reset(engine):
    """The session's engine leaves every test of this module ungrouped and unfiltered."""
    yield
    engine.set_grouping(None)
    engine.clear_function_filter()
    engine.clear_depth_filter()


def _sizes_of(recs, width, grouping):
    """The host reference: each group's size, groups in ascending id (= rank) order."""
    c = Counter(R.group_ids(recs["key"], width, grouping).tolist())
    return np.array([c[i] for i in sorted(c)], dtype=np.uint64)


def _check_sizes(engine, width, orders, recs, seed):
    """Both groupings (and none) against the host sizes of `recs`, the ungrouped set under the
    installed filters: all ranks, and 300 shuffled ranks with repeats."""
    for g in (None,) + GROUPINGS:
        want = _sizes_of(recs, width, g)
        if g is None or width == 3:
            assert np.all(want == 1)
        engine.set_grouping(g)
        e = _run(engine, width, orders, 0)
        assert e.total == len(want)
        if e.total == 0:
            assert len(recs) == 0
            continue
        got = engine.group_sizes(np.arange(e.total))
        assert got.dtype == np.uint64
        assert np.array_equal(got, want), (g, int(np.argmax(got != want)))
        assert int(got.sum()) == len(recs)
        ranks = np.random.RandomState(seed).randint(0, e.total, 300)
        assert np.array_equal(engine.group_sizes(ranks), want[ranks])
    engine.set_grouping(None)


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_sizes_equal_host_counts(engine, case):
    width = case[0]
    _, orders = _load(engine, case)
    full = _all(engine, width, orders)
    assert len(full) > 0
    _check_sizes(engine, width, orders, full, case[4])


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_sizes_under_the_function_filters(engine, case):
    """Every filter of _filters, including a restricted inner set (the 7-LUT visit loop)."""
    width = case[0]
    _, orders = _load(engine, case)
    full = _all(engine, width, orders)
    for name, (o, m, i) in _filters(full, width, case[4]).items():
        engine.set_function_filter(o, m, i)
        _check_sizes(engine, width, orders, full[_allowed(full, o, m, i)], case[4])


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_sizes_under_the_depth_filter(engine, case):
    width, n = case[0], case[1]
    _, orders = _load(engine, case)
    full = _all(engine, width, orders)
    depth = _random_depth(n, case[4] + 50)
    dep = E.record_depths(full, depth)
    med = int(np.median(dep))
    for bound in sorted({sb.SBG_DEPTH_BINS - 1, med}):
        engine.set_depth_filter(depth, bound)
        _check_sizes(engine, width, orders, full[dep <= bound], bound)
    # with the function filter too: an outer set, and a restricted inner set
    for o, i in ((sorted(sb.AFFINE_FUNCTIONS | set(range(100))), None),
                 (None, sorted(range(0, 256, 3)))):
        engine.set_depth_filter(depth, med)
        engine.set_function_filter(o, None, i)
        _check_sizes(engine, width, orders, full[_allowed(full, o, None, i) & (dep <= med)], 3)
        engine.clear_function_filter()


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_sizes_match_oracle(engine, case):
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
        c = Counter(sb.match_group(int(k), width, g) for k in keys)
        engine.set_grouping(g)
        e = _run(engine, width, orders, 0)
        groups = engine.fetch_matches(0, e.total)
        assert [sb.match_group(int(k), width, g) for k in groups["key"]] == sorted(c)
        assert engine.group_sizes(np.arange(e.total)).tolist() == [c[i] for i in sorted(c)]


# -- closed forms: under the empty mask every candidate matches -----------------------------------

def _check_closed(engine, total, size, rs, picks=300):
    ranks = np.concatenate([[0, total - 1], rs.randint(0, total, picks)])
    assert np.all(engine.group_sizes(ranks) == size)


def test_5lut_empty_mask_closed_form(engine):
    n = 40
    tabs = S.synthetic_state(n, seed=5100 + n)
    tgt = S.sbox_target(S.rijndael_sbox(), 6)
    engine.load(tabs, tgt, np.zeros(4, dtype=np.uint64), [])
    order = E.orders(n)[0]
    combos = 658_008
    for g, size, groups in (("tuple", 2_560, combos), ("shape", 256, 10 * combos)):
        engine.set_grouping(g)
        e = engine.enumerate5(order, 0)
        assert e.total == groups
        _check_closed(engine, e.total, size, np.random.RandomState(len(g)))
    # one call over the whole tuple range adds up to the ungrouped total
    engine.set_grouping("tuple")
    e = engine.enumerate5(order, 0)
    assert int(engine.group_sizes(np.arange(e.total)).sum()) == 1_684_500_480 == 2_560 * combos


def test_7lut_n40_empty_mask_closed_form(engine):
    n = 40
    tabs = S.synthetic_state(n, seed=5200)
    tgt = S.sbox_target(S.rijndael_sbox(), 4)
    engine.load(tabs, tgt, np.zeros(4, dtype=np.uint64), [])
    _, outer, middle = E.orders(77)
    for g, size, groups in (("tuple", 4_587_520, 100_000), ("shape", 65_536, 7_000_000)):
        engine.set_grouping(g)
        e = engine.enumerate7(outer, middle, 0)
        assert e.total == groups
        _check_closed(engine, e.total, size, np.random.RandomState(len(g) + 7))


def test_long_7lut_list(engine):
    """bench.py's n = 40 32-position state: 3,954 tuple and 7,506 shape sizes over its 251,784
    matches."""
    tabs, tgt, mask, inb, outer, middle = _n40_state()
    engine.load(tabs, tgt, mask, inb)
    orders = (outer, middle)
    unf = _run(engine, 7, orders, 0)
    full = engine.fetch_matches(0, unf.total)
    assert len(full) == 251_784
    for g, groups in (("tuple", 3_954), ("shape", 7_506)):
        want = _sizes_of(full, 7, g)
        assert len(want) == groups
        engine.set_grouping(g)
        e = _run(engine, 7, orders, 0)
        assert e.total == groups
        assert np.array_equal(engine.group_sizes(np.arange(groups)), want)
        ranks = np.random.RandomState(9).permutation(groups)[:1000]
        assert np.array_equal(engine.group_sizes(ranks), want[ranks])


# -- shares -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("grouping", (None,) + GROUPINGS)
@pytest.mark.parametrize("nparts", [2, 3, 7])
@pytest.mark.parametrize("case", [CASES[1], CASES[3], CASES[6]], ids=lambda c: "w%d" % c[0])
def test_shares_add_up(engine, case, nparts, grouping):
    width = case[0]
    engs = [sb.LutEngine(0) for _ in range(nparts)]
    try:
        _, orders = _load(engine, case)
        engine.set_grouping(grouping)
        t = _run(engine, width, orders, 0).total
        ranks = np.concatenate([np.arange(t), np.random.RandomState(2).randint(0, t, 200)])
        whole = engine.group_sizes(ranks)
        for q, e in enumerate(engs):
            _load(e, case)
            e.set_grouping(grouping)
            fn = {3: e.enumerate3, 5: e.enumerate5, 7: e.enumerate7}[width]
            fn(*orders, 0, True, q, nparts)
        counts = [e.enum_block_count() for e in engs]
        sums = np.zeros((nparts, max(max(counts), 1)), dtype=np.uint64)
        for q, e in enumerate(engs):
            sums[q, :counts[q]] = e.enum_block_sums()
        assert {e.enum_set_global(sums, counts) for e in engs} == {t}
        shares = [e.group_sizes(ranks) for e in engs]
        # each rank is owned by exactly one share; the others write 0
        assert np.all(sum((s != 0).astype(int) for s in shares) == 1)
        assert np.array_equal(sum(shares), whole)
        # a share's nonzero slots are its own: its pick writes records exactly there
        for e, s in zip(engs, shares):
            assert np.array_equal(e.pick_matches(ranks)["width"] != 0, s != 0)
    finally:
        for e in engs:
            e.close()


# -- lifetime and errors ----------------------------------------------------------------------------

def _sizes_rc(engine, ranks, out):
    r = np.ascontiguousarray(ranks, dtype=np.uint64)
    return engine.lib.sbg_enum_group_sizes(engine._h, r.ctypes.data_as(native.u64p), len(r),
                                           out.ctypes.data_as(native.u64p))


def test_lifetime_and_errors(engine):
    (tabs, tgt, mask, inb), (order,) = _load(engine, CASES[3])
    n = tabs.shape[0]
    out = np.full(4, 77, dtype=np.uint64)
    engine.set_grouping("tuple")            # no cursor
    assert _sizes_rc(engine, [0], out) == ERR_STATE
    assert np.all(out == 77)
    engine.set_depth_filter(_random_depth(n, 5), sb.SBG_DEPTH_BINS - 1)
    e = engine.enumerate5(order, 0)
    assert e.total > 2
    hist = engine.depth_counts()
    a = engine.fetch_matches(0, e.total)
    ranks = np.random.RandomState(4).randint(0, e.total, 50)
    b = engine.pick_matches(ranks)
    s = engine.group_sizes(ranks)
    # a rank at or past the total: SBG_ERR_ARG, nothing written
    assert _sizes_rc(engine, [0, e.total], out) == ERR_ARG
    assert _sizes_rc(engine, [2**64 - 1], out) == ERR_ARG
    assert np.all(out == 77)
    # null pointers with nranks > 0; nranks == 0 is fine
    assert engine.lib.sbg_enum_group_sizes(engine._h, None, 1, out.ctypes.data_as(native.u64p)) \
        == ERR_ARG
    r = np.zeros(1, dtype=np.uint64)
    assert engine.lib.sbg_enum_group_sizes(engine._h, r.ctypes.data_as(native.u64p), 1, None) \
        == ERR_ARG
    assert engine.lib.sbg_enum_group_sizes(engine._h, None, 0, None) == 0
    assert engine.lib.sbg_enum_group_sizes(None, None, 0, None) == ERR_ARG
    assert np.all(out == 77)
    assert engine.group_sizes([]).shape == (0,)
    # the call keeps the cursor and changes nothing fetch, pick or the histogram read
    assert engine.fetch_matches(0, e.total).tobytes() == a.tobytes()
    assert engine.pick_matches(ranks).tobytes() == b.tobytes()
    assert np.array_equal(engine.depth_counts(), hist)
    assert np.array_equal(engine.group_sizes(ranks), s)
    # set_grouping ends the cursor
    engine.set_grouping("shape")
    assert _sizes_rc(engine, [0], out) == ERR_STATE
    with pytest.raises(RuntimeError):
        engine.group_sizes([0])
    # the Python checks
    engine.enumerate5(order, 0)
    for bad in ([-1], [[0]], [0.5]):
        with pytest.raises(ValueError):
            engine.group_sizes(bad)


def test_7lut_cursor_kept(engine):
    """A 7-LUT sizes pass under a restricted inner set (the visit loop) keeps the cursor, and a
    recount over the installed list finds the same groups."""
    _, orders = _load(engine, CASES[6])
    engine.set_function_filter(None, None, sorted(range(0, 256, 3)))
    engine.set_grouping("tuple")
    e = _run(engine, 7, orders, 0)
    assert e.total > 0
    a = engine.fetch_matches(0, e.total)
    s = engine.group_sizes(np.arange(e.total))
    assert engine.fetch_matches(0, e.total).tobytes() == a.tobytes()
    assert np.array_equal(engine.group_sizes(np.arange(e.total)[::-1]), s[::-1])
    assert _run(engine, 7, orders, 0).total == e.total
    assert engine.fetch_matches(0, e.total).tobytes() == a.tobytes()


def test_searches_unchanged_by_sizes(engine):
    (tabs, tgt, mask, inb), (order,) = _load(engine, CASES[3])
    _, outer, middle = E.orders(CASES[3][4])
    go = [int(x) for x in np.random.RandomState(3).permutation(tabs.shape[0])]

    def res(r):
        return (r.found, r.key, r.ordering, list(r.gates), r.func_outer, r.func_middle,
                r.func_inner, r.inner_seen)

    def results(interleave):
        out = []
        for step in range(4):
            engine.load(tabs, tgt, mask, inb)
            if interleave:
                engine.set_grouping(GROUPINGS[step % 2])
                t = engine.enumerate5(order, 0).total
                engine.group_sizes(np.arange(min(t, 500)))
                engine.set_grouping(None)
            if step == 0:
                out.append(res(engine.search5(order)))
            elif step == 1:
                out.append(res(engine.search7(outer, middle)))
            elif step == 2:
                x = engine.search_node(0, order, outer, middle, go)
                out.append((x.found_stage, x.key3, list(x.gates3), res(x.r5), res(x.r7)))
            else:
                batch = engine.search_batch([{"order5": order, "gate_order": go},
                                             {"outer": outer, "middle": middle, "order5": order}])
                out.append([(x.found_stage, x.key3, list(x.gates3), res(x.r5), res(x.r7))
                            for x in batch])
        return out

    assert results(True) == results(False)


# -- DistributedLutSearch over gloo ----------------------------------------------------------------

DIST_CASES = [CASES[3], CASES[6]]   # widths 5 and 7


def _dist_run(drv_or_engine, engine, case, grouping, dist_api):
    """One grouped enumeration of `case` over the whole phase-1 list, and the sizes of 80 ranks."""
    width, n, ms, inb, seed = case
    engine.load(*_state(n, ms, inb, seed, width))
    order, outer, middle = E.orders(seed)
    orders = (order,) if width == 5 else (outer, middle)
    drv_or_engine.set_grouping(grouping)
    if dist_api:
        e = drv_or_engine.enumerate5(orders[0], 0) if width == 5 else \
            drv_or_engine.enumerate7(*orders, 0)
    else:
        e = _run(engine, width, orders, 0)
    ranks = np.random.RandomState(case[4]).randint(0, e.total, 80)
    return (e.total, drv_or_engine.group_sizes(ranks).tolist())


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
def test_distributed_group_sizes_gloo(engine, world):
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
