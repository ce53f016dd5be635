"""GPU: the depth filter at its edges.  Each test compares the filtered enumeration with the
unfiltered matches of depth <= bound (the unfiltered set is pinned to the CPU oracle elsewhere, and
tests/_enum_support.record_depths filters it on the host): total, first K, histogram, pages and picks,
byte for byte.

  1. the pruning edges: a 5-tuple with exactly two gates at depth B - 1 is kept and one with three
     is dropped, a 7-tuple likewise with one and two, a 3-LUT pair with a gate at B - 1 is kept;
     `feasible` of the 5-LUT enumeration against a brute force over C(n, 5);
  2. the deepest histogram bins (1,021 and 1,022), the clamp of the bound, and a cut histogram copy;
  3. count-free windows whose first two hold no ticket the filter keeps;
  4. bench.py's n = 40 7-LUT list (71,023 entries) under the depths of its own circuit;
  5. a real circuit's depths: the des_s1 golden graph, shallowest_matches against a brute force;
  6. DistributedLutSearch at world 2 and 3 over gloo against one engine."""
import glob
import math
import os

import numpy as np
import pytest

import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import graph, native
from test_enum3_gpu import _pair_ticket, _window3
from test_enum_depth_gpu import CASES, FULL_CAP, _hist, _load, _mask, _nw, _run, _state
from test_enum_global_gpu import _free_port
from test_oracle_large_gpu import _count_free_windows, _n40_state, _prefix_ticket, _seams

pytestmark = pytest.mark.gpu

B_EDGE = 2          # the bound of the pruning-edge states; their gates have depths B - 2 .. B
DEEP = (1016, 1020)  # gate depths of the deepest-bin states


@pytest.fixture(autouse=True)
def _clear_filter(engine):
    """The session's engine leaves every test of this module without a filter."""
    yield
    engine.clear_depth_filter()


def _full(engine, width, orders):
    """Every unfiltered match, in key order."""
    engine.clear_depth_filter()
    e = _run(engine, width, orders, 0)
    assert 0 < e.total <= FULL_CAP
    return engine.fetch_matches(0, e.total)


def _compare(engine, width, orders, full, depth, bound, k=100, pages=(), seed=0):
    """The filtered enumeration at `bound` against full[record_depths(full) <= bound]: total, the
    first k, depth_counts, pages (at 0, the middle, the end and `pages`) and seeded picks.
    Returns (the counted enumeration, the reference matches)."""
    dep = E.record_depths(full, depth)
    want = full[dep <= bound]
    engine.set_depth_filter(depth, bound)
    e = _run(engine, width, orders, k)
    assert e.total == len(want), (width, bound, e.total, len(want))
    assert e.matches.tobytes() == want[:k].tobytes(), (width, bound)
    assert np.array_equal(engine.depth_counts(), _hist(dep[dep <= bound])), (width, bound)
    t = e.total
    for first in sorted({0, t // 2, max(t - 5, 0), t} | {int(p) for p in pages}):
        assert engine.fetch_matches(first, 64).tobytes() == want[first:first + 64].tobytes(), \
            (width, bound, first)
    if t:
        ranks = np.random.RandomState(seed + bound % 997).randint(0, t, 200)
        assert engine.pick_matches(ranks).tobytes() == want[ranks].tobytes(), (width, bound)
    return e, want


# -- 1. pruning edges -----------------------------------------------------------------------------

def _edge_depth(gates, n, width, seed):
    """Gate depths in {B - 2, B - 1, B} (B = B_EDGE) such that the first match (gates in record
    order) has depth exactly B with the most gates at B - 1 a kept match may have -- two inner
    gates (width 5), the last gate (width 7), a gate of the position pair (width 3) -- and a second
    match is dropped by the B - 1 rule alone (three or two gates at B - 1, none at B; width 3: a
    gate at B)."""
    B = B_EDGE
    depth = np.random.RandomState(seed).randint(B - 2, B + 1, n)
    g0 = [int(x) for x in gates[0]]
    low = {3: g0[1:], 5: g0[:3], 7: g0[:6]}[width]
    depth[g0] = B - 1
    depth[low] = B - 2
    need, value = {3: (1, B), 5: (3, B - 1), 7: (2, B - 1)}[width]
    for g in gates[1:]:
        free = sorted(set(int(x) for x in g) - set(g0 if width == 3 else low))
        if len(free) >= need:
            depth[free] = value
            break
    return depth.astype(np.uint16)


EDGE_CASES = [c for c in CASES if _nw(_mask(c[2], c[4])) in (1, 8)]


def test_edge_cases_cover_nw_1_and_8():
    assert {(c[0], _nw(_mask(c[2], c[4]))) for c in EDGE_CASES} == \
        {(w, nw) for w in (3, 5, 7) for nw in (1, 8)}


@pytest.mark.parametrize("case", EDGE_CASES, ids=lambda c: "w%d-n%d-m%s" % c[:3])
def test_pruning_edges(engine, case):
    width, n = case[:2]
    B = B_EDGE
    (tabs, tgt, mask, inb), orders = _load(engine, case)
    full = _full(engine, width, orders)
    gates = full["gates"][:, :width].astype(np.int64)
    depth = _edge_depth(gates, n, width, case[4])
    d = depth[gates].astype(np.int64)
    at = np.sum(d == B - 1, axis=1)
    dep = E.record_depths(full, depth)
    # the states reach both sides of the edge
    if width == 3:
        assert np.sum((d[:, :2] == B - 1).any(axis=1) & (dep <= B)) > 0
        assert np.sum((d == B).any(axis=1)) > 0
    else:
        most = {5: 2, 7: 1}[width]
        assert np.sum((at == most) & (dep <= B)) > 0, case
        assert np.sum((at > most) & (d.max(axis=1) < B)) > 0, case
    for bound in range(0, B + 3):
        e, _ = _compare(engine, width, orders, full, depth, bound, seed=case[4])
        if width == 5:
            assert e.feasible == E.feasible5_under_bound(tabs, tgt, mask, inb, depth, bound), bound
    if width == 5:
        assert E.feasible5_under_bound(tabs, tgt, mask, inb, depth, B) > 0


# -- 2. deepest bins and the clamp ----------------------------------------------------------------

DEEP_CASES = [CASES[10], CASES[11], CASES[13]]   # widths 3, 5, 7; NW 4, 8, 1


@pytest.mark.parametrize("case", DEEP_CASES, ids=lambda c: "w%d" % c[0])
def test_deepest_bins_and_clamp(engine, case):
    width, n = case[:2]
    _, orders = _load(engine, case)
    full = _full(engine, width, orders)
    depth = np.random.RandomState(case[4] + 1).randint(DEEP[0], DEEP[1] + 1, n).astype(np.uint16)
    assert int(depth.max()) == native.SBG_MAX_DEPTH
    dep = E.record_depths(full, depth)
    ref = np.zeros(sb.SBG_DEPTH_BINS, dtype=np.uint64)
    ref[:int(dep.max()) + 1] = _hist(dep)
    # the deepest bins the width allows are filled: 1,021 (width 3), 1,021 and 1,022 (5 and 7)
    assert ref[1021] > 0 and (width == 3 or ref[1022] > 0), ref[1016:]
    results = []
    for bound in (1020, 1021, 1022, sb.SBG_DEPTH_BINS - 1, 2**32 - 1):
        e, want = _compare(engine, width, orders, full, depth, bound, seed=case[4])
        results.append((e.total, e.matches.tobytes(), engine.depth_counts().tobytes()))
    assert results[-1] == results[-2]
    assert results[-1][0] == len(full) > results[0][0]
    # a histogram copy cut at 1,021 bins: those bins, and nothing written past them
    sentinel = np.uint64(0xA5A5A5A5A5A5A5A5)
    out = np.full(sb.SBG_DEPTH_BINS, sentinel, dtype=np.uint64)
    assert engine.lib.sbg_enum_depth_counts(engine._h, out.ctypes.data_as(native.u64p), 1021) == 0
    assert np.array_equal(out[:1021], ref[:1021])
    assert np.all(out[1021:] == sentinel)


# -- 3. count-free windows under a filter ---------------------------------------------------------

def _window_check(engine, width, orders, want, ticket_of, skipped, seams):
    """The first K count-free matches equal the first K counted and the reference, for K = 1, K
    ending just past the first window seam beyond `skipped`, and every match; the first kept
    match lies past the second window."""
    t = len(want)
    tickets = np.array([ticket_of(int(k)) for k in want["key"]], dtype=np.int64)
    assert tickets[0] >= skipped, (tickets[0], skipped)
    later = [s for s in seams if s > tickets[0]]
    ks = {1, t}
    if later:
        ks.add(min(t, int(np.sum(tickets < later[0])) + 1))
    for k in sorted(ks):
        free = _run(engine, width, orders, k, count=False)
        counted = _run(engine, width, orders, k)
        assert counted.total == t
        assert free.matches.tobytes() == want[:k].tobytes(), k
        assert counted.matches.tobytes() == want[:k].tobytes(), k
        assert tickets[k - 1] >= skipped
    return len(ks)


def _deep_first(n, width, windows, order=None):
    """How many of the first gates (width 3: of the gate order) must be deep so that the first two
    count-free windows (windows[0] + windows[1] tickets) hold no kept ticket."""
    for r in range(1, n):
        if width == 3:
            covered = sum(n - 1 - i for i in range(r))
        else:
            covered = math.comb(n - 2, 3) - math.comb(n - 2 - r, 3)
        if covered >= windows[0] + windows[1]:
            return r
    raise AssertionError("the state is too small for two windows")


def test_count_free_windows_width3(engine):
    w = _window3()
    n, B = 200, 5
    rs = np.random.RandomState(23000)
    tabs = S.synthetic_state(n, seed=23001)
    mask = _mask("r16", 23002)
    tgt = S.sbox_target(S.rijndael_sbox(), 3)
    order = rs.permutation(n).astype(np.uint16)
    engine.load(tabs, tgt, mask, [])
    full = _full(engine, 3, (order,))
    r = _deep_first(n, 3, (w, 2 * w))
    depth = rs.randint(0, B + 1, n)
    depth[order[:r]] = rs.randint(B, B + 3, r)
    depth = depth.astype(np.uint16)
    _, want = _compare(engine, 3, (order,), full, depth, B)
    seams = _seams(w, n * (n - 1) // 2)
    assert len(seams) >= 3
    _window_check(engine, 3, (order,), want, lambda k: _pair_ticket(n, k), seams[1], seams)


def test_count_free_windows_width5(engine):
    w5, _ = _count_free_windows()
    n, B = 64, 6
    rs = np.random.RandomState(24000)
    tabs = S.synthetic_state(n, seed=24001)
    mask = _mask("r24", 24002)
    tgt = S.sbox_target(S.rijndael_sbox(), 1)
    order = E.orders(24003)[0]
    engine.load(tabs, tgt, mask, [])
    full = _full(engine, 5, (order,))
    r = _deep_first(n, 5, (w5, 2 * w5))
    depth = rs.randint(0, B - 1, n)
    depth[:r] = B
    depth = depth.astype(np.uint16)
    _, want = _compare(engine, 5, (order,), full, depth, B)
    seams = _seams(w5, math.comb(n - 2, 3))
    assert len(seams) >= 3
    _window_check(engine, 5, (order,), want, lambda k: _prefix_ticket(n, k), seams[1], seams)


# -- 4. the long 7-LUT list -----------------------------------------------------------------------

def _synthetic_circuit(n, seed, num_inputs=8):
    """S.synthetic_state's tables rebuilt with the same draws, and the depth of every gate."""
    rs = np.random.RandomState(seed)
    tabs = [S.input_table(i) for i in range(num_inputs)]
    depth = [0] * num_inputs
    while len(tabs) < n:
        i, j, k = rs.choice(len(tabs), 3, replace=False)
        f = int(rs.randint(1, 255))
        tabs.append(S.lut_table(f, tabs[i], tabs[j], tabs[k]))
        depth.append(1 + max(depth[i], depth[j], depth[k]))
    return np.stack(tabs[:n]).astype(np.uint64), np.array(depth[:n], dtype=np.uint16)


def _n40_seed():
    """The synthetic_state seed of _n40_state, from the same draws."""
    rs = np.random.RandomState(1)
    for i in range(4):
        bits = rs.choice(8, i, replace=False)
        for _ in bits:
            rs.randint(0, 2)
        for _ in range(3):
            rs.permutation(256)
        seed = int(rs.randint(1 << 30))
    return seed


def test_long_7lut_list(engine):
    _, w7 = _count_free_windows()
    tabs, tgt, mask, inb, outer, middle = _n40_state()
    circuit, depth = _synthetic_circuit(40, _n40_seed())
    assert np.array_equal(circuit, tabs)
    engine.load(tabs, tgt, mask, inb)
    lst = E.unpack_list(engine.filter7_part(0, 1))
    orders = (outer, middle)
    full = _full(engine, 7, orders)
    assert (len(lst), len(full)) == (71_023, 251_784)
    dep = E.record_depths(full, depth)
    seams = _seams(w7, len(lst))
    levels = np.unique(dep)
    assert len(levels) >= 4, levels
    bounds = [int(levels[0]), int(levels[1]), int(levels[-2])]
    for bound in bounds:
        want = full[dep <= bound]
        idx = (want["key"] >> np.uint64(23)).astype(np.int64)
        pages = [max(0, int(np.searchsorted(idx, s)) - 3) for s in seams]
        e, _ = _compare(engine, 7, orders, full, depth, bound, k=500, pages=pages, seed=bound)
        assert e.total > 0
        r, m = sb.sample_matches(engine, e, min(e.total, 300), seed=bound)
        assert m.tobytes() == want[r.astype(np.int64)].tobytes()
    # count-free: every entry holding gate 1 (the first gate of the first entries) is dropped
    first_out = int(np.argmax(lst[:, 0] != 1))
    assert first_out >= seams[1], (first_out, seams[:3])
    deep = depth.copy()
    bound = int(dep.max())
    deep[1] = bound
    _, want = _compare(engine, 7, orders, full, deep, bound)
    _window_check(engine, 7, orders, want, lambda k: k >> 23, seams[1], seams)


# -- 5. a real circuit's depths -------------------------------------------------------------------

def _graph_state():
    path = glob.glob(os.path.join(S.GOLDEN, "graphs", "des_s1_*.xml"))[0]
    g = graph.load_graph(path)
    words = [[(gt.table >> (64 * w)) & (2**64 - 1) for w in range(4)] for gt in g.gates]
    tabs = np.array(words, dtype=np.uint64)
    mask = np.array([2**64 - 1, 0, 0, 0], dtype=np.uint64)   # the 64 inputs of a 6-bit S-box
    return tabs, graph.gate_depths(g), mask


# (width, planted gates, LUT functions).  Gate 7 of the graph is 3 XOR 6, so an outer XOR of 3 and 6
# is also one of 7 and a third gate: each target has realisations at two depths at least.
GRAPH_TARGETS = [(3, (3, 6, 12), (0x96,)), (5, (1, 12, 19, 9, 22), (0xCA, 0x6B)),
                 (7, (3, 6, 1, 0, 2, 4, 5), (0x96, 0xE8, 0x72))]


LIST_GRAPH = 100   # list entries of the width-7 target (the first ones hold every input gate)


@pytest.mark.parametrize("target", GRAPH_TARGETS, ids=lambda t: "w%d" % t[0])
def test_shallowest_on_a_real_circuit(engine, target):
    width, gates, funcs = target
    tabs, depth, mask = _graph_state()
    n = tabs.shape[0]
    assert n == 26
    g = [tabs[x] for x in gates]
    if width == 3:
        tgt = S.lut_table(funcs[0], *g)
    else:
        outer = S.lut_table(funcs[0], g[0], g[1], g[2])
        mid = g[3] if width == 5 else S.lut_table(funcs[1], g[3], g[4], g[5])
        tgt = S.lut_table(funcs[-1], outer, mid, g[-1])
    engine.load(tabs, tgt, mask, [])
    go = np.random.RandomState(26).permutation(n).astype(np.uint16)
    order, outer_o, middle_o = E.orders(26)
    if width == 7:
        engine.set_list7(engine.filter7_part(0, 1)[:LIST_GRAPH])
    orders = {3: (go,), 5: (order,), 7: (outer_o, middle_o)}[width]
    full = _full(engine, width, orders)
    dep = E.record_depths(full, depth)
    assert len(np.unique(dep)) >= 2, np.unique(dep)
    dmin = int(dep.min())
    want = full[dep == dmin]
    got_min, count, recs = sb.shallowest_matches(engine, width, orders, depth, 50)
    assert (got_min, count) == (dmin, len(want))
    assert recs.tobytes() == want[:50].tobytes()
    assert engine.fetch_matches(0, count).tobytes() == want.tobytes()


# -- 6. across ranks ------------------------------------------------------------------------------

DIST_CASES = [CASES[1], CASES[3], CASES[5]]   # widths 3, 5, 7 (7: phase 1's whole list)


def _dist_case(drv, eng, case, check=None):
    """One width's filtered calls on drv (a LutEngine or a DistributedLutSearch over eng): the
    histogram at the loosest bound, the enumeration, histogram, a page and a pick at a middle
    bound, and shallowest_matches; plus the collectives each depth_counts call added.  The later
    calls depend on the histograms, so where check(i, out[i]) says that the ranks do not all
    hold the expected one, the run stops there (on every rank, so that no collective is left
    waiting)."""
    width, n, ms, inb, seed = case
    tabs, tgt, mask, inb = _state(n, ms, inb, seed, width)
    eng.load(tabs, tgt, mask, inb)
    order, outer, middle = E.orders(seed)
    go = np.random.RandomState(seed).permutation(n).astype(np.uint16)
    orders = {3: (go,), 5: (order,), 7: (outer, middle)}[width]
    run = getattr(drv, "enumerate%d" % width)
    depth = np.random.RandomState(seed + 9).randint(0, 7, n)
    out, added = [], []

    def counts():
        c0 = getattr(drv, "collectives", 0)
        h = drv.depth_counts()
        added.append(getattr(drv, "collectives", 0) - c0)
        return h.tobytes()
    drv.set_depth_filter(depth, sb.SBG_DEPTH_BINS - 1)
    e = run(*orders, 10)
    out += [e.total, e.matches.tobytes(), counts()]
    if check is not None and not check(2, out[2]):
        return out, added
    hist = np.frombuffer(out[-1], dtype=np.uint64)
    nz = np.flatnonzero(hist)
    drv.set_depth_filter(depth, int(nz[len(nz) // 2]))
    e = run(*orders, 25)
    t = e.total
    out += [t, e.matches.tobytes(), counts()]
    if check is not None and not check(5, out[5]):
        return out, added
    out += [drv.fetch_matches(t // 3, 40).tobytes(),
            drv.pick_matches(np.random.RandomState(seed).randint(0, t, 50)).tobytes()]
    dmin, count, recs = sb.shallowest_matches(drv, width, orders, depth, 30)
    out += [dmin, count, recs.tobytes()]
    return out, added


def _dist_worker(rank, world, port, q, want):
    import torch
    import torch.distributed as dist
    from sboxgates_b200.distributed import DistributedLutSearch
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    eng = sb.LutEngine(0)

    def agree(ok):
        """Whether every rank's value equals one engine's (an all-reduce of our own, not the
        driver's)."""
        t = torch.tensor([0 if ok else 1], dtype=torch.int64)
        dist.all_reduce(t)
        return int(t.item()) == 0
    try:
        drv = DistributedLutSearch(eng)
        out = [_dist_case(drv, eng, case, lambda i, v, w=w: agree(v == w[i]))
               for case, w in zip(DIST_CASES, want)]
        q.put((rank, out))
    except BaseException as exc:
        q.put((rank, repr(exc)))
        raise
    finally:
        eng.close()
        dist.destroy_process_group()


def _spawn(world, want):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dist_worker, args=(r, world, port, q, want))
             for r in range(world)]
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
    assert all(isinstance(g[1], list) for g in got), got
    assert all(p.exitcode == 0 for p in procs)
    return got


@pytest.mark.parametrize("world", [2, 3])
def test_distributed_depth_filter_gloo(engine, world):
    want = [_dist_case(engine, engine, case)[0] for case in DIST_CASES]
    for w, case in zip(want, DIST_CASES):
        assert w[0] > 0 and w[3] > 0 and w[8] > 0, case
    for rank, out in _spawn(world, want):
        assert isinstance(out, list), (rank, out)
        for case, wnt, (got, added) in zip(DIST_CASES, want, out):
            assert got == wnt, (rank, case)
            # each depth_counts call adds exactly one all-reduce
            assert added == [1, 1], (rank, case, added)
