"""GPU: the searches' work counters (sbg_result::tuples_swept, tuples_feasible) against exact sweep
sizes, on every search path.

tuples_swept is the combinations this device put through the feasibility test, inbits rejections
included.  bench.py's headline counts it, so it is pinned to closed forms (checked against the
oracle in test_work_counters_cpu.py), not to the library's own other paths:
  - 7-LUT, list below the cap: C(n,7) whole; the parts' sweeps add up to C(n,7);
  - 7-LUT, capped list: the reference's count (last entry's rank + 1) <= swept <= C(n,7), and the
    parts add up to at most C(n,7);
  - 5-LUT miss: C(n,5) whole and exactly the part's Deal5 share; hit: index + 1 <= swept <= C(n,5).
Every phase-1 and search_5lut kernel form is forced through the environment (read at sbg_create),
over tiny states (n = 7, 8, 9), the window and head states of the list tests, full-mask states up to
n = 160 (C(n,7) far past 2^32) and a dense capped state, each with no inbits, gate 0 excluded and 3
or 4 input bits excluded.  Then every entry point: search_node after SCAN3 and SEARCH5, batches
(two waves, repeated slots, an overflowed lane), the sharded steps with finish5 / finish7, the
in-process all-gather (sbg_allgather_merge7) on one device, and DistributedLutSearch over gloo.

On a list that reaches SBG_LIST_CAP only the bounds hold: warps finish the tickets they were handed
before the stop, so the device's sweep may pass the reference's count, and bench.py's T-units count
the device's work there, not the reference's."""
import ctypes as C
import os
from functools import lru_cache
from math import comb

import numpy as np
import pytest

import _counter_support as W
import _enum_support as E
import _support as S
import sboxgates_b200 as sb
import test_filter_sieve_gpu as FS
import test_filter_windows_gpu as FW
from sboxgates_b200 import native
from sboxgates_b200.native import SBG_LIST_CAP
from test_handle_calls_gpu import device_list

pytestmark = pytest.mark.gpu

NONE = E.NONE
FULL = np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)
INBITS = ([], [0], [1, 3, 5], [0, 2, 4, 6])
FORMS = {
    "default": {},
    "pm4": {"SBG_PM_PREFIX": "4"}, "pm5": {"SBG_PM_PREFIX": "5"},
    "head0": {"SBG_HEAD": "0"}, "head1": {"SBG_HEAD": "1"}, "head2": {"SBG_HEAD": "2"},
    "shift0": {"SBG_SHIFT": "0"}, "shift1": {"SBG_SHIFT": "1"},
    "sieve0": {"SBG_SIEVE": "0"}, "sieve2": {"SBG_SIEVE": "2"},
    "packed0": {"SBG_PACKED": "0"},
    "table": {"SBG_TICKET_TABLE": "4096"},
    "hits1": {"SBG_HITS_CAP": "1"},
    "two": {"SBG_SEARCH5": "two"}, "fused": {"SBG_SEARCH5": "fused"},
    "two_hits1": {"SBG_SEARCH5": "two", "SBG_HITS_CAP": "1"},
}
SEARCH5_FORMS = ("default", "two", "fused", "two_hits1", "head0")


def _fresh(env):
    mp = pytest.MonkeyPatch()
    try:
        for k, v in env.items():
            mp.setenv(k, v)
        return sb.LutEngine(0)   # the knobs are read when the handle is created
    finally:
        mp.undo()


@pytest.fixture(scope="module")
def engines():
    out = {name: _fresh(env) for name, env in FORMS.items()}
    yield out
    for e in out.values():
        e.close()


ORDER5, OUTER, MIDDLE = E.orders(9300)


# ------------------------------------------------------------------------------------------------
# states: (name, tables, target, mask, inbits)

def _tiny():
    sbox = S.rijndael_sbox()
    out = []
    for n in (7, 8, 9):
        tabs = S.synthetic_state(n, seed=9400 + n, num_inputs=min(8, n))
        for i, inb in enumerate(INBITS):
            inb = [b for b in inb if b < n]
            # a target every 7-tuple can realise under a one-position mask: the list is everything
            # the inbits allow, so at n = 7 with gate 0 excluded the one tuple is rejected
            mask = S.mux_mask([(0, 1), (1, 0), (2, 1), (3, 0), (4, 1), (5, 0), (6, 1), (7, 0)])
            out.append(("tiny%d_%d" % (n, i), tabs, S.sbox_target(sbox, i), mask, inb))
            out.append(("tinyfull%d_%d" % (n, i), tabs, S.sbox_target(sbox, i), FULL, inb))
    return out


def _windows():
    return [("win%d" % i, tabs, tgt, mask, inb)
            for i, (n, tabs, tgt, mask, inb, _) in enumerate(FW._states())] + \
        [("head%d" % n, tabs, tgt, mask, inb) for n, tabs, tgt, mask, inb, _ in FS._head_states()]


FULL_NS = (64, 96, 128, 129, 160)


def _full():
    sbox = S.rijndael_sbox()
    return [("full%d_%d" % (n, i), S.synthetic_state(n, seed=9500 + n), S.sbox_target(sbox, n % 8),
             FULL, inb) for n in FULL_NS for i, inb in enumerate(INBITS)]


def _dense():
    """n = 48 under a depth-3 mux mask: the list reaches the cap (test_gpu_parity's overflow case)."""
    return [("dense48", S.synthetic_state(48, seed=48), S.sbox_target(S.rijndael_sbox(), 0),
             S.mux_mask([(0, 1), (5, 0), (3, 1)]), [0, 5, 3])]


STATES = {s[0]: s for s in _tiny() + _windows() + _full() + _dense()}
# the states every forced form runs (the default form runs all of them)
FORM_STATES = ["tiny7_1", "tiny9_3", "win4", "win20", "win27", "head48", "full96_1", "full129_3",
               "dense48"]


def load(eng, name):
    _, tabs, tgt, mask, inb = STATES[name]
    eng.load(tabs, tgt, mask, inb)
    return len(tabs), inb


def bounds7(n, lst):
    """(least, most) tuples_swept of a phase 1 that produced `lst` (packed, ascending)."""
    count = len(lst)
    lo = W.reference_sweep7(n, int(lst[-1]) if count else 0, count)
    return lo, comb(n, 7)


def check_sweep7(swept, n, lst, what):
    lo, hi = bounds7(n, lst)
    if len(lst) < SBG_LIST_CAP:
        assert swept == hi, (what, swept, hi)
    else:
        assert lo <= swept <= hi, (what, lo, swept, hi)


def part_sweep7(eng, p, P):
    """filter7_part(p, P) and the sweep finish7 reports for it (the part's list installed by
    set_list7, which carries the part's sweep over)."""
    lst = eng.filter7_part(p, P)
    eng.set_list7(lst)
    return lst, eng.finish7(NONE, OUTER, MIDDLE).tuples_swept


def run7(eng, name, parts=(2, 3, 7)):
    n, _ = load(eng, name)
    r = eng.search7(OUTER, MIDDLE)
    lst = eng.filter7_part(0, 1)
    assert r.tuples_feasible == len(lst), (name, r.tuples_feasible, len(lst))
    check_sweep7(r.tuples_swept, n, lst, (name, "search7"))
    key = eng.decomp7_part(0, 1, OUTER, MIDDLE)
    f = eng.finish7(key, OUTER, MIDDLE)
    assert (f.key, f.tuples_feasible) == (r.key, len(lst)), name
    check_sweep7(f.tuples_swept, n, lst, (name, "filter7_part + finish7"))
    for P in parts:
        sweeps, merged = [], []
        for p in range(P):
            lp, sw = part_sweep7(eng, p, P)
            sweeps.append(sw)
            merged.append(lp)
        total = sum(sweeps)
        if len(lst) < SBG_LIST_CAP:
            assert total == comb(n, 7), (name, P, sweeps)
            assert np.array_equal(np.sort(np.concatenate(merged)), lst), (name, P)
        else:
            assert total <= comb(n, 7), (name, P, sweeps)
    return n, lst


def test_sweep7_every_state_default_form(engines):
    eng = engines["default"]
    capped = big = 0
    for name in STATES:
        n, lst = run7(eng, name, parts=(2, 3, 7) if n_of(name) <= 96 else (3,))
        capped += len(lst) == SBG_LIST_CAP
        big += comb(n, 7) >= 2**32
    assert capped >= 2 and big >= 8


def n_of(name):
    return len(STATES[name][1])


def test_sweep7_tiny_states_against_the_oracle(engines):
    """n = 7, 8, 9: the list length and the oracle's feasible count agree, a part count above the
    number of tickets leaves parts empty and the sum intact, and the fully rejected tuple (n = 7,
    gate 0 excluded) is still swept."""
    eng = engines["default"]
    for name, tabs, tgt, mask, inb in _tiny():
        n = len(tabs)
        want, st = S.oracle_filter7(tabs, tgt, mask, inb)
        eng.load(tabs, tgt, mask, inb)
        r = eng.search7(OUTER, MIDDLE)
        assert r.tuples_feasible == len(want) == st.tuples_feasible, name
        assert r.tuples_swept == st.tuples_filtered == comb(n, 7), name
        sweeps = [part_sweep7(eng, p, 64)[1] for p in range(64)]
        assert sum(sweeps) == comb(n, 7) and sweeps.count(0) > 0, (name, sweeps)
    eng.load(*STATES["tiny7_1"][1:])
    r = eng.search7(OUTER, MIDDLE)
    assert (r.tuples_feasible, r.tuples_swept) == (0, 1)


@pytest.mark.parametrize("form", [f for f in FORMS if f != "default"])
def test_sweep7_forced_forms(engines, form):
    eng = engines[form]
    for name in FORM_STATES:
        run7(eng, name, parts=(3,))


# ------------------------------------------------------------------------------------------------
# search_5lut

@lru_cache(maxsize=None)
def _deal_sizes(n, inb, head):
    deal = E.Deal5(n, list(inb), head)
    sizes = [sum(hi - lo for lo, hi in deal.block_ranges(j)) for j in range(deal.blocks())]
    return deal, sizes, W.head_skipped5(deal, list(inb))


def share5(n, inb, head, p, P):
    deal, sizes, skipped = _deal_sizes(n, tuple(inb), head)
    return sum(sizes[j] for j in deal.part_blocks(p, P, skip_excluded=False)) + \
        (skipped if p == 0 else 0)


def run5(eng, form, name, parts=(2, 3, 7)):
    n, inb = load(eng, name)
    r = eng.search5(ORDER5)
    if r.found:
        assert r.index + 1 <= r.tuples_swept <= comb(n, 5), (form, name, r.index, r.tuples_swept)
        return r
    assert r.tuples_swept == comb(n, 5), (form, name, r.tuples_swept)
    two_first = form in ("two", "two_hits1") or (form != "fused" and comb(n, 5) <= 4_000_000)
    head = not two_first and form != "head0" and n >= 128
    for P in parts:
        feas = 0
        for p in range(P):
            key = eng.search5_part(p, P, ORDER5)
            f = eng.finish5(key, ORDER5)
            assert key == NONE and not f.found, (form, name, P, p)
            assert f.tuples_swept == share5(n, inb, head, p, P), (form, name, P, p, f.tuples_swept)
            feas += f.tuples_feasible
        assert feas == r.tuples_feasible, (form, name, P, feas, r.tuples_feasible)
    return r


S5_STATES = ["tiny7_0", "tiny9_2", "win0", "win8", "win14", "win21", "full64_0", "full64_3",
             "full128_1", "full129_2", "full160_0", "full160_3", "dense48"]


@pytest.mark.parametrize("form", SEARCH5_FORMS)
def test_sweep5_every_form(engines, form):
    misses = 0
    for name in S5_STATES:
        r = run5(engines[form], form, name, parts=(2, 3, 7) if n_of(name) <= 64 else (3,))
        misses += not r.found
        n = n_of(name)
        if not r.found and n <= 20:
            _, tabs, tgt, mask, inb = STATES[name]
            found, _, st = S.oracle_search(5, tabs, tgt, mask, inb, S.OrcRng.from_seed(n))
            assert not found and st.tuples_feasible == r.tuples_feasible, (form, name)
    assert misses >= 8


def test_sweep5_hits_are_bounded(engines):
    """Planted 5-LUT targets: the sweep stops after the hit but covers at least its rank."""
    eng = engines["default"]
    rs = np.random.RandomState(9600)
    for n in (9, 40, 130):
        tabs = S.synthetic_state(n, seed=9600 + n)
        for inb in INBITS:
            allowed = [g for g in range(n) if g not in inb]
            gates = sorted(int(x) for x in rs.choice(allowed, 5, replace=False))
            eng.load(tabs, E.planted5(tabs, gates, int(rs.randint(10)), 0x96, 0xCA), FULL, inb)
            r = eng.search5(ORDER5)
            assert r.found and r.index + 1 <= r.tuples_swept <= comb(n, 5), (n, inb, r.index)


# ------------------------------------------------------------------------------------------------
# entry points

def test_search_node_stage7_after_scan3_and_search5(engines):
    eng = engines["default"]
    for name in ("win4", "full96_1", "dense48"):
        n, _ = load(eng, name)
        node = eng.search_node(0, order5=ORDER5, outer=OUTER, middle=MIDDLE,
                               gate_order=list(range(n)))
        if node.found_stage != 0:
            continue
        lst = eng.filter7_part(0, 1)
        assert node.r5.tuples_swept == comb(n, 5), name
        check_sweep7(node.r7.tuples_swept, n, lst, (name, "node"))
        assert node.r7.tuples_feasible == len(lst)


def test_search_batch_lanes(engines):
    """Two waves (10 jobs), slots repeated on several lanes, and on the hits1 handle the dense
    state's chain overflowing on lanes other than 0 (its redo runs phase 1 step by step): every
    lane reports its own sweep."""
    for form in ("default", "hits1"):
        eng = engines[form]
        names = ["win4", "dense48", "win20", "full96_1", "win4", "dense48", "tiny9_3", "win27",
                 "dense48", "win20"]
        slots = {nm: i for i, nm in enumerate(dict.fromkeys(names))}
        for nm, slot in slots.items():
            _, tabs, tgt, mask, inb = STATES[nm]
            eng.stage(slot, tabs, tgt, mask, inb)
        jobs = [dict(slot=slots[nm], outer=OUTER, middle=MIDDLE) for nm in names]
        res = eng.search_batch(jobs)
        lists = {}
        for nm in slots:
            eng.use(slots[nm])
            lists[nm] = eng.filter7_part(0, 1)
        for nm, r in zip(names, res):
            check_sweep7(r.r7.tuples_swept, n_of(nm), lists[nm], (form, nm, "batch"))
            assert r.r7.tuples_feasible == len(lists[nm]), (form, nm)


def test_finish7_after_batch_reports_the_batch_sweep():
    """Sequence: load, search_batch([slot 0, SEARCH7]), decomp7_part(0, 1), finish7 on a fresh
    handle.  finish7 reports the batch's phase-1 sweep (it reported 0: nothing had set the handle's
    sweep)."""
    eng = sb.LutEngine(0)
    try:
        for name in ("win4", "full129_3"):
            n, _ = load(eng, name)
            r = eng.search_batch([dict(slot=0, outer=OUTER, middle=MIDDLE)])[0]
            key = eng.decomp7_part(0, 1, OUTER, MIDDLE)
            f = eng.finish7(key, OUTER, MIDDLE)
            assert f.key == r.r7.key and f.tuples_swept == r.r7.tuples_swept == comb(n, 7), \
                (name, f.tuples_swept, r.r7.tuples_swept)
    finally:
        eng.close()


def test_finish7_after_search5_part_reports_phase1():
    """Sequence: filter7_part(0, 1), search5_part, decomp7_part, finish7.  finish7 reports the
    phase-1 sweep C(n,7) (it reported search_5lut's C(n,5))."""
    eng = sb.LutEngine(0)
    try:
        for name in ("win4", "full96_0"):
            n, _ = load(eng, name)
            lst = eng.filter7_part(0, 1)
            eng.search5_part(0, 1, ORDER5)
            key = eng.decomp7_part(0, 1, OUTER, MIDDLE)
            f = eng.finish7(key, OUTER, MIDDLE)
            assert f.tuples_feasible == len(lst) < SBG_LIST_CAP
            assert f.tuples_swept == comb(n, 7), (name, f.tuples_swept)
    finally:
        eng.close()


@pytest.mark.parametrize("between", ["filter7_part", "search7", "node7", "node3", "enumerate7"])
def test_finish5_reports_its_own_search5_part(between):
    """Sequence: search5_part, then a call that runs phase 1 or a node, then finish5.  finish5
    reports search5_part's sweep and feasible count (it reported the 7-LUT sweep, or 0 after a node
    without stage 7)."""
    eng = sb.LutEngine(0)
    try:
        n, _ = load(eng, "win4")
        key = eng.search5_part(0, 1, ORDER5)
        want = eng.finish5(key, ORDER5)
        assert not want.found and want.tuples_swept == comb(n, 5)
        if between == "filter7_part":
            eng.filter7_part(0, 1)
        elif between == "search7":
            eng.search7(OUTER, MIDDLE)
        elif between == "node7":
            eng.search_node(0, outer=OUTER, middle=MIDDLE)
        elif between == "node3":
            eng.search_node(0, gate_order=list(range(n)))
        else:
            eng.enumerate7(OUTER, MIDDLE, 1)
        got = eng.finish5(key, ORDER5)
        assert (got.tuples_swept, got.tuples_feasible) == (comb(n, 5), want.tuples_feasible), \
            (between, got.tuples_swept)
    finally:
        eng.close()


def test_set_list7_device_carries_the_part_sweep(engines):
    """filter7_part(p, P), list7_device, set_list7_device of the part lists: finish7 reports the
    part's sweep; set_list7 of a list of another problem's staging reports 0."""
    import torch
    eng = engines["default"]
    n, _ = load(eng, "win4")
    sweeps, lists = [], []
    for p in range(3):
        lp, sw = part_sweep7(eng, p, 3)
        sweeps.append(sw)
        lists.append(lp)
    whole = eng.filter7_part(0, 1)
    assert len(whole) < SBG_LIST_CAP
    assert np.array_equal(np.sort(np.concatenate(lists)), whole)
    assert sum(sweeps) == comb(n, 7), sweeps
    for p in range(3):
        cnt = eng.filter7_part_device(p, 3)
        ptr, c2 = eng.list7_device()
        assert c2 == cnt
        buf = torch.zeros(max(cnt, 1), dtype=torch.int64, device="cuda")
        if cnt:
            buf[:cnt] = torch.from_numpy(device_list(ptr, cnt).view(np.int64)).cuda()
        torch.cuda.synchronize()
        eng.set_list7_device(buf.data_ptr(), max(cnt, 1), [cnt])
        assert eng.finish7(NONE, OUTER, MIDDLE).tuples_swept == sweeps[p], p
    eng.stage(0, *STATES["win4"][1:])   # an identical restage keeps the list and its sweep
    assert eng.finish7(NONE, OUTER, MIDDLE).tuples_swept == sweeps[2]
    load(eng, "win20")   # another problem: no list of it, so a list installed now has no sweep
    eng.set_list7(lists[0])
    assert eng.finish7(NONE, OUTER, MIDDLE).tuples_swept == 0


# ------------------------------------------------------------------------------------------------
# sbg_allgather_merge7 with every handle on the one device

@pytest.mark.parametrize("nh", [1, 2, 3, 8])
def test_allgather_merge7_on_one_device(nh):
    lib = native.load_library()
    engs = [sb.LutEngine(0) for _ in range(nh)]
    try:
        empty = 0
        for name in ("win4", "tiny8_0", "tiny7_1", "dense48", "full129_3"):
            n, _ = load(engs[0], name)
            ref = engs[0]
            whole = ref.filter7_part(0, 1)
            rkey = ref.decomp7_part(0, 1, OUTER, MIDDLE)
            want = ref.finish7(rkey, OUTER, MIDDLE)
            parts = []
            for i, e in enumerate(engs):
                load(e, name)
                parts.append(e.filter7_part(i, nh))
            # an enumeration cursor on every handle, which the merge must end
            for e in engs:
                e.enumerate3(list(range(n)), 0)
            hs = (C.c_void_p * nh)(*[e._h.value for e in engs])
            total = C.c_int()
            assert lib.sbg_allgather_merge7(hs, nh, C.byref(total)) == 0, \
                lib.sbg_last_error(engs[0]._h)
            assert total.value == len(whole), (name, nh, total.value, len(whole))
            keys, sweeps = [], []
            for i, e in enumerate(engs):
                with pytest.raises(RuntimeError):
                    e.fetch_matches(0, 1)
                ptr, cnt = e.list7_device()
                assert np.array_equal(device_list(ptr, cnt), whole), (name, nh, i)
                keys.append(e.decomp7_part(i, nh, OUTER, MIDDLE))
            for i, e in enumerate(engs):
                res = e.finish7(min(keys), OUTER, MIDDLE)
                assert E.result7_fields(res) == E.result7_fields(want), (name, nh, i)
                assert res.tuples_feasible == len(whole)
                sweeps.append(res.tuples_swept)
            if len(whole) < SBG_LIST_CAP:
                assert sum(sweeps) == comb(n, 7), (name, nh, sweeps)
            empty += min(len(p) for p in parts) == 0
        assert empty >= 1   # a part with an empty list (tiny7_1's list is empty)
    finally:
        for e in engs:
            e.close()


# ------------------------------------------------------------------------------------------------
# DistributedLutSearch over gloo, world 2 and 3 on the one GPU

DIST_STATES = ("win8", "full129_3")


def _counter_worker(rank, world, port, backend, q):
    import torch.distributed as dist
    from sboxgates_b200.distributed import DistributedLutSearch
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group(backend, rank=rank, world_size=world)
    eng = sb.LutEngine(0)
    try:
        drv = DistributedLutSearch(eng, shard_min_tuples5=0, shard_min_tuples7=0, shard_min_list=0)
        out = []
        for name in DIST_STATES:
            load(eng, name)
            r5 = drv.search5_sharded(ORDER5)
            r7 = drv.search7_sharded(OUTER, MIDDLE)
            out.append((int(r5.found), int(r5.tuples_swept), int(r7.key), int(r7.tuples_feasible),
                        int(r7.tuples_swept)))
        q.put((rank, out))
    finally:
        eng.close()
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_counts_add_up_over_gloo(engine, world):
    from test_enum_global_gpu import _spawn
    got = dict(_spawn(world, "gloo", _counter_worker))
    for i, name in enumerate(DIST_STATES):
        n, _ = load(engine, name)
        r5 = engine.search5(ORDER5)
        r7 = engine.search7(OUTER, MIDDLE)
        rows = [got[r][i] for r in range(world)]
        assert not r5.found and all(row[0] == 0 for row in rows), name
        assert sum(row[1] for row in rows) == r5.tuples_swept == comb(n, 5), (name, rows)
        assert all(row[2:4] == (int(r7.key), int(r7.tuples_feasible)) for row in rows), name
        assert r7.tuples_feasible < SBG_LIST_CAP
        assert sum(row[4] for row in rows) == r7.tuples_swept == comb(n, 7), (name, rows)
