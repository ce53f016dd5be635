"""GPU: the state one sbg_handle keeps between calls, against single calls on a fresh handle and the
CPU oracle.

A graph build, bench.py and DistributedLutSearch keep one handle alive and interleave staged
slots, node calls, batches of up to SBG_LANES concurrent chains, the sharded phase-1 / phase-2
steps and enumerations on it.  Every expected value here comes from a reference handle `ref` that
loads the state in question and makes the single call; where n <= 24 the deterministic cases also
check it against the CPU oracle.

  a. The installed 7-LUT list belongs to one staged state of one slot: after a batch whose lane 0
     searched another slot, after restaging the current slot, after a second wave, a list consumer
     (enumerate7, decomp7_part + finish7, list7_device) must see the current problem's list or none.
     An identical restage keeps the list; search_node moves the current slot and its list along;
     a search_5lut or 5-LUT enumeration between the install and phase 2 leaves the list whole.
  b. Batches that put one slot on several lanes of a wave, after a lazy load, after an eager
     stage and with nothing pending, at sizes that take the bulk copy and the shifted-window sieve.
  c. Seeded call sequences over a pool of states (tests/_handle_support.py), each step checked
     against `ref` and a model of the handle state."""
import numpy as np
import pytest

import _enum_support as E
import _handle_support as H
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200.distributed import _DeviceArray
from sboxgates_b200.native import SBG_LIST_CAP

pytestmark = pytest.mark.gpu

NONE = E.NONE
SCAN3, SEARCH5, SEARCH7 = H.SCAN3, H.SEARCH5, H.SEARCH7
FULL = np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)
FUNCS = [0x96, 0xE8, 0xCA, 0xD8, 0x1B, 0x6A, 0xB4, 0x78, 0x3C, 0xA6]


def state_error(code):
    return pytest.raises(RuntimeError, match=r"\(code %d\)" % code)


@pytest.fixture(scope="module")
def ref():
    eng = sb.LutEngine(0)
    yield eng
    eng.close()


@pytest.fixture
def eng():
    e = sb.LutEngine(0)
    yield e
    e.close()


def device_list(ptr, cnt):
    """A copy of `cnt` packed list entries at device address ptr, as uint64."""
    import torch
    torch.cuda.synchronize()
    if cnt == 0:
        return np.zeros(0, dtype=np.uint64)
    return torch.as_tensor(_DeviceArray(ptr, cnt), device="cuda").cpu().numpy().view(np.uint64)


def result_fields(res, width, skip=()):
    """The fields of an SbgResult of search_`width`lut.  The work counters are left out where they
    depend on when a stop landed among the concurrently running warps: search_5lut's feasible and
    swept counts once it matched, search_7lut's phase-1 sweep once the list reached its cap."""
    if width == 5 and res.found:
        skip = tuple(skip) + ("tuples_feasible", "tuples_swept")
    if width == 7 and res.tuples_feasible >= SBG_LIST_CAP:
        skip = tuple(skip) + ("tuples_swept",)
    out = {}
    for name, _ in res._fields_:
        if name not in skip:
            v = getattr(res, name)
            out[name] = list(v) if hasattr(v, "__len__") else v
    return out


def node_fields(r):
    """Every field of an SbgNodeResult, r5 and r7 flattened (work counters as result_fields)."""
    out = {"found_stage": r.found_stage, "gates3": list(r.gates3), "func3": r.func3,
           "seen3": r.seen3, "key3": r.key3}
    for part, width in (("r5", 5), ("r7", 7)):
        for k, v in result_fields(getattr(r, part), width).items():
            out[part + "." + k] = v
    return out


def assert_same(got, want, what):
    diff = {k: (got[k], want[k]) for k in want if got.get(k) != want[k]}
    assert not diff, (what, diff)


def enum_fields(e):
    return {"total": e.total, "feasible": e.feasible, "matches": e.matches.tobytes()}


# ------------------------------------------------------------------------------------------------
# a. the installed list

def _planted(n, seed, mask, row, last):
    """A state of n gates whose target a 7-gate circuit on gates 0-5 and `last` realises on
    ordering row `row`: its list entry sits among the first few, so the oracle's first key is
    cheap."""
    rs = np.random.RandomState(seed)
    tabs = S.synthetic_state(n, seed=seed)
    gates = [0, 1, 2, 3, 4, 5, last]
    tgt = E.planted7(tabs, gates, row, *rs.choice(FUNCS, 3))
    return tabs, tgt, mask


# A: 24 gates, 64 positions (a long list, gates up to 23); B: 14 gates, 128 positions.
STATE_A = _planted(24, 8101, S.mux_mask([(6, 0), (2, 1)]), 5, 9)
STATE_B = _planted(14, 8102, S.mux_mask([(7, 1)]), 11, 8)
ORDERS = E.orders(8103)   # (order5, outer, middle)


def load(e, st, slot=None):
    if slot is None:
        e.load(st[0], st[1], st[2], [])
    else:
        e.stage(slot, st[0], st[1], st[2], [])


def oracle_b():
    """B's phase-1 list (all of C(14, 7)), its first 7-LUT key under ORDERS and that key's result."""
    tabs, tgt, mask = STATE_B
    lst = E.filter7_range(tabs, tgt, mask, [], 0, 3432)
    _, outer, middle = ORDERS
    key = E.decomp7_key(tabs, tgt, mask, lst, outer, middle)
    assert key != NONE
    return lst, key, E.expected_result7(key, lst, tabs, tgt, mask, outer, middle)


def check_consumer(e, ref, consumer, what):
    """The list consumer on `e`, whose current problem is B with no list of B installed: the same
    as on a handle that has just loaded B, and as the oracle says."""
    _, outer, middle = ORDERS
    lst, key, want = oracle_b()
    load(ref, STATE_B)
    if consumer == "enumerate7":
        got = e.enumerate7(outer, middle, 16)
        exp = ref.enumerate7(outer, middle, 16)
        assert_same(enum_fields(got), enum_fields(exp), what)
        # the oracle's list, and the first match's record rebuilt from it
        assert got.feasible == len(lst) and len(got.matches) > 0, what
        rec = got.matches[0]
        k = int(rec["key"])
        assert k <= key, what
        assert E.record_fields(rec) == tuple(E.expected_record(
            7, k, STATE_B[0], STATE_B[1], STATE_B[2], outer, middle, tuple7=lst[k >> 23])), what
    elif consumer == "decomp7_part":
        # phase 2 needs a list of the current problem: there is none
        with state_error(-4):
            e.decomp7_part(0, 1, outer, middle)
        with state_error(-4):
            e.finish7(key, outer, middle)
        # ... and after B's phase 1 the key and result are B's
        assert np.array_equal(e.filter7_part(0, 1), ref.filter7_part(0, 1)), what
        k = e.decomp7_part(0, 1, outer, middle)
        assert k == ref.decomp7_part(0, 1, outer, middle) == key, what
        res = e.finish7(k, outer, middle)
        assert_same(result_fields(res, 7), result_fields(ref.finish7(k, outer, middle), 7), what)
        assert_same(E.result7_fields(res), want, what)
    else:
        ptr, cnt = e.list7_device()
        assert cnt == ref.list7_device()[1] == 0, (what, cnt)
        e.filter7_part(0, 1)
        ptr, cnt = e.list7_device()
        assert np.array_equal(E.unpack_list(device_list(ptr, cnt)), lst), what


CONSUMERS = ["enumerate7", "decomp7_part", "list7_device"]


@pytest.mark.parametrize("consumer", CONSUMERS)
@pytest.mark.parametrize("form", ["batch", "two_waves", "restage"])
def test_list_consumer_sees_the_current_problem(eng, ref, form, consumer):
    """Lane 0's list of state A, then a list consumer with B current: B's answers, never A's.
    batch: a batch on slot 1 (A) while slot 2 (B) is current; two_waves: the same as job 0 of the
    second wave of a 10-job batch; restage: load(A), search7, stage(0, B)."""
    order5, outer, middle = ORDERS
    if form == "restage":
        load(eng, STATE_A)
        load(ref, STATE_A)
        assert_same(result_fields(eng.search7(outer, middle), 7),
                    result_fields(ref.search7(outer, middle), 7), (form, "search7"))
        load(eng, STATE_B, slot=0)
    else:
        load(eng, STATE_A, slot=1)
        load(eng, STATE_B, slot=2)
        eng.use(2)
        jobs = [dict(slot=1, outer=outer, middle=middle)]
        if form == "two_waves":
            jobs = [dict(slot=2, order5=order5)] * 8 + jobs + [dict(slot=2, order5=order5)]
        res = eng.search_batch(jobs)
        load(ref, STATE_A)
        want = ref.search_node(0, outer=outer, middle=middle)
        assert_same(node_fields(res[len(jobs) - 1 if form == "batch" else 8]), node_fields(want),
                    (form, "batch result"))
    check_consumer(eng, ref, consumer, (form, consumer))


def test_identical_restage_keeps_the_list(eng):
    """Restaging the state a slot already holds ships nothing and keeps its list: enumerate7
    afterwards runs no phase 1 (the same launches as right after search7) and gives the same."""
    _, outer, middle = ORDERS
    load(eng, STATE_B)
    eng.search7(outer, middle)
    l0 = eng.launches
    first = eng.enumerate7(outer, middle, 16)
    reuse = eng.launches - l0
    skipped = eng.transfer_stats()[4]
    load(eng, STATE_B, slot=0)
    assert eng.transfer_stats()[4] == skipped + 1
    l0 = eng.launches
    again = eng.enumerate7(outer, middle, 16)
    assert eng.launches - l0 == reuse
    assert_same(enum_fields(again), enum_fields(first), "identical restage")
    k = eng.decomp7_part(0, 1, outer, middle)
    assert k == oracle_b()[1]


def test_search_node_moves_the_current_slot_and_its_list(eng, ref):
    """search_node(slot = A) makes A current and installs A's list, so enumerate7 and
    decomp7_part afterwards legitimately reuse it: A's answers, no phase 1."""
    order5, outer, middle = ORDERS
    load(eng, STATE_B)
    eng.search7(outer, middle)
    l0 = eng.launches
    eng.enumerate7(outer, middle, 16)
    reuse = eng.launches - l0
    load(eng, STATE_A, slot=1)
    load(eng, STATE_B, slot=2)
    eng.use(2)
    eng.search_node(1, outer=outer, middle=middle)
    l0 = eng.launches
    got = eng.enumerate7(outer, middle, 16)
    assert eng.launches - l0 == reuse
    load(ref, STATE_A)
    want = enum_fields(ref.enumerate7(outer, middle, 16))
    assert_same(enum_fields(got), want, "node moved")
    assert eng.decomp7_part(0, 1, outer, middle) == ref.decomp7_part(0, 1, outer, middle)
    # a batch leaves the current slot (A) alone; its lane 0 searched B, so A has no list now
    eng.search_batch([dict(slot=2, outer=outer, middle=middle), dict(slot=1, order5=order5)])
    with state_error(-4):
        eng.decomp7_part(0, 1, outer, middle)
    assert_same(enum_fields(eng.enumerate7(outer, middle, 16)), want, "after the batch")


@pytest.mark.parametrize("between", ["search5", "enumerate5", "enumerate3"])
def test_phase2_after_other_searches_on_the_installed_list(eng, ref, between):
    """An installed list outlives a search_5lut or an enumeration of the same problem: phase 2
    after it decides the whole list (B's first key from the oracle)."""
    order5, outer, middle = ORDERS
    lst, key, want = oracle_b()
    load(eng, STATE_B)
    assert eng.filter7_part(0, 1).shape[0] == len(lst)
    if between == "search5":
        eng.search5(order5)
    elif between == "enumerate5":
        eng.enumerate5(order5, 4)
    else:
        eng.enumerate3(list(range(14)), 4)
    k = eng.decomp7_part(0, 1, outer, middle)
    assert k == key, (between, hex(k), hex(key))
    assert_same(E.result7_fields(eng.finish7(k, outer, middle)), want, between)


# ------------------------------------------------------------------------------------------------
# b. batches that repeat a slot

def _repeat_state(n, mask_spec, seed):
    rs = np.random.RandomState(seed)
    tabs = S.synthetic_state(n, seed=seed)
    if mask_spec == "full":
        mask = FULL
    elif isinstance(mask_spec, int):
        mask = H.random_mask(rs, mask_spec)
    else:
        mask = S.mux_mask(mask_spec)
    if n > 60:   # a 5-LUT on low gates: the searches end early
        tgt = S.lut_table(0xCA, S.lut_table(0x96, tabs[9], tabs[12], tabs[17]), tabs[20], tabs[23])
    else:
        tgt = S.sbox_target(S.rijndael_sbox(), seed % 8)
    return tabs, tgt, mask


A_ = SCAN3 | SEARCH5 | SEARCH7
REPEAT_CASES = [
    # (name, n, mask, how the slot gets its state, flags of the wave's jobs on it, other jobs)
    ("lazy_mixed", 20, [(1, 0)], "load", [SCAN3, SEARCH7, SEARCH5 | SEARCH7, SEARCH7], 0),
    ("lazy_scan3_only", 33, [(3, 1), (5, 0)], "load", [SCAN3] * 8, 0),
    ("lazy_search7_only", 24, [(0, 1), (4, 0), (6, 1)], "load", [SEARCH7] * 5, 0),
    ("eager_rows_later", 40, 100, "stage", [SCAN3, SEARCH5, SEARCH7, SCAN3 | SEARCH7, SEARCH7], 2),
    ("eager_search7_only", 48, 70, "stage", [SEARCH7] * 8, 0),
    ("eager_sieve", 56, [(2, 1)], "stage", [SEARCH5, SEARCH7, A_], 3),
    ("pending_none", 30, [(7, 0)], "again", [SEARCH7, SCAN3 | SEARCH7, SEARCH7, A_], 1),
    ("bulk130_lazy", 130, "full", "load", [SEARCH5, SEARCH7, SEARCH7, SCAN3 | SEARCH7], 0),
    ("bulk130_eager", 130, "full", "stage", [SCAN3, A_, SEARCH7], 2),
    ("bulk500_lazy", 500, "full", "load", [SCAN3, SEARCH5 | SEARCH7, SEARCH5, A_], 0),
]


@pytest.mark.parametrize("case", REPEAT_CASES, ids=[c[0] for c in REPEAT_CASES])
def test_batch_repeating_a_slot_equals_single_calls(eng, ref, case):
    """One slot on 2-8 lanes of a wave, after a lazy load (every field of the problem block
    pending, or taking the bulk copy at n = 130 / 500), after an eager stage (rows pending; the
    first job on the slot without search_7lut and a later one with it) or with nothing pending
    (the same batch twice).  Each job's result equals the same job as a single search_node on
    `ref`, field for field.  The batch runs once: the ordering it checks is a data race on the
    shared slot, so this guards it but may pass without it."""
    name, n, mask_spec, how, flags, others = case
    st = _repeat_state(n, mask_spec, 8200 + n)
    other = _repeat_state(18, [(4, 1)], 8300)
    slot = 0 if how == "load" else 7
    load(eng, other, slot=3)
    if how == "load":
        load(eng, st)
    else:
        load(eng, st, slot=slot)
    jobs = []
    for j, f in enumerate(flags):
        if j < others:   # other slots on the lanes in front
            jobs.append(dict(slot=3, **H.job_kwargs(A_, 8400 + j, 18)))
        jobs.append(dict(slot=slot, **H.job_kwargs(f, 8500 + j, n)))
    jobs = jobs[:H.LANES]
    if how == "again":
        eng.search_batch(jobs)
    got = eng.search_batch(jobs)
    for j, (job, r) in enumerate(zip(jobs, got)):
        load(ref, other if job["slot"] == 3 else st)
        kw = {k: v for k, v in job.items() if k != "slot"}
        assert_same(node_fields(r), node_fields(ref.search_node(0, **kw)), (name, j))


# ------------------------------------------------------------------------------------------------
# c. seeded call sequences

class Runner:
    """Runs one generated sequence on `eng`, each step checked against `ref` (memoised per state
    and call) and the model."""

    def __init__(self, seed, ref):
        import torch
        self.seed, self.ref = seed, ref
        self.pool = H.make_pool(seed)
        self.ops = H.generate(seed, self.pool)
        self.eng = sb.LutEngine(0)
        self.model = H.Model(self.pool)
        self.side = torch.cuda.Stream()
        self.filter = None
        self.memo = {}

    def close(self):
        self.eng.close()

    def want(self, st, key, fn):
        k = (st.idx, key)
        if k not in self.memo:
            self.ref.load(*st.args())
            self.memo[k] = fn(self.ref)
        return self.memo[k]

    def ref_node(self, st, flags, seed):
        kw = H.job_kwargs(flags, seed, st.n)
        return self.want(st, ("node", flags, seed),
                         lambda r: node_fields(r.search_node(0, **kw)))

    def run(self):
        for i, op in enumerate(self.ops):
            try:
                self.step(op)
            except AssertionError as e:
                last = "\n  ".join(repr(o)[:200] for o in self.ops[max(0, i - 9):i + 1])
                raise AssertionError("seed %d, step %d: %s\nlast operations:\n  %s"
                                     % (self.seed, i, e, last)) from None

    def step(self, op):
        eng, m = self.eng, self.model
        kind = op[0]
        st = m.state()
        stages = None
        if kind == "load":
            eng.load(*self.pool[op[1]].args())
        elif kind == "stage":
            eng.stage(op[1], *self.pool[op[2]].args())
        elif kind == "use":
            eng.use(op[1])
        elif kind == "search5":
            o = H.job_orders(op[1], st.n)
            got = result_fields(eng.search5(o["order5"]), 5)
            assert_same(got, self.want(st, op, lambda r: result_fields(r.search5(o["order5"]), 5)),
                        op)
        elif kind == "search7":
            o = H.job_orders(op[1], st.n)
            got = result_fields(eng.search7(o["outer"], o["middle"]), 7)
            assert_same(got, self.want(st, op, lambda r: result_fields(
                r.search7(o["outer"], o["middle"]), 7)), op)
        elif kind == "node":
            slot, flags, seed = op[1:]
            tgt = m.state(slot)
            got = node_fields(eng.search_node(slot, **H.job_kwargs(flags, seed, tgt.n)))
            want = self.ref_node(tgt, flags, seed)
            assert_same(got, want, op[:3])
            stages = [want["found_stage"]]
        elif kind == "batch":
            jobs = [dict(slot=s, **H.job_kwargs(f, sd, m.state(s).n)) for s, f, sd in op[1]]
            got = eng.search_batch(jobs)
            stages = []
            for j, ((s, f, sd), r) in enumerate(zip(op[1], got)):
                want = self.ref_node(m.state(s), f, sd)
                assert_same(node_fields(r), want, ("batch job", j, s, f))
                stages.append(want["found_stage"])
        elif kind == "filter":
            self.phase_steps(st, *op[1:])
        elif kind == "enum":
            if not self.enumerate(st, *op[1:]):
                return
        elif kind == "consume":
            if not self.consume(st, op[1], op[2]):
                return
        elif kind == "stream":
            eng.set_stream(self.side.cuda_stream if op[1] else None)
        elif kind == "depth":
            if op[1]:
                rs = np.random.RandomState(op[3])
                self.filter = (rs.randint(0, 6, op[2]), int(rs.randint(2, 9)))
                eng.set_depth_filter(*self.filter)
            else:
                self.filter = None
                eng.clear_depth_filter()
        m.apply(op, stages)

    def phase_steps(self, st, nparts, on_device, seed):
        """filter7_part of every part, the lists merged (set_list7, or set_list7_device from
        list7_device's pointers), decomp7_part of every part, the minimum key to finish7."""
        import torch
        eng = self.eng
        o = H.job_orders(seed, st.n)

        def steps(r, device):
            lists = []
            if device:
                for p in range(nparts):
                    cnt = r.filter7_part_device(p, nparts)
                    ptr, c2 = r.list7_device()
                    assert c2 == cnt, (p, nparts, c2, cnt)
                    lists.append(device_list(ptr, cnt))
                stride = max(1, max(len(x) for x in lists))
                buf = torch.zeros((nparts, stride), dtype=torch.int64, device="cuda")
                for p, x in enumerate(lists):
                    if len(x):
                        buf[p, :len(x)] = torch.from_numpy(x.view(np.int64)).cuda()
                torch.cuda.synchronize()
                r.set_list7_device(buf.data_ptr(), stride, [len(x) for x in lists])
            else:
                lists = [r.filter7_part(p, nparts) for p in range(nparts)]
                r.set_list7(np.concatenate(lists))
            keys = [r.decomp7_part(p, nparts, o["outer"], o["middle"]) for p in range(nparts)]
            res = r.finish7(min(keys), o["outer"], o["middle"])
            return [x.tobytes() for x in lists], keys, result_fields(res, 7)

        got = steps(eng, on_device)
        want = self.want(st, ("filter", nparts, seed), lambda r: steps(r, False))
        assert got[0] == want[0], ("part lists", nparts, on_device)
        assert got[1] == want[1], ("part keys", got[1], want[1])
        assert_same(got[2], want[2], ("finish7", nparts))

    def enumerate(self, st, width, count, max_matches, seed):
        """enumerate3/5/7 (counted or not) and, after a count, a fetch and a pick; under the depth
        filter when one is set.  Returns False where the call must fail (a filter of another
        size)."""
        eng = self.eng
        o = H.job_orders(seed, st.n)
        args = {3: [o["gate_order"]], 5: [o["order5"]], 7: [o["outer"], o["middle"]]}[width]
        if self.filter is not None and len(self.filter[0]) != st.n:
            with state_error(-1):
                getattr(eng, "enumerate%d" % width)(*args, max_matches, count=count)
            return False
        flt = self.filter

        def calls(r):
            if flt is not None:
                r.set_depth_filter(*flt)
            try:
                e = getattr(r, "enumerate%d" % width)(*args, max_matches, count=count)
                out = [enum_fields(e)]
                if count and e.total:
                    rs = np.random.RandomState(seed)
                    out.append(r.fetch_matches(int(rs.randint(e.total)), 7).tobytes())
                    out.append(r.pick_matches(rs.randint(0, e.total, 5)).tobytes())
                return out
            finally:
                if flt is not None:
                    r.clear_depth_filter()

        key = ("enum", width, count, max_matches, seed,
               None if flt is None else (flt[0].tobytes(), flt[1]))
        want = self.want(st, key, calls)
        e = getattr(eng, "enumerate%d" % width)(*args, max_matches, count=count)
        got = [enum_fields(e)]
        if count and e.total:
            rs = np.random.RandomState(seed)
            got.append(eng.fetch_matches(int(rs.randint(e.total)), 7).tobytes())
            got.append(eng.pick_matches(rs.randint(0, e.total, 5)).tobytes())
        assert_same(got[0], want[0], ("enumerate", width, count, max_matches))
        assert got[1:] == want[1:], ("fetch / pick", width)
        return True

    def consume(self, st, what, seed):
        """A consumer of the installed list: what the model says lane 0 holds for the current
        problem decides between the list's answers and SBG_ERR_STATE / an empty list."""
        eng = self.eng
        if what == "enum7":
            return self.enumerate(st, 7, True, 16, seed)
        o = H.job_orders(seed, st.n)
        have = self.model.list_of_current()
        if what == "decomp":
            if have != ("whole",):
                with state_error(-4):
                    eng.decomp7_part(0, 1, o["outer"], o["middle"])
                with state_error(-4):
                    eng.finish7(0, o["outer"], o["middle"])
                return True

            # finish7's sweep is that of the phase 1 behind the installed list: the whole space's,
            # or the last part's where the parts' lists were merged
            parts = self.model.lst_parts

            def calls(r):
                if parts == 1:
                    r.filter7_part(0, 1)
                else:
                    r.set_list7(np.concatenate([r.filter7_part(p, parts) for p in range(parts)]))
                k = r.decomp7_part(0, 1, o["outer"], o["middle"])
                return k, result_fields(r.finish7(k, o["outer"], o["middle"]), 7)
            k = eng.decomp7_part(0, 1, o["outer"], o["middle"])
            got = (k, result_fields(eng.finish7(k, o["outer"], o["middle"]), 7))
            want = self.want(st, ("decomp", seed, parts), calls)
            assert got[0] == want[0], ("decomp7_part", hex(got[0]), hex(want[0]))
            assert_same(got[1], want[1], "finish7")
            return True
        ptr, cnt = eng.list7_device()
        if have is None:
            assert cnt == 0, ("list7_device without a list of the current problem", cnt)
        else:
            assert have == ("whole",), have
            want = self.want(st, ("list",), lambda r: r.filter7_part(0, 1).tobytes())
            assert device_list(ptr, cnt).tobytes() == want, ("list7_device", cnt)
        return True


@pytest.mark.parametrize("seed", H.SEEDS)
def test_seeded_call_sequence(ref, seed):
    """About 300 calls over a pool of 12 states on one handle (see tests/_handle_support.py): every
    result equals `ref`'s for the state the model says is current, and every call the header says
    fails with SBG_ERR_STATE does."""
    run = Runner(seed, ref)
    try:
        run.run()
    finally:
        run.close()
