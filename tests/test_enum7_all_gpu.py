"""GPU: the whole-space 7-LUT enumeration (sbg_enum7_all, LutEngine.enumerate7_all).

- Seeded small states (n = 7..20, every words-per-table width with a partly padded last word,
  excluded input bits, degenerate gates; plain, filtered and grouped forms) against the test-side
  reference (tests/_enum7_all_reference.py): totals, feasible counts, first K counted and
  count-free, pages, picks, samples, group sizes and depth histograms byte for byte, and shares in
  2, 3 and 5 parts with global ranks.
- Against the list form: on a state whose list is not cut, the same matches; on states whose list
  is cut, the list's matches are exactly the whole space's first ones.
- Closed-form totals under the empty mask.
- A shallow 7-LUT on the highest-numbered gates of a state whose list is cut: found with
  shallowest_matches(whole=True), out of reach of the list form.
- The installed list is left alone, and bad arguments are refused."""
import ctypes as C
from math import comb

import numpy as np
import pytest

import _enum7_all_reference as W
import _enum_reference as R
import _enum_support as E
import _support as S
import bench
import sboxgates_b200 as sb
from sboxgates_b200 import lut, native
from test_enum_depth_gpu import _nw
from test_handle_calls_gpu import result_fields
from test_enum_fuzz_gpu import DEGENERATE, MUX, RANDOM_POSITIONS, _Checker, _cut, _random_mask

pytestmark = pytest.mark.gpu

SBG_ERR_ARG, SBG_ERR_STATE = -1, -4
NWS = (1, 2, 4, 8)
FORMS = ("plain", "filtered", "grouped")
MAX_FEASIBLE = 40   # the key oracle tries all 70 x 65,536 positions of every feasible combination
LOW23 = (1 << 23) - 1


class Config:
    """One drawn state and its settings; words per table and kernel form follow from idx."""

    def __init__(self, seed, idx, attempt):
        rs = self.rs = np.random.RandomState([seed, idx, attempt])
        self.seed, self.idx, self.attempt = seed, idx, attempt
        self.width, self.nw, self.form = 7, NWS[idx % 4], FORMS[(idx // 4) % 3]
        self.n = n = int(rs.randint(7, max(8, 21 - attempt)))
        if rs.rand() < 0.3:
            self.mask_spec, self.mask = "mux", S.mux_mask(MUX[self.nw])
        else:
            lo, hi = RANDOM_POSITIONS[self.nw][int(rs.randint(2))]
            count = int(rs.randint(lo, hi + 1))
            self.mask_spec, self.mask = "r%d" % count, _random_mask(rs, count)
        assert _nw(self.mask) == self.nw
        self.inbits = sorted(int(x) for x in rs.choice(8, int(rs.randint(0, 4)), replace=False))
        allowed = [g for g in range(n) if g not in self.inbits]
        tabs = S.synthetic_state(n, seed=int(rs.randint(1 << 30)))
        self.planted = []
        if len(allowed) >= 7 and rs.rand() < 0.8:
            g = [int(x) for x in rs.choice(allowed, 7, replace=False)]
            f = [int(x) for x in rs.randint(1, 255, 3)]
            tgt = S.lut_table(f[2], S.lut_table(f[0], tabs[g[0]], tabs[g[1]], tabs[g[2]]),
                              S.lut_table(f[1], tabs[g[3]], tabs[g[4]], tabs[g[5]]), tabs[g[6]])
            self.planted = g
        else:
            tgt = S.sbox_target(S.rijndael_sbox(), int(rs.randint(8)))
        self.degenerate = []
        free = [g for g in range(8, n) if g not in self.planted]
        if free and rs.rand() < 0.5:
            for g in rs.choice(free, min(len(free), int(rs.randint(1, 4))), replace=False):
                d = str(rs.choice(DEGENERATE))
                src = int(rs.randint(n))
                tabs[g] = {"duplicate": tabs[src], "complement": ~tabs[src],
                           "zero": np.zeros(4, dtype=np.uint64), "one": np.full(4, R.ONES),
                           "target": tgt, "not_target": ~tgt}[d]
                self.degenerate.append((int(g), d))
        self.tables, self.target = tabs, tgt
        self.orders = (bytes(rs.permutation(256).astype(np.uint8)),
                       bytes(rs.permutation(256).astype(np.uint8)))
        self.gate_depth = rs.randint(0, 9, n).astype(np.uint16)
        self.nparts = (2, 3, 5)[idx % 3]

    def tag(self):
        return "seed %d config %d attempt %d: n %d NW %d mask %s inbits %s degenerate %s form %s" % (
            self.seed, self.idx, self.attempt, self.n, self.nw, self.mask_spec, self.inbits,
            self.degenerate, self.form)

    def settings(self, ref):
        """depth / bound, function sets and grouping for the config's form."""
        rs = self.rs
        st = dict(depth=None, bound=None, outer=None, middle=None, inner=None, grouping=None,
                  functions=False)
        if self.form == "plain":
            return st
        dep = E.record_depths(ref.all, self.gate_depth)
        if self.form == "grouped":
            st["grouping"] = ("shape", "tuple")[self.idx % 2]
        use_depth = rs.rand() < 0.6 or self.form == "filtered"
        if use_depth:
            st["depth"] = self.gate_depth
            st["bound"] = int(rs.randint(dep.min(), dep.max() + 1)) if len(dep) else 4
        if rs.rand() < 0.6 or (self.form == "filtered" and not use_depth):
            st["functions"] = True
            pick = ref.all[int(rs.randint(len(ref.all)))] if len(ref.all) else None
            if pick is not None and rs.rand() < 0.5:
                st["middle"] = [int(pick["func_middle"])]
            else:
                st["outer"] = sorted(int(x) for x in rs.choice(256, 128, replace=False))
            if rs.rand() < 0.4:
                st["inner"] = sorted(sb.AFFINE_FUNCTIONS)
        return st


def _apply(eng, cfg, st):
    eng.load(cfg.tables, cfg.target, cfg.mask, cfg.inbits)
    if st["depth"] is not None:
        eng.set_depth_filter(st["depth"], st["bound"])
    else:
        eng.clear_depth_filter()
    if st["functions"]:
        eng.set_function_filter(st["outer"], st["middle"], st["inner"])
    else:
        eng.clear_function_filter()
    eng.set_grouping(st["grouping"])


def _reset(eng):
    eng.set_grouping(None)
    eng.clear_function_filter()
    eng.clear_depth_filter()


def _draw(seed, idx):
    for attempt in range(40):
        cfg = Config(seed, idx, attempt)
        feas = W.feasible_tuples(cfg.tables, cfg.target, cfg.mask, cfg.inbits)
        if not 1 <= len(feas) <= MAX_FEASIBLE:
            continue
        total, keys, _ = R.oracle_keys(7, cfg.tables, cfg.target, cfg.mask, cfg.inbits,
                                       cfg.orders, tuples=feas)
        if keys is not None:
            return cfg, W.WholeReference(cfg.tables, cfg.target, cfg.mask, cfg.inbits,
                                         cfg.orders, tuples=feas, keys=keys)
    raise AssertionError("seed %d config %d: no state drawn" % (seed, idx))


@pytest.fixture(scope="module")
def shares():
    engs = [sb.LutEngine(0) for _ in range(5)]
    yield engs
    for e in engs:
        e.close()


@pytest.mark.parametrize("idx", range(12))
def test_random_states_match_the_reference(engine, shares, idx):
    import collections
    cfg, ref = _draw(17, idx)
    st = cfg.settings(ref)
    ref.select(st["depth"], st["bound"], st["outer"], st["middle"], st["inner"], st["grouping"],
               st["functions"])
    want, t = ref.recs, ref.total
    chk = _Checker(cfg, collections.Counter())
    tag = chk.tag
    rs = np.random.RandomState([cfg.seed, idx, 99])
    try:
        _apply(engine, cfg, st)
        for k in sorted({0, 1, int(rs.randint(0, t + 2)), t, t + 1}):
            e = engine.enumerate7_all(*cfg.orders, k)
            assert (e.total, e.feasible) == (t, ref.feasible), (tag, k, e.total, t, e.feasible,
                                                                ref.feasible)
            chk.same(e.matches, want[:k], "first", "first %d" % k)
            if st["depth"] is not None:
                assert np.array_equal(engine.depth_counts(), ref.hist), (tag, "depth_counts")
            f = engine.enumerate7_all(*cfg.orders, k, count=False)
            assert f.total is None, tag
            chk.same(f.matches, want[:k], "free", "count-free first %d" % k)
        e = engine.enumerate7_all(*cfg.orders, 0)
        for first, count in _cut(rs, t, ref.seams()):
            chk.same(engine.fetch_matches(first, count), want[first:first + count], "page",
                     "page (%d, %d)" % (first, count))
        if t:
            ranks = rs.randint(0, t, int(rs.randint(1, 300)))
            ranks = np.concatenate([ranks, ranks[:10], [t - 1, 0]])
            rs.shuffle(ranks)
            chk.same(engine.pick_matches(ranks), want[ranks], "pick", "pick")
            r, got = sb.sample_matches(engine, e, min(t, 100), seed=idx)
            chk.same(got, want[r.astype(np.int64)], "sample", "sample")
            sizes = engine.group_sizes(ranks)
            want_sizes = ref.group_sizes(**st)[ranks] if st["grouping"] else np.ones(len(ranks))
            assert np.array_equal(sizes, want_sizes.astype(np.uint64)), (tag, "group sizes")
        _check_shares(shares[:cfg.nparts], cfg, st, ref, chk, rs)
    finally:
        _reset(engine)


def _check_shares(engs, cfg, st, ref, chk, rs):
    P = len(engs)
    tag, want, t = chk.tag, ref.recs, ref.total
    counts = []
    try:
        for q, eng in enumerate(engs):
            _apply(eng, cfg, st)
            mine = ref.share(q, P)
            k = min(len(mine), int(rs.randint(0, 200)))
            e = eng.enumerate7_all(*cfg.orders, k, True, q, P)
            assert e.total == len(mine), (tag, "share", q, P, e.total, len(mine))
            chk.same(e.matches, mine[:k], "share", "share %d/%d first %d" % (q, P, k))
            f = eng.enumerate7_all(*cfg.orders, k, False, q, P)
            chk.same(f.matches, mine[:k], "share", "share %d/%d count-free" % (q, P))
            eng.enumerate7_all(*cfg.orders, 0, True, q, P)
            sums = eng.enum_block_sums()
            assert sums.tobytes() == ref.share_sums(q, P).tobytes(), (tag, "block sums", q, P)
            counts.append(len(sums))
        sums = np.zeros((P, max(max(counts), 1)), dtype=np.uint64)
        for q in range(P):
            sums[q, :counts[q]] = ref.share_sums(q, P)
        assert [eng.enum_set_global(sums, counts) for eng in engs] == [t] * P, (tag, "global")
        for first, count in _cut(rs, t, ref.seams())[:4]:
            got = sum(eng.fetch_matches(first, count).view(np.uint64) for eng in engs)
            chk.same(got.view(sb.MATCH_DTYPE).reshape(-1), want[first:first + count], "global",
                     "global page (%d, %d)" % (first, count))
        if t:
            ranks = rs.randint(0, t, int(rs.randint(1, 200)))
            got = sum(eng.pick_matches(ranks).view(np.uint64) for eng in engs)
            chk.same(got.view(sb.MATCH_DTYPE).reshape(-1), want[ranks], "global", "global pick")
    finally:
        for eng in engs:
            _reset(eng)


# ------------------------------------------------------------------------------------------------
# Against the list form.

def _list_ranks(eng, n):
    """The combination rank of every entry of the installed (freshly built) phase-1 list."""
    return W.lex_ranks(E.unpack_list(eng.filter7_part(0, 1)), n)


def _to_whole(recs, ranks):
    out = recs.copy()
    idx = (out["key"] >> np.uint64(23)).astype(np.int64)
    out["key"] = (ranks[idx].astype(np.uint64) << np.uint64(23)) | (out["key"] & np.uint64(LOW23))
    return out


def test_uncut_list_gives_the_same_matches(engine):
    st = bench.build_batch(40, 4, 1)[3]   # n = 40 under 32 positions
    engine.load(st["tables"], st["target"], st["mask"], st["inbits"])
    ranks = _list_ranks(engine, 40)
    assert 0 < len(ranks) < lut.SBG_LIST_CAP
    lst = engine.enumerate7(st["outer"], st["middle"], 1 << 16)
    whole = engine.enumerate7_all(st["outer"], st["middle"], 1 << 16)
    assert lst.feasible == len(ranks)
    assert (whole.total, whole.feasible) == (lst.total, len(ranks))
    assert whole.matches.tobytes() == _to_whole(lst.matches, ranks).tobytes()
    t = lst.total
    pick = np.random.RandomState(5).randint(0, t, 4096) if t else np.zeros(0, dtype=np.int64)
    page = max(t // 2 - 2048, 0)
    engine.enumerate7(st["outer"], st["middle"], 0)
    want = [engine.fetch_matches(page, 4096), engine.pick_matches(pick)]
    engine.enumerate7_all(st["outer"], st["middle"], 0)
    got = [engine.fetch_matches(page, 4096), engine.pick_matches(pick)]
    for g, w in zip(got, want):
        assert g.tobytes() == _to_whole(w, ranks).tobytes()


@pytest.mark.parametrize("case", ["bench64", "empty24"])
def test_cut_list_is_the_start_of_the_whole_space(engine, case):
    """The list is the first SBG_LIST_CAP feasible combinations in rank order, so its matches are
    the whole space's matches up to its last combination: the same records at the same ranks."""
    if case == "bench64":
        st = bench.build_batch(64, 4, 1)[3]
        tables, target, mask, inbits = st["tables"], st["target"], st["mask"], st["inbits"]
        outer, middle = st["outer"], st["middle"]
    else:
        st = bench.build_batch(40, 4, 1)[0]
        tables, target, mask, inbits = bench._state(24, 1024), st["target"], \
            np.zeros(4, dtype=np.uint64), []
        outer, middle = st["outer"], st["middle"]
    engine.load(tables, target, mask, inbits)
    ranks = _list_ranks(engine, len(tables))
    assert len(ranks) == lut.SBG_LIST_CAP
    lst = engine.enumerate7(outer, middle, 4096)
    L = lst.total
    whole = engine.enumerate7_all(outer, middle, 4096)
    assert whole.total >= L and whole.feasible > lut.SBG_LIST_CAP
    k = min(L, 4096)
    assert whole.matches[:k].tobytes() == _to_whole(lst.matches[:k], ranks).tobytes()
    rs = np.random.RandomState(3)
    at = sorted({0, max(L - 4096, 0), L // 2, int(rs.randint(0, max(L, 1)))})
    picks = rs.randint(0, max(L, 1), 4096) if L else np.zeros(0, dtype=np.int64)
    engine.enumerate7(outer, middle, 0)
    want = [engine.fetch_matches(a, 4096) for a in at] + [engine.pick_matches(picks)]
    engine.enumerate7_all(outer, middle, 0)
    got = [engine.fetch_matches(a, 4096) for a in at] + [engine.pick_matches(picks)]
    for g, w in zip(got, want):
        assert g.tobytes() == _to_whole(w, ranks).tobytes()
    if whole.total > L:
        nxt = engine.fetch_matches(L, 1)
        assert int(nxt["key"][0]) >> 23 > int(ranks[-1])


# ------------------------------------------------------------------------------------------------
# Closed forms under the empty mask: every combination is feasible, every position matches.

def _empty(engine, n):
    engine.load(bench._state(n, 1000 + n), bench._rijndael_bit(0), np.zeros(4, dtype=np.uint64),
                [])
    return bench.build_batch(40, 4, 1)[0]


def test_empty_mask_totals_n24(engine):
    st = _empty(engine, 24)
    try:
        for grouping, want in ((None, 346104 * 4587520), ("shape", 346104 * 70),
                               ("tuple", 346104)):
            engine.set_grouping(grouping)
            e = engine.enumerate7_all(st["outer"], st["middle"], 8)
            assert (e.total, e.feasible) == (want, 346104), grouping
            assert R.check_realises(e.matches, bench._state(24, 1024), bench._rijndael_bit(0),
                                    np.zeros(4, dtype=np.uint64)) == 8
    finally:
        engine.set_grouping(None)


def test_empty_mask_tuple_groups_n40(engine):
    st = _empty(engine, 40)
    try:
        engine.set_grouping("tuple")
        e = engine.enumerate7_all(st["outer"], st["middle"], 0)
        assert (e.total, e.feasible) == (comb(40, 7), comb(40, 7)) == (18643560, 18643560)
        last = engine.fetch_matches(e.total - 1, 1)
        assert int(last["key"][0]) >> 23 == comb(40, 7) - 1
    finally:
        engine.set_grouping(None)


# ------------------------------------------------------------------------------------------------
# What the feature is for: a shallow realisation on late gates.

def test_shallowest_realisation_on_late_gates(engine):
    rs = np.random.RandomState(8)
    n = 44
    tables = bench._state(n, 4400)
    late = list(range(n - 7, n))
    f = [0x96, 0xE8, 0xCA]
    target = S.lut_table(f[2], S.lut_table(f[0], *tables[late[:3]]),
                         S.lut_table(f[1], *tables[late[3:6]]), tables[late[6]])
    mask = _random_mask(rs, 24)
    depth = np.full(n, 3, dtype=np.uint16)
    depth[:8] = 2
    depth[late] = 0   # the planted circuit has depth 2, anything with another gate at least 3
    outer, middle = (bytes(rs.permutation(256).astype(np.uint8)) for _ in range(2))
    try:
        engine.load(tables, target, mask, [])
        d, total, recs = sb.shallowest_matches(engine, 7, (outer, middle), depth, 64, whole=True)
        assert d == 2 and total >= 1
        assert all(sorted(int(g) for g in r["gates"]) == late for r in recs)
        assert R.check_realises(recs, tables, target, mask) == len(recs)
        engine.clear_depth_filter()
        e = engine.enumerate7_all(outer, middle, 0)
        assert e.feasible > lut.SBG_LIST_CAP   # the list form's list is cut
        d_list, _, recs_list = sb.shallowest_matches(engine, 7, (outer, middle), depth, 64)
        assert d_list is None or d_list > 2
        assert not any(sorted(int(g) for g in r["gates"]) == late for r in recs_list)
    finally:
        engine.clear_depth_filter()


# ------------------------------------------------------------------------------------------------
# The installed list, and bad arguments.

def test_installed_list_is_left_alone(engine):
    rs = np.random.RandomState(12)
    n = 14
    tables = S.synthetic_state(n, seed=1212)
    g = [int(x) for x in rs.choice(range(1, n), 7, replace=False)]
    target = S.lut_table(0x6A, S.lut_table(0x96, *tables[g[:3]]),
                         S.lut_table(0xE8, *tables[g[3:6]]), tables[g[6]])
    mask = S.mux_mask([(2, 1)])
    outer, middle = (bytes(rs.permutation(256).astype(np.uint8)) for _ in range(2))
    engine.load(tables, target, mask, [0])
    r1 = engine.search7(outer, middle)
    e1 = engine.enumerate7(outer, middle, 1000)
    engine.enumerate7_all(outer, middle, 1000)
    e2 = engine.enumerate7(outer, middle, 1000)
    engine.enumerate7_all(outer, middle, 10, count=False)
    r2 = engine.search7(outer, middle)
    assert r1.found and result_fields(r1, 7) == result_fields(r2, 7)
    assert (e1.total, e1.feasible, e1.matches.tobytes()) == \
        (e2.total, e2.feasible, e2.matches.tobytes())


def test_bad_arguments(engine):
    lib = native.load_library()
    n_out, total, feas = C.c_uint64(), C.c_uint64(), C.c_uint64()
    out = np.zeros(4, dtype=sb.MATCH_DTYPE)
    order = (C.c_uint8 * 256)(*range(256))

    def call(eng):
        return lib.sbg_enum7_all(eng._h, 0, 1, order, order, 4,
                                 out.ctypes.data_as(C.c_void_p), C.byref(n_out), C.byref(total),
                                 C.byref(feas))
    fresh = sb.LutEngine(0)
    try:
        assert call(fresh) == SBG_ERR_STATE
    finally:
        fresh.close()
    for n in (6, 65):
        tabs = bench._state(n, n)
        engine.load(tabs, bench._rijndael_bit(0), S.mux_mask([]), [])
        engine.enumerate5(order, 0)
        assert call(engine) == SBG_ERR_ARG, n
        with pytest.raises(RuntimeError):   # the failed call ended the cursor
            engine.fetch_matches(0, 1)
    tabs = bench._state(12, 12)
    engine.load(tabs, bench._rijndael_bit(0), S.mux_mask([]), [])
    try:
        engine.set_depth_filter(np.zeros(11, dtype=np.uint16), 5)
        assert call(engine) == SBG_ERR_ARG
    finally:
        engine.clear_depth_filter()
    assert call(engine) == 0
