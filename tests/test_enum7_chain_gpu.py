"""GPU: the 7-LUT chain enumeration (sbg_enum7_chain, LutEngine.enumerate7_chain).

- Seeded small states (n = 7..20, every words-per-table width with a partly padded last word,
  excluded input bits, degenerate gates; plain, filtered and grouped forms) against the test-side
  chain oracle (tests/enum_chain_oracle.c through tests/_enum_chain_reference.py): totals,
  feasible counts, first K counted and count-free, pages, picks, samples, group sizes and depth
  histograms byte for byte, and shares in 2, 3 and 5 parts with global ranks.  Every returned
  record is rebuilt on the host.
- Closed-form totals under the empty mask.
- Against sbg_enum5: the chain matches whose L2 is the projection onto L1 are the 5-LUT matches.
- A chain planted on the highest-numbered gates, found by shallowest_matches(shape="chain").
- The installed list is left alone, and bad arguments are refused."""
import collections
import ctypes as C
from math import comb

import numpy as np
import pytest

import _enum7_all_reference as W
import _enum_chain_reference as CR
import _enum_reference as R
import _support as S
import bench
import sboxgates_b200 as sb
from sboxgates_b200 import lut, native
from test_enum_depth_gpu import _nw
from test_enum_fuzz_gpu import DEGENERATE, MUX, RANDOM_POSITIONS, _random_mask
from test_handle_calls_gpu import result_fields

pytestmark = pytest.mark.gpu

SBG_ERR_ARG, SBG_ERR_STATE = -1, -4
NWS = (1, 2, 4, 8)
FORMS = ("plain", "filtered", "grouped")
MAX_FEASIBLE = 24   # the oracle decides all 210 x 65,536 candidates of every feasible combination
MAX_MATCHES = 1 << 20
PER_COMB = 210 * 65536
SHIFT = {"shape": 16, "tuple": 24}


def _planted_chain(rs, tabs, gates):
    f = [int(x) for x in rs.randint(1, 255, 3)]
    x1 = S.lut_table(f[0], tabs[gates[0]], tabs[gates[1]], tabs[gates[2]])
    x2 = S.lut_table(f[1], x1, tabs[gates[3]], tabs[gates[4]])
    return S.lut_table(f[2], x2, tabs[gates[5]], tabs[gates[6]])


class Config:
    def __init__(self, seed, idx, attempt):
        rs = self.rs = np.random.RandomState([seed, idx, attempt])
        self.idx = idx
        self.nw, self.form = NWS[idx % 4], FORMS[(idx // 4) % 3]
        self.n = n = int(rs.randint(7, max(8, 21 - attempt)))
        if rs.rand() < 0.3:
            self.mask = S.mux_mask(MUX[self.nw])
        else:
            lo, hi = RANDOM_POSITIONS[self.nw][int(rs.randint(2))]
            self.mask = _random_mask(rs, int(rs.randint(lo, hi + 1)))
        assert _nw(self.mask) == self.nw
        self.inbits = sorted(int(x) for x in rs.choice(8, int(rs.randint(0, 4)), replace=False))
        allowed = [g for g in range(n) if g not in self.inbits]
        tabs = S.synthetic_state(n, seed=int(rs.randint(1 << 30)))
        planted = []
        if len(allowed) >= 7 and rs.rand() < 0.8:
            planted = sorted(int(x) for x in rs.choice(allowed, 7, replace=False))
            tgt = _planted_chain(rs, tabs, [planted[i] for i in rs.permutation(7)])
        else:
            tgt = S.sbox_target(S.rijndael_sbox(), int(rs.randint(8)))
        self.degenerate = []
        free = [g for g in range(8, n) if g not in planted]
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
        self.tag = "config %d attempt %d: n %d NW %d inbits %s degenerate %s form %s" % (
            idx, attempt, n, self.nw, self.inbits, self.degenerate, self.form)

    def settings(self, recs):
        rs = self.rs
        st = dict(depth=None, bound=None, outer=None, middle=None, inner=None, grouping=None)
        if self.form == "plain":
            return st
        if self.form == "grouped":
            st["grouping"] = ("shape", "tuple")[self.idx % 2]
        if rs.rand() < 0.6 or self.form == "filtered":
            dep = CR.chain_depths(recs, self.gate_depth)
            st["depth"] = self.gate_depth
            st["bound"] = int(rs.randint(dep.min(), dep.max() + 1)) if len(dep) else 5
        if rs.rand() < 0.6:
            if len(recs) and rs.rand() < 0.5:
                st["middle"] = [int(recs[int(rs.randint(len(recs)))]["func_middle"])]
            else:
                st["outer"] = sorted(int(x) for x in rs.choice(256, 128, replace=False))
            if rs.rand() < 0.4:
                st["inner"] = sorted(sb.AFFINE_FUNCTIONS)
        return st


class ChainReference:
    """The oracle's matches of a state under one setting: recs in key order (one per group when
    grouped), total, feasible, the depth histogram, group sizes, and each record's 6-gate prefix
    ticket for the shares."""

    def __init__(self, cfg, feas, allrecs, st):
        n = cfg.n
        ok = np.ones(len(allrecs), dtype=bool)
        self.feasible = len(feas)
        if st["depth"] is not None:
            dep = CR.chain_depths(allrecs, st["depth"])
            ok &= dep <= st["bound"]
            d = np.asarray(st["depth"], dtype=np.int64)[feas.astype(np.int64)]
            srt = np.sort(d, axis=1)
            B = st["bound"]
            # a chain row within B: all below B, at most two at >= B - 1, four at >= B - 2
            self.feasible = int(((srt[:, 6] < B) & (srt[:, 4] < B - 1) & (srt[:, 2] < B - 2)).sum())
        if st["outer"] is not None or st["middle"] is not None or st["inner"] is not None:
            ok &= R.function_ok(allrecs, st["outer"], st["middle"], st["inner"])
        kept = allrecs[ok]
        g = st["grouping"]
        ids = kept["key"] >> np.uint64(SHIFT[g]) if g else kept["key"]
        uniq, first, counts = np.unique(ids, return_index=True, return_counts=True)
        self.recs = kept[first] if g else kept
        self.sizes = counts.astype(np.uint64) if g else np.ones(len(kept), dtype=np.uint64)
        self.total = len(self.recs)
        self.hist = None
        if st["depth"] is not None:
            self.hist = lut._trim(np.bincount(CR.chain_depths(self.recs, st["depth"]),
                                              minlength=1).astype(np.uint64))
        combos = np.sort(self.recs["gates"].astype(np.int64), axis=1)
        self.items = W.lex_ranks(combos[:, :6], n - 1) if self.total else np.zeros(0, np.int64)
        self.nblocks = -(-comb(n - 1, 6) // R.KDEAL)

    def share(self, q, P):
        return self.recs[(self.items // R.KDEAL) % P == q]

    def share_sums(self, q, P):
        blocks = self.items // R.KDEAL
        mine = np.arange(q, self.nblocks, P)
        return np.array([(blocks == b).sum() for b in mine], dtype=np.uint64)


def _draw(seed, idx):
    for attempt in range(60):
        cfg = Config(seed, idx, attempt)
        feas = W.feasible_tuples(cfg.tables, cfg.target, cfg.mask, cfg.inbits)
        if not 1 <= len(feas) <= MAX_FEASIBLE:
            continue
        ref = CR.chain_reference(cfg.tables, cfg.target, cfg.mask, cfg.inbits, cfg.orders,
                                 cap=MAX_MATCHES)
        if ref is not None:
            return (cfg,) + ref
    raise AssertionError("config %d: no state drawn" % idx)


def _apply(eng, cfg, st):
    eng.load(cfg.tables, cfg.target, cfg.mask, cfg.inbits)
    if st["depth"] is not None:
        eng.set_depth_filter(st["depth"], st["bound"])
    else:
        eng.clear_depth_filter()
    if st["outer"] is not None or st["middle"] is not None or st["inner"] is not None:
        eng.set_function_filter(st["outer"], st["middle"], st["inner"])
    else:
        eng.clear_function_filter()
    eng.set_grouping(st["grouping"])


def _reset(eng):
    eng.set_grouping(None)
    eng.clear_function_filter()
    eng.clear_depth_filter()


def _same(got, want, cfg, what):
    assert got.tobytes() == want.tobytes(), (cfg.tag, what, len(got), len(want))
    for r in got[:64]:
        fill = lut.allowed_fill(r["func_inner"], r["inner_seen"])
        assert CR.rebuild_ok(r, cfg.tables, cfg.target, cfg.mask, fill), (cfg.tag, what, r)


@pytest.fixture(scope="module")
def shares():
    engs = [sb.LutEngine(0) for _ in range(5)]
    yield engs
    for e in engs:
        e.close()


@pytest.mark.parametrize("idx", range(12))
def test_random_states_match_the_oracle(engine, shares, idx):
    cfg, feas, allrecs = _draw(23, idx)
    st = cfg.settings(allrecs)
    ref = ChainReference(cfg, feas, allrecs, st)
    want, t = ref.recs, ref.total
    rs = np.random.RandomState([idx, 99])
    try:
        _apply(engine, cfg, st)
        for k in sorted({0, 1, int(rs.randint(0, t + 2)), t, t + 1}):
            e = engine.enumerate7_chain(*cfg.orders, k)
            assert (e.total, e.feasible) == (t, ref.feasible), (cfg.tag, k, e.total, t,
                                                                e.feasible, ref.feasible)
            _same(e.matches, want[:k], cfg, "first %d" % k)
            if st["depth"] is not None:
                assert np.array_equal(engine.depth_counts(), ref.hist), (cfg.tag, "depth_counts")
            f = engine.enumerate7_chain(*cfg.orders, k, count=False)
            assert f.total is None
            _same(f.matches, want[:k], cfg, "count-free first %d" % k)
        e = engine.enumerate7_chain(*cfg.orders, 0)
        for first in sorted({0, t // 2, max(t - 50, 0), t}):
            _same(engine.fetch_matches(first, 100), want[first:first + 100], cfg, "page %d" % first)
        if t:
            ranks = rs.randint(0, t, int(rs.randint(1, 300)))
            ranks = np.concatenate([ranks, ranks[:10], [t - 1, 0]])
            rs.shuffle(ranks)
            _same(engine.pick_matches(ranks), want[ranks], cfg, "pick")
            r, got = sb.sample_matches(engine, e, min(t, 100), seed=idx)
            _same(got, want[r.astype(np.int64)], cfg, "sample")
            assert np.array_equal(engine.group_sizes(ranks), ref.sizes[ranks]), (cfg.tag, "sizes")
        _check_shares(shares[:cfg.nparts], cfg, st, ref, rs)
    finally:
        _reset(engine)


def _check_shares(engs, cfg, st, ref, rs):
    P, want, t = len(engs), ref.recs, ref.total
    counts = []
    try:
        for q, eng in enumerate(engs):
            _apply(eng, cfg, st)
            mine = ref.share(q, P)
            k = min(len(mine), int(rs.randint(0, 200)))
            e = eng.enumerate7_chain(*cfg.orders, k, True, q, P)
            assert e.total == len(mine), (cfg.tag, "share", q, P, e.total, len(mine))
            _same(e.matches, mine[:k], cfg, "share %d/%d first %d" % (q, P, k))
            f = eng.enumerate7_chain(*cfg.orders, k, False, q, P)
            _same(f.matches, mine[:k], cfg, "share %d/%d count-free" % (q, P))
            eng.enumerate7_chain(*cfg.orders, 0, True, q, P)
            sums = eng.enum_block_sums()
            assert sums.tobytes() == ref.share_sums(q, P).tobytes(), (cfg.tag, "block sums", q, P)
            counts.append(len(sums))
        sums = np.zeros((P, max(max(counts), 1)), dtype=np.uint64)
        for q in range(P):
            sums[q, :counts[q]] = ref.share_sums(q, P)
        assert [eng.enum_set_global(sums, counts) for eng in engs] == [t] * P, (cfg.tag, "global")
        for first in sorted({0, t // 3, max(t - 40, 0)}):
            got = sum(eng.fetch_matches(first, 80).view(np.uint64) for eng in engs)
            _same(got.view(sb.MATCH_DTYPE).reshape(-1), want[first:first + 80], cfg,
                  "global page %d" % first)
        if t:
            ranks = rs.randint(0, t, int(rs.randint(1, 200)))
            got = sum(eng.pick_matches(ranks).view(np.uint64) for eng in engs)
            _same(got.view(sb.MATCH_DTYPE).reshape(-1), want[ranks], cfg, "global pick")
    finally:
        for eng in engs:
            _reset(eng)


# ------------------------------------------------------------------------------------------------
# Closed forms under the empty mask: every combination is feasible, every candidate matches.

def test_empty_mask_closed_forms(engine):
    n, inbits = 16, [1, 5]
    engine.load(bench._state(n, 1000 + n), bench._rijndael_bit(0), np.zeros(4, dtype=np.uint64),
                inbits)
    st = bench.build_batch(40, 4, 1)[0]
    c = comb(n - len(inbits), 7)
    try:
        for grouping, want in ((None, c * PER_COMB), ("shape", c * 210), ("tuple", c)):
            engine.set_grouping(grouping)
            e = engine.enumerate7_chain(st["outer"], st["middle"], 8)
            assert (e.total, e.feasible) == (want, c), grouping
            assert all(int(r["shape"]) == 1 and not set(int(g) for g in r["gates"]) & set(inbits)
                       for r in e.matches)
        engine.set_grouping("tuple")
        e = engine.enumerate7_chain(st["outer"], st["middle"], 0)
        sizes = engine.group_sizes(np.array([0, e.total - 1]))
        assert list(sizes) == [PER_COMB, PER_COMB]
        engine.set_grouping("shape")
        e = engine.enumerate7_chain(st["outer"], st["middle"], 0)
        assert list(engine.group_sizes(np.array([0, e.total // 2]))) == [65536, 65536]
    finally:
        engine.set_grouping(None)


# ------------------------------------------------------------------------------------------------
# Against sbg_enum5: with L2 = 0xF0 (the projection onto x1) the chain is the 5-LUT L3(L1(a,b,c),
# f, g), once for each allowed pair {d, e} outside the combination.

def test_projection_middle_matches_the_5lut_enumeration(engine):
    rs = np.random.RandomState(31)
    n, inbits = 11, [2]
    tabs = S.synthetic_state(n, seed=77)
    g5 = [0, 3, 6, 8, 10]
    tgt = S.lut_table(0xB4, S.lut_table(0x69, tabs[0], tabs[3], tabs[6]), tabs[8], tabs[10])
    mask = _random_mask(rs, 40)
    outer = bytes(rs.permutation(256).astype(np.uint8))
    middle = bytes(rs.permutation(256).astype(np.uint8))
    engine.load(tabs, tgt, mask, inbits)
    e5 = engine.enumerate5(outer, 1 << 20)
    assert e5.total < 1 << 20
    want = collections.Counter()
    for r in e5.matches:
        # a 5-LUT record is (a, b, c) = its outer gates ascending, then its two others ascending,
        # with inner cells x<<2 | y<<1 | z: the chain's (x2, f, g) when x2 = x1
        g = [int(x) for x in r["gates"][:5]]
        for d in range(n):
            for e in range(d + 1, n):
                if d in g or e in g or d in inbits or e in inbits:
                    continue
                want[(tuple(g[:3]), (d, e), (g[3], g[4]), int(r["func_outer"]),
                      int(r["func_inner"]), int(r["inner_seen"]))] += 1
    engine.set_function_filter(None, [0xF0], None)
    try:
        ec = engine.enumerate7_chain(outer, middle, 1 << 20)
    finally:
        engine.clear_function_filter()
    assert ec.total < 1 << 20
    got = collections.Counter()
    for r in ec.matches:
        g = [int(x) for x in r["gates"]]
        got[(tuple(g[:3]), (g[3], g[4]), (g[5], g[6]), int(r["func_outer"]),
             int(r["func_inner"]), int(r["inner_seen"]))] += 1
    assert got == want
    assert any(k[0] == (0, 3, 6) and k[2] == (8, 10) for k in got)


# ------------------------------------------------------------------------------------------------
# What the feature is for: a chain on late gates, found as the shallowest chain realisation.

def test_planted_chain_on_late_gates(engine):
    rs = np.random.RandomState(8)
    n = 40
    tables = bench._state(n, 4000)
    late = list(range(n - 7, n))
    target = S.lut_table(0xCA, S.lut_table(0xE8, S.lut_table(0x96, *tables[late[:3]]),
                                           tables[late[3]], tables[late[4]]),
                         tables[late[5]], tables[late[6]])
    mask = _random_mask(rs, 28)
    depth = np.full(n, 4, dtype=np.uint16)
    depth[late] = 0   # the planted chain has depth 3; anything with another gate at least 5
    outer, middle = (bytes(rs.permutation(256).astype(np.uint8)) for _ in range(2))
    try:
        engine.load(tables, target, mask, [])
        d, total, recs = sb.shallowest_matches(engine, 7, (outer, middle), depth, 64, shape="chain")
        assert d == 3 and total >= 1
        assert all(sorted(int(g) for g in r["gates"]) == late for r in recs)
        # the planted one itself: the last combination, row 0, L1 = 0x96, L2 = 0xE8
        planted = ((comb(n, 7) - 1) << 24) | (outer.index(0x96) << 8) | middle.index(0xE8)
        engine.set_function_filter([0x96], [0xE8], None)
        e = engine.enumerate7_chain(outer, middle, 1 << 16)
        engine.clear_function_filter()
        assert planted in set(int(k) for k in e.matches["key"])
        for r in recs:
            luts = sb.chain_luts(r, lut.allowed_fill(r["func_inner"], r["inner_seen"]))
            assert CR.rebuild_ok(r, tables, target, mask, luts[2][0])
            with pytest.raises(ValueError):
                sb.match_to_ret(r, sb.Xorshift1024(bytes(128)))
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
    c = engine.enumerate7_chain(outer, middle, 1000)
    assert c.feasible > 0 and all(int(r["shape"]) == 1 for r in c.matches)
    e2 = engine.enumerate7(outer, middle, 1000)
    engine.enumerate7_chain(outer, middle, 10, count=False)
    r2 = engine.search7(outer, middle)
    assert r1.found and result_fields(r1, 7) == result_fields(r2, 7)
    assert (e1.total, e1.feasible, e1.matches.tobytes()) == \
        (e2.total, e2.feasible, e2.matches.tobytes())
    assert all(int(r["shape"]) == 0 for r in e2.matches)


def test_bad_arguments(engine):
    lib = native.load_library()
    n_out, total, feas = C.c_uint64(), C.c_uint64(), C.c_uint64()
    out = np.zeros(4, dtype=sb.MATCH_DTYPE)
    order = (C.c_uint8 * 256)(*range(256))
    bad = (C.c_uint8 * 256)(*([0] + list(range(255))))

    def call(eng, o=order):
        return lib.sbg_enum7_chain(eng._h, 0, 1, o, order, 4,
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
    assert call(engine, bad) == SBG_ERR_ARG
    try:
        engine.set_depth_filter(np.zeros(11, dtype=np.uint16), 5)
        assert call(engine) == SBG_ERR_ARG
    finally:
        engine.clear_depth_filter()
    assert call(engine) == 0
