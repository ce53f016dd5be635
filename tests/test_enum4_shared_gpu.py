"""GPU: the shared-input two-LUT circuits L2(L1(a,b,c), u, v), {u, v} = {s, d} with s one of a, b, c
(sbg_enum4_shared, sbg_search4_shared) and the opt-in stage of lut_search and of the drop-in
(SBG_LUT_SHARED=1), against the CPU oracle (tests/enum_shared_oracle.c).

- Seeded states at every table width (NW = 1, 2, 4, 8) in every kernel form (plain, filtered,
  grouped by shape and by tuple), with and without excluded input bits: totals, feasible counts,
  the first K, the count-free first K, pages, picks, group sizes and depth counts, and sharded
  cursors with global ranks; sbg_search4_shared equals the first match.
- n = 128 and n = 500 with a circuit planted late in the order; the empty mask's closed form.
- A record whose L2 ignores the shared gate is an sbg_enum5 match once a fifth gate is added.
- The installed 7-LUT list is left alone; bad arguments are refused.
- The 192 recorded search_5lut calls that found nothing; lut_search(shared=True) against
  shared=False on the recorded nodes; the drop-in on des_s1 under both seeds."""
import ctypes as C
import json
import os
import re
import subprocess
import tempfile
from math import comb

import numpy as np
import pytest

import _enum_shared_reference as R
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import lut, native
from test_dropin_gpu import _run, _verify
from test_enum_depth_gpu import _nw
from test_enum_fuzz_gpu import MUX, RANDOM_POSITIONS, _random_mask

pytestmark = pytest.mark.gpu

SBG_ERR_ARG, SBG_ERR_STATE = -1, -4
NWS = (1, 2, 4, 8)
FORMS = ("plain", "filtered", "shape", "tuple")
FULL = np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)


def _planted(rs, tabs, gates):
    """A target realised by L2(L1(a,b,c), s, d) on four gates, s one of a, b, c."""
    a, b, c, d = gates
    f1, f2 = (int(x) for x in rs.randint(1, 255, 2))
    x1 = S.lut_table(f1, tabs[a], tabs[b], tabs[c])
    return S.lut_table(f2, x1, tabs[(a, b, c)[int(rs.randint(3))]], tabs[d])


class Case:
    def __init__(self, idx):
        rs = self.rs = np.random.RandomState([77, idx])
        self.idx = idx
        self.nw, self.form = NWS[idx % 4], FORMS[(idx // 4) % 4]
        self.n = n = int(rs.randint(8, 15))
        if rs.rand() < 0.4:
            self.mask = S.mux_mask(MUX[self.nw])
        else:
            lo, hi = RANDOM_POSITIONS[self.nw][int(rs.randint(2))]
            self.mask = _random_mask(rs, int(rs.randint(lo, hi + 1)))
        assert _nw(self.mask) == self.nw
        self.inbits = sorted(int(x) for x in rs.choice(8, int(rs.randint(0, 3)), replace=False))
        self.tables = S.synthetic_state(n, seed=int(rs.randint(1 << 30)))
        allowed = [g for g in range(n) if g not in self.inbits]
        gates = [int(x) for x in rs.choice(allowed, 4, replace=False)]
        self.target = _planted(rs, self.tables, gates)
        self.order = bytes(rs.permutation(256).astype(np.uint8))
        self.depth = rs.randint(0, 6, n).astype(np.uint16)
        self.tag = "case %d: n %d NW %d inbits %s form %s" % (idx, n, self.nw, self.inbits,
                                                             self.form)


def _filtered(case, recs, st):
    """The reference records under the case's settings: (records, depth histogram, group sizes)."""
    ok = np.ones(len(recs), dtype=bool)
    if st.get("bound") is not None:
        ok &= R.shared_depths(recs, case.depth) <= st["bound"]
    if st.get("outer") is not None or st.get("inner") is not None:
        ok &= np.array([sb.match_functions_allowed(r, st.get("outer"), None, st.get("inner"))
                        for r in recs], dtype=bool)
    recs = recs[ok]
    shift = {"shape": 8, "tuple": 12}.get(case.form)
    sizes = np.ones(len(recs), dtype=np.uint64)
    if shift is not None and len(recs):
        ids = recs["key"] >> np.uint64(shift)
        first = np.concatenate([[True], ids[1:] != ids[:-1]])
        sizes = np.diff(np.append(np.flatnonzero(first), len(recs))).astype(np.uint64)
        recs = recs[first]
    return recs, sizes


def _settings(case, recs):
    rs, st = case.rs, {}
    if case.form == "plain":
        return st
    if len(recs):
        dep = R.shared_depths(recs, case.depth)
        st["bound"] = int(rs.randint(dep.min(), dep.max() + 1))
    if rs.rand() < 0.6:
        st["outer"] = sorted(int(x) for x in rs.choice(256, 160, replace=False))
    if rs.rand() < 0.4:
        st["inner"] = sorted(sb.AFFINE_FUNCTIONS)
    return st


def _apply(eng, case, st):
    if st.get("bound") is not None:
        eng.set_depth_filter(case.depth, st["bound"])
    if st.get("outer") is not None or st.get("inner") is not None:
        eng.set_function_filter(outer=st.get("outer"), inner=st.get("inner"))
    if case.form in ("shape", "tuple"):
        eng.set_grouping(case.form)


def _reset(eng):
    eng.clear_depth_filter()
    eng.clear_function_filter()
    eng.set_grouping(None)


def _same(got, want, tag):
    assert got.tobytes() == want.tobytes(), (tag, got[:3], want[:3])


@pytest.fixture(scope="module")
def shares():
    engs = [sb.LutEngine(0) for _ in range(3)]
    yield engs
    for e in engs:
        e.close()


@pytest.mark.parametrize("idx", range(16))
def test_states_match_the_oracle(engine, shares, idx):
    case = Case(idx)
    feas, allrecs = R.shared_reference(case.tables, case.target, case.mask, case.inbits, case.order)
    assert len(allrecs) > 0, case.tag
    st = _settings(case, allrecs)
    want, sizes = _filtered(case, allrecs, st)
    t = len(want)
    engine.load(case.tables, case.target, case.mask, case.inbits)
    # the search ignores the settings and returns the unfiltered first match
    _apply(engine, case, st)
    res = engine.search4_shared(case.order)
    assert res.found and res.key == int(allrecs[0]["key"]), case.tag
    assert (res.index, res.ordering, res.pos_outer) == sb.decode_key5(res.key)
    assert list(res.gates[:5]) == list(allrecs[0]["gates"][:5])
    assert (res.func_outer, res.func_inner, res.inner_seen) == (
        allrecs[0]["func_outer"], allrecs[0]["func_inner"], allrecs[0]["inner_seen"])
    assert res.tuples_feasible <= feas and res.index < res.tuples_swept <= comb(case.n, 4)
    try:
        _apply(engine, case, st)
        k = min(t, int(case.rs.randint(1, 300)))
        e = engine.enumerate4_shared(case.order, k)
        assert e.total == t, (case.tag, e.total, t)
        if st.get("bound") is None:
            assert e.feasible == feas, case.tag
        _same(e.matches, want[:k], case.tag + " first K")
        f = engine.enumerate4_shared(case.order, k, count=False)
        _same(f.matches, want[:k], case.tag + " count-free")
        engine.enumerate4_shared(case.order, 0)
        for first in sorted({0, t // 2, max(t - 30, 0)}):
            _same(engine.fetch_matches(first, 60), want[first:first + 60], case.tag + " page")
        ranks = case.rs.randint(0, t, 100) if t else np.zeros(0, dtype=np.int64)
        _same(engine.pick_matches(ranks), want[ranks], case.tag + " pick")
        assert engine.group_sizes(ranks).tolist() == sizes[ranks].tolist(), case.tag
        if st.get("bound") is not None:
            hist = engine.depth_counts()
            d = R.shared_depths(want, case.depth)
            assert hist.tolist() == np.bincount(d, minlength=len(hist)).tolist()[:len(hist)]
        # shares with global ranks
        P = len(shares)
        counts, rows = [], []
        for q, eng in enumerate(shares):
            eng.load(case.tables, case.target, case.mask, case.inbits)
            _apply(eng, case, st)
            eng.enumerate4_shared(case.order, 0, True, q, P)
            rows.append(eng.enum_block_sums())
            counts.append(len(rows[-1]))
        sums = np.zeros((P, max(max(counts), 1)), dtype=np.uint64)
        for q in range(P):
            sums[q, :counts[q]] = rows[q]
        assert [eng.enum_set_global(sums, counts) for eng in shares] == [t] * P, case.tag
        got = sum(eng.fetch_matches(0, 200).view(np.uint64) for eng in shares)
        _same(got.view(sb.MATCH_DTYPE).reshape(-1), want[:200], case.tag + " global page")
        got = sum(eng.pick_matches(ranks).view(np.uint64) for eng in shares)
        _same(got.view(sb.MATCH_DTYPE).reshape(-1), want[ranks], case.tag + " global pick")
    finally:
        _reset(engine)
        for eng in shares:
            _reset(eng)


def test_every_record_rebuilds(engine):
    case = Case(3)
    engine.load(case.tables, case.target, case.mask, case.inbits)
    e = engine.enumerate4_shared(case.order, 5000)
    assert e.total > 0
    for rec in e.matches:
        assert rec["width"] == 4 and rec["shape"] == sb.SBG_SHAPE_SHARED
        assert not rec["gates"][5] and not rec["gates"][6] and not rec["func_middle"]
        g = [int(x) for x in rec["gates"][:5]]
        assert len(set(g)) == 4 and g[:3] == sorted(g[:3]) and g[3] < g[4]
        assert R.rebuild_ok(rec["func_outer"], rec["func_inner"], g, case.tables, case.target,
                            case.mask)


@pytest.mark.parametrize("n", [128, 500])
def test_planted_late_circuit_at_large_n(engine, n):
    rs = np.random.RandomState(n)
    tabs = S.synthetic_state(n, seed=n)
    gates = [n - 9, n - 6, n - 3, n - 1]
    tgt = _planted(rs, tabs, gates)
    mask = _random_mask(rs, 200)
    order = bytes(rs.permutation(256).astype(np.uint8))
    engine.load(tabs, tgt, mask, [])
    res = engine.search4_shared(order)
    assert res.found
    assert R.rebuild_ok(res.func_outer, res.func_inner, res.gates[:5], tabs, tgt, mask)
    e = engine.enumerate4_shared(order, 1 << 12)
    assert e.total >= 1 and int(e.matches[0]["key"]) == res.key
    assert res.tuples_feasible == e.feasible or res.tuples_swept < comb(n, 4)
    # the planted combination is among the matches
    r = R.combination_rank(gates, n)
    assert any(int(k) >> 12 == r for k in e.matches["key"]) or e.total > len(e.matches)
    for rec in e.matches[:256]:
        assert R.rebuild_ok(rec["func_outer"], rec["func_inner"], rec["gates"][:5], tabs, tgt, mask)


def test_empty_mask_closed_form(engine):
    zero = np.zeros(4, dtype=np.uint64)
    for n, inbits in ((12, []), (20, [0, 3]), (40, [1])):
        tabs = S.synthetic_state(n, seed=n)
        engine.load(tabs, zero, zero, inbits)
        order = bytes(np.random.RandomState(n).permutation(256).astype(np.uint8))
        e = engine.enumerate4_shared(order, 10)
        feasible = comb(n - len(inbits), 4)
        assert (e.total, e.feasible) == (feasible * 12 * 256, feasible)
        engine.set_grouping("tuple")
        try:
            assert engine.enumerate4_shared(order, 0).total == feasible
            engine.set_grouping("shape")
            assert engine.enumerate4_shared(order, 0).total == feasible * 12
        finally:
            engine.set_grouping(None)


def test_ignored_shared_gate_is_a_5lut_match(engine):
    """A record whose L2 does not read s is a 5-LUT circuit over (a, b, c, d, e) for any fifth
    gate e, so sbg_enum5 has it once e is added.  The target is planted as L2(L1(a,b,c), d)."""
    rs = np.random.RandomState(5)
    n = 12
    tabs = S.synthetic_state(n, seed=5)
    a, b, c, d = 3, 6, 8, 10
    x1 = S.lut_table(0x96, tabs[a], tabs[b], tabs[c])
    tgt = S.lut_table(0x6C, x1, tabs[d], tabs[d])   # L2 = x1 XOR d, ignoring its middle input
    mask = _random_mask(rs, 200)
    order = bytes(rs.permutation(256).astype(np.uint8))
    engine.load(tabs, tgt, mask, [])
    e = engine.enumerate4_shared(order, 1 << 16)
    e5 = engine.enumerate5(order, 1 << 16)
    assert e.total <= len(e.matches) and e5.total <= len(e5.matches)
    keys5 = {(int(k) >> 12, int(k) & 255) for k in e5.matches["key"]}
    checked = 0
    for rec in e.matches:
        g = [int(x) for x in rec["gates"][:5]]
        s_pos = 3 if g[3] in g[:3] else 4
        f2, seen = int(rec["func_inner"]), int(rec["inner_seen"])
        bit = 2 if s_pos == 3 else 1   # L2's cell bit of the shared gate
        if any((seen >> cc) & 1 and (seen >> (cc ^ bit)) & 1
               and ((f2 >> cc) & 1) != ((f2 >> (cc ^ bit)) & 1) for cc in range(8)):
            continue
        other = g[7 - s_pos]
        for spare in (x for x in range(n) if x not in g):
            five = sorted(g[:3] + [other, spare])
            po = int(rec["key"]) & 255
            assert (R.combination_rank(five, n), po) in keys5, (g, five)
            checked += 1
    assert checked > 0


def test_installed_list_is_left_alone(engine):
    case = Case(6)
    engine.load(case.tables, case.target, case.mask, case.inbits)
    outer, middle = (bytes(np.random.RandomState(s).permutation(256).astype(np.uint8))
                     for s in (1, 2))
    r7 = engine.search7(outer, middle)
    launches = engine.launches
    e = engine.enumerate4_shared(case.order, 0)
    engine.search4_shared(case.order)
    e7a = engine.enumerate7(outer, middle, 0)
    assert e.total > 0
    r7b = engine.search7(outer, middle)
    assert (r7b.found, r7b.key, r7b.tuples_swept) == (r7.found, r7.key, r7.tuples_swept)
    assert e7a.feasible == r7.tuples_feasible and engine.launches > launches


def test_bad_arguments(engine):
    case = Case(7)
    lib, h = engine.lib, engine._h
    engine.load(case.tables, case.target, case.mask, [])
    bad = bytes([0] * 256)
    res = native.SbgResult()
    n_out, total, feas = C.c_uint64(), C.c_uint64(), C.c_uint64()
    order = lut._order_ptr(bad)
    assert lib.sbg_enum4_shared(h, 0, 1, order, 0, None, C.byref(n_out), C.byref(total),
                                C.byref(feas)) == SBG_ERR_ARG
    assert lib.sbg_search4_shared(h, order, C.byref(res)) == SBG_ERR_ARG
    assert lib.sbg_enum4_shared(h, 2, 2, lut._order_ptr(case.order), 0, None, C.byref(n_out),
                                C.byref(total), C.byref(feas)) == SBG_ERR_ARG
    engine.load(case.tables[:3], case.target, case.mask, [])
    assert lib.sbg_search4_shared(h, lut._order_ptr(case.order), C.byref(res)) == SBG_ERR_ARG
    fresh = sb.LutEngine(0)
    try:
        assert fresh.lib.sbg_search4_shared(fresh._h, lut._order_ptr(case.order),
                                            C.byref(res)) == SBG_ERR_STATE
        assert fresh.lib.sbg_enum4_shared(fresh._h, 0, 1, lut._order_ptr(case.order), 0, None,
                                          C.byref(n_out), C.byref(total),
                                          C.byref(feas)) == SBG_ERR_STATE
    finally:
        fresh.close()


def test_recorded_unmatched_search5_calls(engine):
    found = 0
    for name, i, rec in R.unmatched_calls():
        total, key, inner, seen, feas = R.oracle_first(rec)
        engine.load(rec.tables, rec.target, rec.mask, rec.inbits_list())
        res = engine.search4_shared(R.call_order(rec))
        assert (bool(res.found), res.key) == (total > 0, key), (name, i)
        if res.found:
            found += 1
            assert (res.func_inner, res.inner_seen) == (inner, seen)
            assert R.rebuild_ok(res.func_outer, res.func_inner, res.gates[:5], rec.tables,
                                rec.target, rec.mask)
            assert res.index < res.tuples_swept <= comb(rec.n, 4)
        else:
            assert (res.tuples_feasible, res.tuples_swept) == (feas, comb(rec.n, 4))
    assert found == 59


def test_lut_search_shared_stage_on_recorded_nodes(engine):
    """Every recorded search_5lut call that found nothing, as a lut_search node: shared=True takes
    the oracle's first match as stage 5 and draws only L2's fill after search_5lut's 256; a node
    without one gets shared=False's result and RNG state, also with chain=True."""
    took = 0
    for name, i, rec in R.unmatched_calls():
        total, key, _, _, _ = R.oracle_first(rec)
        n = rec.n
        order = list(range(n))
        for chain in (False, True):
            rng_a = sb.Xorshift1024.from_state(rec.rng_s, rec.rng_p)
            rng_b = rng_a.copy()
            a = sb.lut_search(engine, rec.tables, rec.target, rec.mask, rec.inbits_list(), order,
                              rng_a, chain=chain, shared=True)
            b = sb.lut_search(engine, rec.tables, rec.target, rec.mask, rec.inbits_list(), order,
                              rng_b, chain=chain)
            if a.shape == "shared":
                assert total > 0 and a.stage == 5 and b.stage != 5
                (f1, x, y, z), (f2, new, u, v) = a.luts
                assert new == ("new", 0)
                assert R.rebuild_ok(f1, f2, [x, y, z, u, v], rec.tables, rec.target, rec.mask)
                took += not chain
            else:
                assert total == 0 or b.stage == 3, (name, i)
                assert (a.stage, a.luts, a.shape) == (b.stage, b.luts, b.shape), (name, i)
                assert rng_a.next() == rng_b.next()
    assert took > 0


# ------------------------------------------------------------------------------------------------
# The drop-in, linked from this tree's node-shim archive (as test_search7_chain_gpu does).

from test_search7_chain_gpu import dropin_exe, needs_objs  # noqa: E402,F401


def _shared_nodes(err):
    m = re.search(r"shared-input pair (\d+)", err)
    assert m, err[-2000:]
    return int(m.group(1))


@needs_objs
@pytest.mark.parametrize("seed", ["seed1", "seed2"])
def test_dropin_shared_stage_on_des_s1(dropin_exe, seed):  # noqa: F811
    with tempfile.TemporaryDirectory() as tmp:
        got, secs, err = _run(dropin_exe, "des_s1.txt", ["-l", "-o", "0"], seed, tmp,
                              extra_env={"SBG_LUT_SHARED": "1"})
        assert got
        graph = _verify(tmp, got[-1], "des_s1.txt", [0])
        assert graph.num_luts == int(got[-1].split("-")[1])
    assert _shared_nodes(err) >= 1 and "shared-input stage:" in err
    with tempfile.TemporaryDirectory() as tmp:
        got2, _, err2 = _run(dropin_exe, "des_s1.txt", ["-l", "-o", "0"], seed, tmp,
                             extra_env={"SBG_LUT_SHARED": "1", "SBG_LUT_CHAIN": "1"})
        assert got2
        _verify(tmp, got2[-1], "des_s1.txt", [0])
    names = json.load(open(os.path.join(S.GOLDEN, "xml_names.json")))
    with tempfile.TemporaryDirectory() as tmp:
        plain, _, err0 = _run(dropin_exe, "des_s1.txt", ["-l", "-o", "0"], seed, tmp)
    assert plain == names["des_s1.txt -l -o 0 %s" % seed]
    assert "shared-input" not in err0
