"""GPU: sbg_enum3 (every match of lut_search's 3-LUT scan) against the CPU oracle's
orc_enum3_range (tests/enum3_oracle.c, checked against a plain count by test_enum3_cpu.py), against
the scan of sbg_search_node, across shards and count-free windows, next to the 7-LUT calls on one
slot, and enumerate_lut_search against lut_search."""
import os
import re

import numpy as np
import pytest

import _enum3_support as E3
import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native
from sboxgates_b200.rng import Xorshift1024

pytestmark = pytest.mark.gpu

NONE = E.NONE
K = 400
MUX = [[], [(3, 1)], [(0, 0), (5, 1)], [(1, 1), (4, 0), (6, 1)]]
SBG_ERR_ARG, SBG_ERR_STATE = -1, -4


def _mask(spec, seed):
    """"m<depth>" = mux mask; int = random mask of that many positions (0 - 3: degenerate; 33,
    65, 129, 200: the last 32-bit word of the compressed tables partly padding)."""
    if isinstance(spec, str):
        return S.mux_mask(MUX[int(spec[1:])])
    rs = np.random.RandomState(seed)
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, spec, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def _target(kind, tabs, rs, i):
    n = len(tabs)
    if kind == 0:     # a 3-LUT of three gates
        g = [int(x) for x in rs.choice(n, 3, replace=False)]
        return S.lut_table(int(rs.randint(1, 255)), *[tabs[x] for x in g])
    if kind == 1:     # a 5-input composition
        g = [int(x) for x in rs.choice(n, 5, replace=False)]
        return S.lut_table(int(rs.randint(1, 255)), S.lut_table(int(rs.randint(1, 255)),
                           *[tabs[x] for x in g[:3]]), tabs[g[3]], tabs[g[4]])
    return S.sbox_target(S.rijndael_sbox(), i % 8)


# (n, mask spec)
CASES = [(12, "m0"), (12, "m3"), (16, "m1"), (16, 33), (20, "m2"), (20, 65), (24, 129), (24, 200),
         (31, "m0"), (32, "m3"), (33, 100), (40, "m1"), (47, 65), (48, "m2"), (63, 200), (64, "m0"),
         (64, 33), (12, 0), (16, 1), (20, 2), (24, 3), (64, 0), (40, 3)]


def _states():
    out = []
    for i, (n, spec) in enumerate(CASES):
        rs = np.random.RandomState(17000 + i)
        tabs = S.synthetic_state(n, seed=17100 + i)
        tgt = _target(i % 3, tabs, rs, i)
        order = [int(x) for x in rs.permutation(n)]
        out.append((tabs, tgt, _mask(spec, 17200 + i), order))
    return out


def _keys(e):
    return [int(k) for k in e.matches["key"]]


def _positions(mask):
    return sum(bin(int(w)).count("1") for w in mask)


def _check_records(e, tabs, tgt, mask, order, limit=80):
    for rec in e.matches[:limit]:
        i, k, m = sb.decode_key3(rec["key"])
        gates = [order[i], order[k], order[m]]
        assert int(rec["width"]) == 3 and [int(g) for g in rec["gates"]] == gates + [0] * 4
        assert int(rec["func_outer"]) == int(rec["func_middle"]) == 0
        assert not rec["pad"].any()
        ok, fi, seen = sb.solve_inner(*[tabs[g] for g in gates], tgt, mask)
        assert ok and (int(rec["func_inner"]), int(rec["inner_seen"])) == (fi, seen), hex(int(rec["key"]))
        got = sb.lut_table(int(rec["func_inner"]), *[tabs[g] for g in gates])
        assert np.array_equal(got & mask, tgt & mask)


def test_enum3_matches_oracle(engine):
    matched = 0
    for i, (tabs, tgt, mask, order) in enumerate(_states()):
        n = len(tabs)
        total, keys = E3.enum3_range(tabs, tgt, mask, order, K)
        if _positions(mask) == 0:
            assert total == n * (n - 1) * (n - 2) // 6, i
        e = sb.enumerate_3lut(engine, tabs, tgt, mask, [0], order, K)
        assert (e.total, e.feasible) == (total, total), (i, e.total, total)
        assert _keys(e) == keys, i
        _check_records(e, tabs, tgt, mask, order)
        for k in (1, 7, K):
            f = engine.enumerate3(order, k, count=False)
            assert f.total is None and _keys(f) == keys[:k], (i, k)
            assert np.array_equal(f.matches, e.matches[:k]), (i, k)
        matched += total > 0
    assert matched >= 15


C_CASES = [(255, 200), (256, "m1"), (257, 129), (500, 255)]


def test_enum3_at_large_n(engine):
    """A planted triple at the last positions of the gate order (key fields >= 256 from n = 257 on)
    and a target no triple realises, against orc_enum3_range in pieces.  C(500,3) = 20.7 M
    triples."""
    for i, (n, spec) in enumerate(C_CASES):
        rs = np.random.RandomState(18200 + i)
        tabs = np.concatenate([S.synthetic_state(n - 3, seed=18000 + i),
                               rs.randint(0, 2**63, (3, 4)).astype(np.uint64) * np.uint64(2)
                               + rs.randint(0, 2, (3, 4)).astype(np.uint64)])
        mask = _mask(spec, 18100 + i)
        order = [int(x) for x in rs.permutation(n - 3)] + [int(x) for x in rs.permutation(3) + n - 3]
        planted = S.lut_table(0x6B ^ i, tabs[n - 3], tabs[n - 2], tabs[n - 1])
        for tgt in (planted, S.sbox_target(S.rijndael_sbox(), i % 8)):
            total, keys = E3.enum3_range(tabs, tgt, mask, order, K)
            e = sb.enumerate_3lut(engine, tabs, tgt, mask, [], order, K)
            assert (e.total, e.feasible) == (total, total) and _keys(e) == keys, (n, spec)
            _check_records(e, tabs, tgt, mask, order)
            f = engine.enumerate3(order, 1, count=False)
            assert _keys(f) == keys[:1], (n, spec)
            if tgt is planted:
                assert total >= 1 and keys[-1] == (n - 3) << 18 | (n - 2) << 9 | (n - 1), (n, spec)
            else:
                assert total == 0, (n, spec)


def test_first_match_is_the_scan(engine):
    checked = none = 0
    for tabs, tgt, mask, order in _states():
        for e in (sb.enumerate_3lut(engine, tabs, tgt, mask, [], order, 1),
                  engine.enumerate3(order, 1, count=False)):
            node = engine.search_node(0, gate_order=order)
            if not e.matches.size:
                assert e.total in (0, None) and int(node.key3) == native.SBG_KEY_NONE
                assert node.found_stage == 0
                none += 1
                continue
            rec = e.matches[0]
            assert int(node.key3) == int(rec["key"]) and node.found_stage == 3
            assert list(node.gates3) == [int(g) for g in rec["gates"][:3]]
            assert (node.func3, node.seen3) == (int(rec["func_inner"]), int(rec["inner_seen"]))
            checked += 1
    assert checked >= 20 and none >= 2


def test_shards_add_up(engine):
    """Target = one gate's table: every triple that holds that gate matches (C(n-1,2) and more),
    so the matches reach every part."""
    for i, (n, positions) in enumerate([(40, 10), (64, 24), (96, 16)]):
        rs = np.random.RandomState(18500 + i)
        tabs = S.synthetic_state(n, seed=18600 + i)
        tgt = tabs[int(rs.randint(8, n))].copy()
        mask = _mask(positions, 18700 + i)
        order = [int(x) for x in rs.permutation(n)]
        idx = (n, positions)
        engine.load(tabs, tgt, mask, [])
        whole = engine.enumerate3(order, K)
        assert whole.total > K, idx
        for nparts in (2, 3, 7):
            parts = [engine.enumerate3(order, K, part=p, nparts=nparts) for p in range(nparts)]
            assert sum(p.total for p in parts) == whole.total, (idx, nparts)
            assert sum(p.feasible for p in parts) == whole.feasible, (idx, nparts)
            merged = np.sort(np.concatenate([p.matches for p in parts]), order="key")[:K]
            assert np.array_equal(merged, whole.matches), (idx, nparts)
            free = [engine.enumerate3(order, K, count=False, part=p, nparts=nparts)
                    for p in range(nparts)]
            for p, f in zip(parts, free):
                assert np.array_equal(f.matches, p.matches), (idx, nparts)


def _window3():
    """Pair tickets in the first count-free window (kEnumWindow3, doubling in run_enum), read from
    the library's source."""
    csrc = os.path.join(S.ROOT, "sboxgates_b200", "csrc")
    api = open(os.path.join(csrc, "sbg_api.cu")).read()
    dev = open(os.path.join(csrc, "sbg_device.cuh")).read()

    def find(pattern, text, where):
        m = re.search(pattern, text)
        assert m is not None, "cannot read %r from %s: update _window3" % (pattern, where)
        return m.group(1)
    threads = int(find(r"constexpr int kThreads = (\d+);", dev, "sbg_device.cuh"))
    factors = find(r"kNominalWarps = ([\d\s*]+)\* kWarpsPerCta;", api, "sbg_api.cu")
    warps = int(np.prod([int(x) for x in factors.split("*") if x.strip()])) * (threads // 32)
    return warps // int(find(r"kEnumWindow3 = kNominalWarps(?: / (\d+))?;()", api, "sbg_api.cu") or 1)


def _pair_ticket(n, key):
    i, k, _ = sb.decode_key3(key)
    return i * (2 * n - i - 1) // 2 + (k - i - 1)


def test_count_free_windows(engine):
    """The K-th match past the end of the second count-free window (tickets = position pairs in
    lexicographic order), K = 0, K = total and K = total + 1, counted and count-free, against the
    oracle."""
    w = _window3()
    n = 160
    assert n * (n - 1) // 2 > 4 * w
    rs = np.random.RandomState(19000)
    tabs = S.synthetic_state(n, seed=19001)
    mask = _mask(14, 19002)
    tgt = S.sbox_target(S.rijndael_sbox(), 5)
    order = [int(x) for x in rs.permutation(n)]
    engine.load(tabs, tgt, mask, [])
    total = engine.enumerate3(order, 0).total
    assert 0 < total <= 10**6
    every = engine.enumerate3(order, total)
    assert every.total == total and len(every.matches) == total
    want_total, want_keys = E3.enum3_range(tabs, tgt, mask, order, 3000)
    assert total == want_total and _keys(every)[:3000] == want_keys
    tickets = np.array([_pair_ticket(n, k) for k in _keys(every)])
    assert np.all(np.diff(tickets) >= 0)
    before = int(np.sum(tickets < 3 * w))      # matches in the first two windows
    assert 0 < before < total - 10
    for k in (0, 1, before, before + 1, before + 7, total - 1, total, total + 1):
        f = engine.enumerate3(order, k, count=False)
        assert np.array_equal(f.matches, every.matches[:k]), k
        c = engine.enumerate3(order, k)
        assert c.total == total and np.array_equal(c.matches, every.matches[:k]), k
    _check_records(every, tabs, tgt, mask, order, limit=40)
    for rec in every.matches[before:before + 40]:
        i, k, m = sb.decode_key3(rec["key"])
        assert S.oracle_check(3, tgt, mask, [tabs[order[i]], tabs[order[k]], tabs[order[m]]])


def test_bad_arguments(engine):
    lib = native.load_library()
    n_out, total, feas = native.C.c_uint64(), native.C.c_uint64(), native.C.c_uint64()
    out = np.zeros(4, dtype=sb.MATCH_DTYPE)

    def call(eng, order, k=4, part=0, nparts=1):
        go = (native.C.c_uint16 * max(1, len(order)))(*order)
        return lib.sbg_enum3(eng._h, part, nparts, go, k, out.ctypes.data_as(native.C.c_void_p),
                             native.C.byref(n_out), native.C.byref(total), native.C.byref(feas))
    fresh = sb.LutEngine(0)
    try:
        assert call(fresh, [0, 1, 2]) == SBG_ERR_STATE
    finally:
        fresh.close()
    tabs = S.synthetic_state(12, seed=5)
    tgt = S.lut_table(0x96, tabs[2], tabs[7], tabs[9])
    engine.load(tabs, tgt, S.mux_mask([]), [])
    good = list(range(12))
    assert call(engine, good) == 0 and total.value >= 1
    assert call(engine, good[:11] + [11 + 1]) == SBG_ERR_ARG       # gate out of range
    assert call(engine, good[:11] + [3]) == SBG_ERR_ARG            # repeated gate
    assert call(engine, good, k=native.SBG_ENUM_MAX_MATCHES + 1) == SBG_ERR_ARG
    assert call(engine, good, part=3, nparts=3) == SBG_ERR_ARG
    engine.load(tabs[:2], tgt, S.mux_mask([]), [])
    assert call(engine, [0, 1]) == SBG_ERR_ARG                      # n < 3
    with pytest.raises(ValueError):
        sb.enumerate_3lut(engine, tabs[:2], tgt, S.mux_mask([]), [], [0, 1], 4)


def _summary(e):
    return None if e is None else (e.total, e.feasible, e.matches.tobytes())


def test_interleaved_calls_on_one_slot(engine):
    """enum3, search7, enum7, enum3 on one slot (and search7, enum3, enum7): each call gives what it
    gives alone on a fresh handle; sbg_enum3 leaves the installed 7-LUT list alone."""
    rs = np.random.RandomState(19500)
    tabs = S.synthetic_state(14, seed=19501)
    g = [int(x) for x in rs.choice(range(1, 14), 7, replace=False)]
    tgt = S.lut_table(0xE8, S.lut_table(0x96, *[tabs[x] for x in g[:3]]),
                      S.lut_table(0x6B, *[tabs[x] for x in g[3:6]]), tabs[g[6]])
    mask, inb = _mask(16, 19502), [0, 5]
    order = [int(x) for x in rs.permutation(14)]
    _, outer, middle = E.orders(19)
    fields = ("found", "key", "func_outer", "func_middle", "func_inner", "inner_seen",
              "tuples_feasible")
    alone = {}
    for what in ("e3", "s7", "e7"):
        fresh = sb.LutEngine(0)
        try:
            fresh.load(tabs, tgt, mask, inb)
            if what == "e3":
                alone[what] = _summary(fresh.enumerate3(order, K))
            elif what == "s7":
                r = fresh.search7(outer, middle)
                alone[what] = [getattr(r, f) for f in fields] + list(r.gates)
            else:
                alone[what] = _summary(fresh.enumerate7(outer, middle, K))
        finally:
            fresh.close()
    assert alone["e7"][0] > 0 and alone["e3"][0] > 0
    for seq in (("e3", "s7", "e7", "e3"), ("s7", "e3", "e7", "e3", "s7")):
        engine.load(tabs, tgt, mask, inb)
        for what in seq:
            if what == "e3":
                got = _summary(engine.enumerate3(order, K))
            elif what == "s7":
                r = engine.search7(outer, middle)
                got = [getattr(r, f) for f in fields] + list(r.gates)
            else:
                got = _summary(engine.enumerate7(outer, middle, K))
            assert got == alone[what], (seq, what)


def _node_cases():
    """States of lut_search nodes that end at stage 3, 5, 7 and 0; gate 0 is always an excluded
    input bit, so that the first 7-LUT match is sbg_search7's result (no stale outer cache)."""
    rs = np.random.RandomState(20000)
    for i in range(40):
        n = int(rs.choice([11, 12, 13]))
        tabs = S.synthetic_state(n, seed=int(rs.randint(1 << 30)))
        fixed = [(int(b), int(rs.randint(0, 2))) for b in rs.choice(range(1, 8), int(rs.randint(0, 3)),
                                                                    replace=False)]
        mask = S.mux_mask(fixed)
        inb = sorted({0} | {b for b, _ in fixed})
        kind = i % 4
        allowed = [x for x in range(n) if x not in inb]
        if kind == 0:
            g = [int(x) for x in rs.choice(n, 3, replace=False)]
            tgt = S.lut_table(int(rs.randint(1, 255)), *[tabs[x] for x in g])
        elif kind == 1:
            g = [int(x) for x in rs.choice(allowed, 5, replace=False)]
            tgt = S.lut_table(int(rs.randint(1, 255)), S.lut_table(int(rs.randint(1, 255)),
                              *[tabs[x] for x in g[:3]]), tabs[g[3]], tabs[g[4]])
        elif kind == 2:
            g = [int(x) for x in rs.choice(allowed, 7, replace=False)]
            tgt = S.lut_table(int(rs.randint(1, 255)),
                              S.lut_table(int(rs.randint(1, 255)), *[tabs[x] for x in g[:3]]),
                              S.lut_table(int(rs.randint(1, 255)), *[tabs[x] for x in g[3:6]]),
                              tabs[g[6]])
        else:
            tgt = S.sbox_target(S.rijndael_sbox(), int(rs.randint(0, 8)))
        order = [int(x) for x in rs.permutation(n)]
        yield tabs, tgt, mask, inb, order, rs.bytes(128)


def test_enumerate_lut_search_reproduces_lut_search(engine):
    stages = {0: 0, 3: 0, 5: 0, 7: 0}
    for tabs, tgt, mask, inb, order, seed in _node_cases():
        rng = Xorshift1024(seed)
        before = (list(rng.s), rng.p, rng.draws)
        en = sb.enumerate_lut_search(engine, tabs, tgt, mask, inb, order, rng, 4)
        assert (list(rng.s), rng.p, rng.draws) == before
        got = sb.lut_search(engine, tabs, tgt, mask, inb, order, Xorshift1024(seed))
        fill = Xorshift1024(seed)
        stage, luts = 0, []
        if en[3].total > 0:
            stage, luts = 3, [sb.match_to_lut3(en[3].matches[0], fill)]
        elif en[5] is not None and en[5].total > 0:
            for _ in range(256):
                fill.next()
            r = sb.match_to_ret(en[5].matches[0], fill)
            stage, luts = 5, [(r[0], r[2], r[3], r[4]), (r[1], ("new", 0), r[5], r[6])]
        elif en[7] is not None and en[7].total > 0:
            for _ in range(256 + 512):
                fill.next()
            r = sb.match_to_ret(en[7].matches[0], fill)
            stage, luts = 7, [(r[1], r[6], r[7], r[8]), (r[0], r[3], r[4], r[5]),
                              (r[2], ("new", 1), ("new", 0), r[9])]
        assert (got.stage, got.luts) == (stage, luts), (got.stage, stage)
        stages[stage] += 1
        # the counts of the stages a node does not reach are still there
        for w, e in en.items():
            assert e is None or len(e.matches) == min(e.total, 4)
    assert min(stages.values()) >= 2, stages


def test_enumerate_lut_search_gating(engine):
    tabs = S.synthetic_state(9, seed=77)
    tgt = S.sbox_target(S.rijndael_sbox(), 1)
    mask, order = S.mux_mask(MUX[1]), list(range(9))
    rng = Xorshift1024(bytes(range(128)))
    full = sb.enumerate_lut_search(engine, tabs, tgt, mask, [0], order, rng, 2)
    assert all(full[w] is not None for w in (3, 5, 7))
    no7 = sb.enumerate_lut_search(engine, tabs, tgt, mask, [0], order, rng, 2, allow7=False)
    assert no7[7] is None and _summary(no7[5]) == _summary(full[5])
    no5 = sb.enumerate_lut_search(engine, tabs, tgt, mask, [0], order, rng, 2, allow5=False)
    assert no5[5] is None and no5[7] is None and _summary(no5[3]) == _summary(full[3])
    small = sb.enumerate_lut_search(engine, tabs[:6], tgt, mask, [0], [5, 2, 0, 4, 1, 3], rng, 2)
    assert small[3] is not None and small[5] is not None and small[7] is None
    tiny = sb.enumerate_lut_search(engine, tabs[:4], tgt, mask, [0], [3, 1, 0, 2], rng, 2)
    assert tiny[3] is not None and tiny[5] is None and tiny[7] is None
    assert rng.draws == 0
