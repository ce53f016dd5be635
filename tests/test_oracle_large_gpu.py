"""GPU: the searches and enumerations against the CPU oracle at large gate counts and under masks of
any size, where the rest of the suite can only compare the library with itself.

The oracle's rank-range forms (tests/enum_oracle.c, pinned to the whole-space oracle by
test_oracle_range_cpu.py) check slices of spaces too large to walk whole, on a thread pool:
  a. phase-1 lists (n = 64 ... 500): every entry sound, every slice of ranks complete -- across the
     aligned two-word windows (n >= 64), the 5-gate-prefix form (n >= 128), the seam between the
     chunked head and the prefix tickets, gate numbers >= 256;
  b. search_5lut keys on both kernel forms (two kernels / fused, the boundary at n = 52 / 53) and
     in the chunk head (n >= 128);
  c. the 3-LUT scan at positions >= 256 of its 9-bit key fields;
  d. enumerations across several count-free windows, and on a 71,000-entry 7-LUT list;
  e. masks of 0 - 3 positions.
Masks are mux masks of depth 0 - 3 and random masks of 1 - 255 positions, whose last 32-bit word is
partly padding; states run with and without gate 0 among the excluded input bits."""
import os
import re

import numpy as np
import pytest

import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native
from sboxgates_b200.rng import Xorshift1024

pytestmark = pytest.mark.gpu

NONE = E.NONE
CAP = native.SBG_LIST_CAP
MUX = [[], [(3, 1)], [(0, 0), (5, 1)], [(1, 1), (4, 0), (6, 1)]]
ODD = [1, 7, 31, 33, 63, 65, 100, 129, 200, 255]


def _mask(spec, seed):
    """(mask, input bits the mask fixes) of a mask spec: "m<depth>" = mux mask, int = random mask
    of that many positions."""
    if isinstance(spec, str):
        fixed = MUX[int(spec[1:])]
        return S.mux_mask(fixed), [b for b, _ in fixed]
    rs = np.random.RandomState(seed)
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, spec, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask, []


def _inbits(fixed, with0):
    """The excluded input bits: those the mask fixes, with or without gate 0."""
    return sorted(set(fixed) | {0}) if with0 else [b for b in fixed if b != 0]


def _positions(mask):
    return sum(bin(int(w)).count("1") for w in mask)


def _plant(tabs, gates, funcs):
    """Target = funcs[-1](funcs[0](g0, g1, g2), g3, g4) (5 gates) or
    funcs[2](funcs[0](g0, g1, g2), funcs[1](g3, g4, g5), g6) (7 gates) or funcs[0](g0, g1, g2)."""
    g = [tabs[x] for x in gates]
    if len(g) == 3:
        return S.lut_table(funcs[0], *g)
    outer = S.lut_table(funcs[0], g[0], g[1], g[2])
    mid = g[3] if len(g) == 5 else S.lut_table(funcs[1], g[3], g[4], g[5])
    return S.lut_table(funcs[-1], outer, mid, g[-1])


def _pack(comb):
    p = 0
    for g in comb:
        p = (p << 9) | int(g)
    return p


def _fresh(monkeypatch, **env):
    """A new handle created under the given environment (knobs are read at handle creation)."""
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))
    eng = sb.LutEngine(0)
    for k in env:
        monkeypatch.delenv(k)
    return eng


def _count_free_windows():
    """Ticket counts of the count-free windows (kEnumWindow5 / kEnumWindow7, doubling in run_enum),
    read from the library's source."""
    csrc = os.path.join(S.ROOT, "sboxgates_b200", "csrc")
    api = open(os.path.join(csrc, "sbg_api.cu")).read()
    dev = open(os.path.join(csrc, "sbg_device.cuh")).read()

    def find(pattern, text, where):
        m = re.search(pattern, text)
        assert m is not None, "cannot read %r from %s: update _count_free_windows" % (pattern, where)
        return m.group(1)
    threads = int(find(r"constexpr int kThreads = (\d+);", dev, "sbg_device.cuh"))
    factors = find(r"kNominalWarps = ([\d\s*]+)\* kWarpsPerCta;", api, "sbg_api.cu")
    warps = int(np.prod([int(x) for x in factors.split("*") if x.strip()])) * (threads // 32)
    w5 = warps // int(find(r"kEnumWindow5 = kNominalWarps(?: / (\d+))?;()", api, "sbg_api.cu") or 1)
    w7 = warps // int(find(r"kEnumWindow7 = kNominalWarps(?: / (\d+))?;()", api, "sbg_api.cu") or 1)
    return w5, w7


def _seams(first, upto):
    """Ends of the doubling windows first, 2 first, 4 first, ... below `upto`."""
    out, end, w = [], 0, first
    while end + w < upto:
        end += w
        out.append(end)
        w *= 2
    return out


# ------------------------------------------------------------------------------------------------
# a. Phase-1 lists

# (n, mask spec, gate 0 excluded).  Above n = 200 the masks are small, so that the list reaches the
# cap early and phase 1 does not have to sweep all of C(n, 7); the states at n = 65 ... 200 leave
# their lists short of the cap, so their sweeps cross the head / prefix seam and every word boundary.
A_CASES = [(64, "m0", True), (65, 200, False), (96, 100, True), (96, 255, False), (127, 65, True),
           (127, "m1", False), (128, 129, True), (128, 63, False), (129, "m2", False),
           (200, 33, True), (255, 31, False), (256, "m3", True), (257, 33, False), (300, 31, True),
           (500, 7, False), (500, 1, True)]
BOUNDARIES = [31, 32, 63, 64, 127, 128, 255, 256]   # fourth gates that start a slice


def _a_state(i, n, spec, with0):
    tabs = S.synthetic_state(n, seed=12000 + i)
    mask, fixed = _mask(spec, 12100 + i)
    return tabs, S.sbox_target(S.rijndael_sbox(), i % 8), mask, _inbits(fixed, with0)


def _slice_size(mask):
    """Ranks per slice, by the oracle's cost: ~0.1-0.2 us per combination under large masks, 3-4 us
    per feasible one under small masks, where most of them are."""
    m = _positions(mask)
    return 4_000_000 if m >= 100 else 1_000_000 if m >= 60 else 400_000


def _a_slices(n, inb, mask, limit, seed):
    """[lo, hi) rank slices: the first and last ranks, the first combination of allowed gates whose
    fourth gate is d for each word boundary d, and seeded random ones; clipped to `limit`."""
    size = _slice_size(mask)
    allowed = [g for g in range(n) if g not in inb]
    starts = [E.comb_rank(n, 7, allowed[:7]), max(0, limit - size)]
    for d in BOUNDARIES:
        lead = [g for g in allowed if g < d][:3]
        tail = [g for g in allowed if g >= d][:4]
        if len(lead) == 3 and len(tail) == 4 and tail[0] == d:
            starts.append(E.comb_rank(n, 7, lead + tail))
    rs = np.random.RandomState(seed)
    starts += [int(rs.randint(0, max(1, limit))) for _ in range(2)]
    return sorted({(lo, min(lo + size, limit)) for lo in starts if lo < limit})


def _check_list(n, tabs, tgt, mask, inb, got, stats):
    """Soundness of a whole device list and completeness on slices of ranks."""
    assert np.all(got[1:] > got[:-1]), n
    gates = E.unpack_list(got)
    assert not np.isin(gates, inb).any(), n
    assert np.all(gates[:, :-1] < gates[:, 1:]) and (gates < n).all(), n
    bad, first = E.check7_list(tabs, tgt, mask, gates)
    assert bad == 0, (n, first, gates[first] if first >= 0 else None)
    total = int(S.oracle_lib().orc_n_choose_k(n, 7))
    # a capped list is a prefix of the feasible combinations: compare up to its last entry
    limit = E.comb_rank(n, 7, gates[-1]) + 1 if len(got) == CAP else total
    for lo, hi in _a_slices(n, inb, mask, limit, n):
        want = E.filter7_range(tabs, tgt, mask, inb, lo, hi)
        a = np.searchsorted(got, np.uint64(_pack(E.nth_comb(n, 7, lo))))
        b = len(got) if hi >= total else np.searchsorted(got, np.uint64(_pack(E.nth_comb(n, 7, hi))))
        assert np.array_equal(gates[a:b], want), (n, lo, hi, b - a, len(want))
        stats["slices"] += 1
        stats["feasible"] += len(want)
    stats["states"] += 1
    stats["capped"] += len(got) == CAP
    stats["entries"] += len(got)


def test_phase1_lists_match_oracle(engine, monkeypatch):
    stats = dict(states=0, slices=0, feasible=0, capped=0, entries=0)
    lists = {}
    for i, (n, spec, with0) in enumerate(A_CASES):
        tabs, tgt, mask, inb = _a_state(i, n, spec, with0)
        engine.load(tabs, tgt, mask, inb)
        got = engine.filter7_part(0, 1)
        _check_list(n, tabs, tgt, mask, inb, got, stats)
        lists[i] = got
    # both prefix forms on one state below n = 128 (default: 4-gate prefixes) and one at n = 128
    # (default: 5-gate prefixes), and one head state without its head
    for env, picks in (({"SBG_PM_PREFIX": 4}, [2, 6]), ({"SBG_PM_PREFIX": 5}, [2, 6]),
                       ({"SBG_HEAD": 0}, [8])):
        eng = _fresh(monkeypatch, **env)
        try:
            for i in picks:
                eng.load(*_a_state(i, *A_CASES[i]))
                assert np.array_equal(eng.filter7_part(0, 1), lists[i]), (env, A_CASES[i])
        finally:
            eng.close()
    print("phase-1 lists:", stats)
    assert stats["capped"] >= 4 and stats["capped"] < stats["states"]
    assert stats["feasible"] >= 100_000, stats


# ------------------------------------------------------------------------------------------------
# b. search_5lut keys

# (n, mask spec, gate 0 excluded, planted gates or None for an S-box target).  Planted circuits put
# the first match at a rank the oracle reaches in seconds; S-box targets are searched whole.
B_CASES = [(33, "m0", True, None), (33, 33, False, None), (47, 65, True, None),
           (47, "m3", False, (5, 9, 20, 33, 46)), (52, 100, True, None), (52, 1, False, None),
           (53, "m1", False, None), (53, 129, True, (2, 8, 30, 40, 52)), (64, 200, True, None),
           (64, 7, True, None), (64, "m2", False, (11, 17, 40, 50, 63)),
           (96, 31, True, (1, 3, 40, 70, 95)), (96, 255, False, (0, 4, 9, 60, 90)),
           (128, 63, True, (1, 2, 64, 100, 127)), (128, "m1", False, (0, 5, 31, 32, 127)),
           (130, 129, True, (1, 4, 63, 64, 129)), (130, "m0", False, (0, 2, 7, 128, 129))]
# Far states (n, mask spec, planted gates, rank of the oracle's first match): the planted circuit
# uses gate 0, so that the first match lies early in C(n, 5); the ranks were found with the oracle.
B_FAR = [(200, "m2", (0, 2, 7, 150, 199), 840),          # {0, 1, 2, 7, 70}
         (300, 100, (0, 1, 5, 256, 299), 173_148),     # the planted combination
         (500, 65, (0, 3, 8, 255, 499), 125_720)]      # {0, 1, 3, 8, 499}


def _b_state(i, n, spec, with0, planted):
    tabs = S.synthetic_state(n, seed=13000 + i)
    mask, fixed = _mask(spec, 13100 + i)
    inb = _inbits(fixed, with0)
    if planted is None:
        tgt = S.sbox_target(S.rijndael_sbox(), i % 8)
    else:
        tgt = _plant(tabs, planted, [0x96 ^ i, 0xB1 + i])
    return tabs, tgt, mask, inb


def _b_far(i):
    n, spec, planted, _ = B_FAR[i]
    tabs = S.synthetic_state(n, seed=13500 + i)
    mask, fixed = _mask(spec, 13600 + i)
    return tabs, _plant(tabs, planted, [0x5A + i, 0xE4]), mask, _inbits(fixed, False)


def _b_oracle(tabs, tgt, mask, inb, order):
    n = tabs.shape[0]
    total = int(S.oracle_lib().orc_n_choose_k(n, 5))
    return E.search5_range(tabs, tgt, mask, inb, order, 0, total, 1_000_000)


def test_search5_keys_match_oracle(engine, monkeypatch):
    engines = {"two": _fresh(monkeypatch, SBG_SEARCH5="two"),
               "fused": _fresh(monkeypatch, SBG_SEARCH5="fused")}
    found = compared = 0
    try:
        for i, case in enumerate(B_CASES):
            n = case[0]
            tabs, tgt, mask, inb = _b_state(i, *case)
            order = E.orders(300 + i)[0]
            want = _b_oracle(tabs, tgt, mask, inb, order)
            extra = [engines["two"], engines["fused"]] if n in (52, 53, 96, 128) else []
            for eng in [engine] + extra:
                eng.load(tabs, tgt, mask, inb)
                assert int(eng.search5(order).key) == want, (case, eng is engine)
                compared += 1
            found += want != NONE
            if n <= 64:
                # ret[10] and the RNG draws, through the reference-shaped call
                seed = np.random.RandomState(i).bytes(128)
                o_rng = S.OrcRng.from_seed(seed)
                ok, ret, _ = S.oracle_search(5, tabs, tgt, mask, inb, o_rng)
                g_rng = Xorshift1024(seed)
                res = sb.search_5lut(engine, tabs, tgt, mask, inb, g_rng)
                assert (res.found, res.ret) == (ok, ret) and g_rng.draws == o_rng.draws, case
        for i, (n, spec, planted, rank) in enumerate(B_FAR):
            tabs, tgt, mask, inb = _b_far(i)
            order = E.orders(400 + i)[0]
            want = E.search5_range(tabs, tgt, mask, inb, order, 0, 2 * 10**8, 1_000_000)
            assert want != NONE and want >> 12 == rank, (n, want >> 12)
            engine.load(tabs, tgt, mask, inb)
            assert int(engine.search5(order).key) == want, n
            compared += 1
            found += 1
    finally:
        for eng in engines.values():
            eng.close()
    print("search_5lut keys: %d comparisons, %d states with a match" % (compared, found))
    assert found >= 10


# ------------------------------------------------------------------------------------------------
# c. 3-LUT scan

C_CASES = [(64, "m0"), (255, 200), (256, "m1"), (257, 129), (500, 255)]


def test_scan3_matches_oracle_at_large_n(engine):
    """lut_search with search_5lut / search_7lut off is the 3-LUT scan alone: its stage, triple,
    function and RNG draws against orc_scan3_key and the oracle's get_lut_function.  The planted
    triple is three random tables at the last positions of the gate order, which no other triple
    realises under these large masks: at n = 257 and 500 its key has fields >= 256."""
    sbox = S.rijndael_sbox()
    hits = high = 0
    for i, (n, spec) in enumerate(C_CASES):
        rs = np.random.RandomState(14200 + i)
        tabs = np.concatenate([S.synthetic_state(n - 3, seed=14000 + i),
                               rs.randint(0, 2**63, (3, 4)).astype(np.uint64) * np.uint64(2)
                               + rs.randint(0, 2, (3, 4)).astype(np.uint64)])
        mask, _ = _mask(spec, 14100 + i)
        order = [int(x) for x in rs.permutation(n - 3)] + [int(x) for x in rs.permutation(3) + n - 3]
        for tgt in (_plant(tabs, [n - 3, n - 2, n - 1], [0x6B ^ i]), S.sbox_target(sbox, i % 8)):
            key = E.scan3_key(tabs, tgt, mask, order)
            seed = rs.bytes(128)
            g_rng, o_rng = Xorshift1024(seed), S.OrcRng.from_seed(seed)
            got = sb.lut_search(engine, tabs, tgt, mask, [], order, g_rng, allow5=False,
                                allow7=False)
            if key == NONE:
                assert got.stage == 0 and g_rng.draws == 0, (n, spec)
                continue
            trip = [order[key >> 18], order[(key >> 9) & 0x1FF], order[key & 0x1FF]]
            ok, func = S.oracle_get_lut_function(*[tabs[x] for x in trip], tgt, mask, o_rng)
            assert ok and got.stage == 3, (n, spec)
            assert int(got.node.key3) == key, (n, spec, hex(int(got.node.key3)), hex(key))
            assert got.luts[0] == (func, *trip) and g_rng.draws == o_rng.draws, (n, spec)
            hits += 1
            high += (key & 0x1FF) >= 256
    assert hits >= 4 and high >= 2


# ------------------------------------------------------------------------------------------------
# d. Enumerations past one count-free window

K5 = 5000
# (seed, n, random mask size, excluded input bits, planted gates or None for an S-box target).  The
# last two states exclude input bits 0 - 3, so that their first allowed 3-gate prefix (4, 5, 6) lies
# past the second count-free window (the windows end at prefix tickets 2,112, 6,336, 14,784, ...).
# Their S-box targets have 29,914 and 102,048 matches, the 5,000th at tickets 12,116 and 8,777.
D_CASES = [(0, 40, 33, [0], (3, 12, 20, 31, 39)), (1, 64, 65, [], (10, 30, 33, 62, 63)),
           (2, 64, 129, [0], (25, 40, 41, 50, 60)), (3, 96, 200, [], (40, 63, 64, 80, 95)),
           (4, 96, 100, [0], (33, 34, 70, 90, 94)), (505, 64, 24, [0, 1, 2, 3], None),
           (508, 64, 24, [0, 1, 2, 3], None)]


def _d_state(s, n, spec, inb, planted):
    tabs = S.synthetic_state(n, seed=15000 + s)
    mask, _ = _mask(spec, 15100 + s)
    tgt = (S.sbox_target(S.rijndael_sbox(), s % 8) if planted is None
           else _plant(tabs, planted, [0xD2 ^ s, 0x35 + s]))
    return tabs, tgt, mask, inb


def _prefix_ticket(n, key):
    """The count-free ticket of a 5-LUT key: the rank of its 3-gate prefix among those of C(n,5)."""
    comb = E.nth_comb(n, 5, key >> 12)
    return E.comb_rank(n - 2, 3, comb[:3])


def test_enum5_across_windows_matches_oracle(engine):
    w5, _ = _count_free_windows()
    beyond = matches = 0
    for case in D_CASES:
        s, n = case[:2]
        tabs, tgt, mask, inb = _d_state(*case)
        order = E.orders(500 + s)[0]
        total, keys, feasible = E.enum5_range(tabs, tgt, mask, inb, order, K5)
        assert total > 0, case
        engine.load(tabs, tgt, mask, inb)
        counted = engine.enumerate5(order, K5)
        assert (counted.total, counted.feasible) == (total, feasible), (case, counted.total, total)
        assert [int(k) for k in counted.matches["key"]] == keys, case
        free = engine.enumerate5(order, K5, count=False)
        assert free.total is None and np.array_equal(free.matches, counted.matches), case
        for rec in list(counted.matches[:40]) + list(counted.matches[-20:]):
            want = E.expected_record(5, int(rec["key"]), tabs, tgt, mask, order)
            assert want is not None and E.record_fields(rec) == want, (case, hex(int(rec["key"])))
        # the count-free run stopped after a window past the second one, on its K-th match
        beyond += total >= K5 and _prefix_ticket(n, keys[-1]) >= w5 + 2 * w5
        matches += len(keys)
    print("enum5: %d states, %d matches compared" % (len(D_CASES), matches))
    assert beyond >= 1


def _n40_state():
    """The fourth state of bench.py's n = 40 step with seed 1, rebuilt here with the same draws:
    32 positions (input bits 5, 2, 0 fixed and excluded), target = bit 0 of the AES S-box."""
    rs = np.random.RandomState(1)
    for i in range(4):
        bits = rs.choice(8, i, replace=False)
        fixed = [(int(b), int(rs.randint(0, 2))) for b in bits]
        _, outer, middle = [bytes(rs.permutation(256).astype(np.uint8)) for _ in range(3)]
        seed = int(rs.randint(1 << 30))
    return (S.synthetic_state(40, seed), S.sbox_target(S.rijndael_sbox(), 0), S.mux_mask(fixed),
            [b for b, _ in fixed], outer, middle)


def test_enum7_long_list_matches_oracle(engine):
    """A state shaped like bench.py's n = 40 state under 32 positions (selector bits 0, 2, 5
    excluded): a 71,000-entry list with about 250,000 matches, fetched whole; about 26 entries
    checked against the oracle, among them both sides of every count-free window seam."""
    _, w7 = _count_free_windows()
    tabs, tgt, mask, inb, outer, middle = _n40_state()
    assert 0 in inb and _positions(mask) == 32
    engine.load(tabs, tgt, mask, inb)
    first = engine.enumerate7(outer, middle, 0)
    total, count = first.total, first.feasible
    assert count > 50_000 and total > 100_000
    e = engine.enumerate7(outer, middle, total)
    assert e.total == total and len(e.matches) == total
    keys = e.matches["key"].astype(np.uint64)
    assert np.all(keys[1:] > keys[:-1])
    lst = E.unpack_list(engine.filter7_part(0, 1))
    assert len(lst) == count
    idx = (keys >> np.uint64(23)).astype(np.int64)
    seams = _seams(w7, count)
    rs = np.random.RandomState(40)
    # matches are rare and clustered: half of the random entries are drawn among those holding some
    with_matches = np.unique(idx)
    entries = sorted({0, count - 1} | {s + d for s in seams for d in (-1, 0)}
                     | {int(x) for x in rs.randint(0, count, 4)}
                     | {int(x) for x in rs.choice(with_matches, 6, replace=False)})
    with E.ThreadPoolExecutor(max_workers=E.workers()) as pool:
        wants = list(pool.map(lambda j: E.oracle_enum7(tabs, tgt, mask, lst[j:j + 1], outer, middle,
                                                       1 << 16), entries))
    checked = 0
    for j, (t, ks) in zip(entries, wants):
        sel = e.matches[idx == j]
        assert len(sel) == t, (j, len(sel), t)
        assert [int(k) for k in sel["key"]] == [(j << 23) | k for k in ks], j
        for rec in sel[:5]:
            want = E.expected_record(7, int(rec["key"]), tabs, tgt, mask, outer, middle, lst[j])
            assert E.record_fields(rec) == want, (j, hex(int(rec["key"])))
        checked += t
    assert checked > 0
    # count-free runs: prefixes of the counted records
    k2 = int(np.sum(idx < seams[1])) if len(seams) > 1 else total
    for k in sorted({1, k2, total - 1, total, total + 1}):
        free = engine.enumerate7(outer, middle, k, count=False)
        assert np.array_equal(free.matches, e.matches[:k]), k
    assert int(engine.search7(outer, middle).key) == int(keys[0])
    print("enum7 long list: %d entries, %d matches, %d entries / %d matches checked by the oracle"
          % (count, total, len(entries), checked))


# ------------------------------------------------------------------------------------------------
# e. Masks of 0 - 3 positions

def _tiny_mask(m, seed):
    return _mask(m, seed)[0] if m else np.zeros(4, dtype=np.uint64)


@pytest.mark.parametrize("m", [0, 1, 2, 3])
def test_degenerate_masks_match_oracle(engine, m):
    """With no masked position the reference finds every combination feasible and matches on its
    first candidate, with every inner bit a random fill; with 1 - 3 positions nearly so."""
    sbox = S.rijndael_sbox()
    for i, (n, inb) in enumerate([(7, []), (9, [0]), (12, [1, 3]), (12, [0, 2])]):
        tabs = S.synthetic_state(n, seed=16000 + 10 * m + i)
        mask = _tiny_mask(m, 16100 + 10 * m + i)
        tgt = S.sbox_target(sbox, (m + i) % 8)
        assert _positions(mask) == m
        seed = np.random.RandomState(m * 10 + i).bytes(128)
        for which, fn in ((5, sb.search_5lut), (7, sb.search_7lut)):
            o_rng, g_rng = S.OrcRng.from_seed(seed), Xorshift1024(seed)
            ok, ret, _ = S.oracle_search(which, tabs, tgt, mask, inb, o_rng)
            res = fn(engine, tabs, tgt, mask, inb, g_rng)
            assert (res.found, res.ret) == (ok, ret), (m, n, which, res.ret, ret)
            assert g_rng.draws == o_rng.draws, (m, n, which)
        # lut_search: the 3-LUT scan finds the first triple of the order
        order = [int(x) for x in np.random.RandomState(i).permutation(n)]
        key = E.scan3_key(tabs, tgt, mask, order)
        o_rng, g_rng = S.OrcRng.from_seed(seed), Xorshift1024(seed)
        got = sb.lut_search(engine, tabs, tgt, mask, inb, order, g_rng)
        assert key != NONE and got.stage == 3, (m, n)
        trip = [order[key >> 18], order[(key >> 9) & 0x1FF], order[key & 0x1FF]]
        _, func = S.oracle_get_lut_function(*[tabs[x] for x in trip], tgt, mask, o_rng)
        assert got.luts[0] == (func, *trip) and g_rng.draws == o_rng.draws, (m, n)
        # enumerations
        order5, outer, middle = E.orders(600 + i)
        total, keys, feasible = E.oracle_enum5(tabs, tgt, mask, inb, order5, 300)
        e5 = sb.enumerate_5lut(engine, tabs, tgt, mask, inb, order5, 300)
        assert (e5.total, e5.feasible) == (total, feasible), (m, n)
        assert [int(k) for k in e5.matches["key"]] == keys, (m, n)
        engine.load(tabs, tgt, mask, inb)
        lst = engine.filter7_part(0, 1)
        want_list, _ = S.oracle_filter7(tabs, tgt, mask, inb)
        assert np.array_equal(E.unpack_list(lst), want_list), (m, n)
        engine.set_list7(lst[:2])
        total7, keys7 = E.oracle_enum7(tabs, tgt, mask, want_list[:2], outer, middle, 300)
        e7 = engine.enumerate7(outer, middle, 300)
        assert e7.total == total7 and [int(k) for k in e7.matches["key"]] == keys7, (m, n)
        for rec in e7.matches[:10]:
            key7 = int(rec["key"])
            want = E.expected_record(7, key7, tabs, tgt, mask, outer, middle, want_list[key7 >> 23])
            assert E.record_fields(rec) == want, (m, n, hex(key7))
