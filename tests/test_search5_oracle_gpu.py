"""GPU: search_5lut (k_sweep, k_decomp5, sbg_finish5) against the CPU oracle at every mask width.

Whole keys and the keys of the library's shares of a sharded search (sbg_search5_part, modelled by
Deal5 in tests/_enum_support.py) at n = 5 ... 500, every ordering row as the first-match row,
outer positions at the end of the shuffled order, ranks past 2^32, the full sbg_result through
every entry path (sbg_search5, search_node, search_batch, search5_part + finish5 on the finding
and on another handle), the feasible counts, and the two-kernel form's overflow fallback.  Each
comparison runs on the default handle and on handles forced to the two-kernel form
(SBG_SEARCH5=two), the fused form (SBG_SEARCH5=fused; its chunk head from n = 128 on) and the fused
form without the head (SBG_HEAD=0).  The oracle's keys come from orc_search5_range, its results from
expected_result5."""
from math import comb

import numpy as np
import pytest

import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200.rng import Xorshift1024

pytestmark = pytest.mark.gpu

NONE = E.NONE
ENVS = {"default": {}, "two": {"SBG_SEARCH5": "two"}, "fused": {"SBG_SEARCH5": "fused"},
        "prefix": {"SBG_SEARCH5": "fused", "SBG_HEAD": "0"}}
MUX = [[], [(3, 1)], [(0, 0), (5, 1)], [(1, 1), (4, 0), (6, 1)]]   # mux masks of depth 0-3
ODD = [1, 7, 31, 33, 63, 65, 100, 129, 200, 255]
FUNCS = [0x96, 0xE8, 0xCA, 0xD8, 0x1B, 0x6A, 0xB4, 0x78, 0x3C, 0xA6]
ASYM = [0xCA, 0xD8, 0xE4, 0xB4, 0xA6, 0x1B, 0x72, 0x4E, 0x2D, 0x8E]   # no two inputs symmetric
TWO_KERNEL_MAX = 4_000_000   # the default form is two kernels up to C(n,5) = 4e6 (n = 52)
LIMIT = 3_000_000            # combinations the oracle walks for one part before giving up on it


def _fresh(**env):
    mp = pytest.MonkeyPatch()
    try:
        for k, v in env.items():
            mp.setenv(k, v)
        return sb.LutEngine(0)   # knobs are read when the handle is created
    finally:
        mp.undo()


@pytest.fixture(scope="module")
def engines():
    out = {name: _fresh(**env) for name, env in ENVS.items()}
    yield out
    for e in out.values():
        e.close()


def form_of(name, n):
    """The kernel form handle `name` runs at n gates: two kernels, fused over prefixes, or fused
    with the chunk head in front."""
    if name == "two" or (name == "default" and comb(n, 5) <= TWO_KERNEL_MAX):
        return "two"
    return "prefix" if name == "prefix" or n < 128 else "head"


def handles_for(n):
    """The handles a state of n gates runs on: the two-kernel form where its sweep stays short (it
    never stops early), the headless fused form where the head exists."""
    return ["default", "fused"] + (["two"] if n <= 130 else []) + (["prefix"] if n >= 128 else [])


def random_mask(rs, size):
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, size, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def nw_of(mask):
    """The words per compressed table the kernels run with: 1, 2, 4 or 8 (with_nw)."""
    m = sum(bin(int(w)).count("1") for w in mask)
    return 1 << (max(1, -(-m // 32)) - 1).bit_length()


def to_end(order, funcs):
    """The order with `funcs` moved to positions 255, 254, ..."""
    o = list(order)
    for i, f in enumerate(funcs):
        j, t = o.index(f), 255 - i
        o[j], o[t] = o[t], o[j]
    return bytes(o)


def check_result(res, want, what):
    got = E.result5_fields(res)
    if want is None:
        assert (got["found"], got["key"]) == (0, NONE), what
        return
    for f, v in want.items():
        assert got[f] == v, (what, f, got[f], v)


COVER = {"nw": set(), "rows": set(), "pos": 0, "rank": 0, "parts": 0, "part_sets": set(),
         "redo5": 0, "redo7": 0}


def note(key, nw, form, rows=True):
    COVER["nw"].add((nw, form))
    if key == NONE:
        return
    if rows:
        COVER["rows"].add(((key >> 8) & 0xF, nw, form))
    COVER["pos"] = max(COVER["pos"], key & 0xFF)
    COVER["rank"] = max(COVER["rank"], key >> 12)


# ------------------------------------------------------------------------------------------------
# a: whole keys and part keys at many sizes and masks

NS = [5, 6, 7, 14, 33, 52, 53, 64, 96, 127, 128, 130, 257, 500]


def _key_cases():
    rs = np.random.RandomState(9090)
    masks = ["m%d" % d for d in range(4)] + ODD
    sbox = S.rijndael_sbox()
    for i in range(2 * len(NS)):
        n = NS[i % len(NS)]
        spec = masks[(3 * i) % len(masks)]
        if n >= 128 and isinstance(spec, int) and spec < 31 and i < len(NS):
            spec = 31   # no two-kernel sweep overflow at n >= 128 (see handles_for)
        if isinstance(spec, str):
            fixed = MUX[int(spec[1:])]
            mask = S.mux_mask(fixed)
        else:
            fixed, mask = [], random_mask(rs, spec)
        with0 = i % 2 == 0
        inb = sorted({b for b, _ in fixed if b < n} | ({0} if with0 else set()))
        tabs = S.synthetic_state(n, seed=9100 + i, num_inputs=min(8, n))
        allowed = [g for g in range(n) if g not in inb]
        if n <= 64 and i % 3 == 0:
            tgt = S.sbox_target(sbox, i % 8)
        elif len(allowed) >= 5:
            # planted on the first two allowed gates, so that the first match comes early
            rest = sorted(int(x) for x in rs.choice(allowed[2:], 3, replace=False))
            tgt = E.planted5(tabs, allowed[:2] + rest, int(rs.randint(10)),
                             *(int(x) for x in rs.choice(FUNCS, 2)))
        else:
            tgt = S.sbox_target(sbox, 0)
        yield tabs, tgt, mask, inb, bytes(rs.permutation(256).astype(np.uint8))


def test_keys_and_part_keys_match_the_oracle(engines):
    found = skipped = 0
    for i, (tabs, tgt, mask, inb, order) in enumerate(_key_cases()):
        n = len(tabs)
        limit = None if n <= 64 else LIMIT
        oracles = {}
        for name in handles_for(n):
            form = form_of(name, n)
            head = form == "head"
            if head not in oracles:
                oracles[head] = E.Search5Oracle(tabs, tgt, mask, inb, order, head)
            orc = oracles[head]
            whole = orc.part_key(0, 1, None if n <= 64 else 50 * LIMIT)
            assert whole is not None, (i, n)
            eng = engines[name]
            eng.load(tabs, tgt, mask, inb)
            got = int(eng.search5(order).key)
            assert got == whole, (i, n, name, hex(got), hex(whole))
            note(got, nw_of(mask), form, rows=False)
            found += whole != NONE
            sets = [2, 3, 7] + ([orc.deal.blocks() + 3] if n <= 14 else [])
            for P in sets:
                for p in range(P):
                    want = orc.part_key(p, P, limit)
                    if want is None:
                        skipped += 1
                        continue
                    got = eng.search5_part(p, P, order)
                    assert got == want, (i, n, name, P, p, hex(got), hex(want))
                    COVER["parts"] += 1
                    COVER["part_sets"].add((form, P if P <= 7 else "blocks+3"))
                    if n <= 14 and P > 7 and not orc.deal.part_blocks(p, P):
                        COVER["part_sets"].add((form, "empty"))
    print("keys: %d whole-key hits, %d parts compared, %d parts past the oracle's reach"
          % (found, COVER["parts"], skipped))
    assert found >= 30
    assert {(f, "empty") for f in ("two", "prefix")} <= COVER["part_sets"]


# ------------------------------------------------------------------------------------------------
# b: every ordering row first, at NW 1, 2, 4, 8, in the two-kernel, fused prefix and head forms

def _row_cases():
    rs = np.random.RandomState(9191)
    sizes = [32, 64, 128, 256]   # NW 1, 2, 4, 8
    for k in range(10):
        for size in sizes:
            for n in (48, 128):
                for s in range(3 if size in (32, 256) else 1):
                    tabs = S.synthetic_state(n, seed=9200 + 1000 * s + 10 * k + size + n)
                    mask = random_mask(rs, size)
                    fo, fi = (int(x) for x in rs.choice(ASYM, 2))
                    # gates 0, 1 and 2 first: the oracle reaches the planted rank in milliseconds
                    gates = [0, 1, 2] + sorted(int(x) for x in rs.choice(np.arange(3, n), 2,
                                                                          replace=False))
                    tgt = E.planted5(tabs, gates, k, fo, fi)
                    order = bytes(rs.permutation(256).astype(np.uint8))
                    if s != 1:
                        rep = min(fo, 255 - fo)
                        order = to_end(order, [rep, 255 - rep] if s == 0 else [255 - rep, rep])
                    yield tabs, tgt, mask, order, k, comb_rank(n, gates)


def comb_rank(n, gates):
    return E.comb_rank(n, 5, gates)


@pytest.fixture(scope="module")
def row_cases():
    out = []
    for tabs, tgt, mask, order, k, rank in _row_cases():
        key = E.search5_range(tabs, tgt, mask, [], order, 0, rank + 1, 20_000)
        assert key != NONE
        out.append((tabs, tgt, mask, order, k, key))
    return out


def test_row_keys_and_results_match_the_oracle(engines, row_cases):
    for tabs, tgt, mask, order, k, key in row_cases:
        n = len(tabs)
        want = E.expected_result5(key, tabs, tgt, mask, order)
        for name in handles_for(n):
            eng = engines[name]
            eng.load(tabs, tgt, mask, [])
            res = eng.search5(order)
            check_result(res, want, (n, k, name))
            note(int(res.key), nw_of(mask), form_of(name, n))
    for form in ("two", "prefix", "head"):
        for nw in (1, 8):
            rows = {r for r, w, f in COVER["rows"] if (w, f) == (nw, form)}
            assert rows == set(range(10)), (form, nw, sorted(set(range(10)) - rows))
    assert COVER["pos"] >= 250, COVER["pos"]


# ------------------------------------------------------------------------------------------------
# c: the result through every entry path

def _path_cases():
    rs = np.random.RandomState(9292)
    specs = [(14, 32), (33, 64), (40, 100), (52, 129), (53, 200), (64, 255), (96, 33), (130, 150),
             (24, 65), (48, 31)]
    for i, (n, size) in enumerate(specs):
        tabs = S.synthetic_state(n, seed=9300 + i)
        mask = random_mask(rs, size)
        gates = sorted(int(x) for x in rs.choice(n, 5, replace=False))
        if n > 64:
            gates = [0, 1] + gates[2:] if gates[1] > 1 else gates
        tgt = E.planted5(tabs, gates, int(rs.randint(10)), *(int(x) for x in rs.choice(FUNCS, 2)))
        if i == 9:   # a miss
            tgt = S.sbox_target(S.rijndael_sbox(), 3)
        yield tabs, tgt, mask, rs.bytes(128)


def test_results_through_every_entry_path(engines):
    cases = []
    for tabs, tgt, mask, seed in _path_cases():
        n = len(tabs)
        order = sb.shuffled_order(Xorshift1024(seed))
        key = E.search5_range(tabs, tgt, mask, [], order, 0, comb(n, 5), 200_000)
        go = [int(x) for x in np.random.RandomState(n).permutation(n)]
        assert E.scan3_key(tabs, tgt, mask, go) == NONE
        cases.append((tabs, tgt, mask, seed, order, go, key,
                      E.expected_result5(key, tabs, tgt, mask, order)))
    assert sum(c[6] == NONE for c in cases) == 1
    names = ["default", "two", "fused"]
    for name in names:
        eng = engines[name]
        other = engines[names[(names.index(name) + 1) % 3]]
        for i, (tabs, tgt, mask, seed, order, go, key, want) in enumerate(cases):
            n = len(tabs)
            what = (name, i, n)
            eng.load(tabs, tgt, mask, [])
            check_result(eng.search5(order), want, what + ("search5",))
            eng.stage(1, tabs, tgt, mask, [])
            node = eng.search_node(1, order5=order, gate_order=go)
            assert node.key3 == NONE and node.found_stage == (5 if want else 0), what
            check_result(node.r5, want, what + ("node",))
            eng.use(1)
            if key == NONE:
                continue
            # search5_part over 3 parts, the winning part last, then finish5 here and on a handle
            # that searched another part
            win = [p for p in range(3) if eng.search5_part(p, 3, order) == key]
            assert len(win) == 1, what
            keys = [eng.search5_part(p, 3, order) for p in range(3) if p != win[0]]
            assert eng.search5_part(win[0], 3, order) == key and min(keys) > key, what
            check_result(eng.finish5(key, order), want, what + ("finish5 here",))
            other.load(tabs, tgt, mask, [])
            other.search5_part((win[0] + 1) % 3, 3, order)
            check_result(other.finish5(key, order), want, what + ("finish5 elsewhere",))
            note(key, nw_of(mask), form_of(name, n), rows=False)
        # search_batch: every state staged, mixed n and NW, some with the 3-LUT scan in front
        for i, c in enumerate(cases):
            eng.stage(i, c[0], c[1], c[2], [])
        jobs = [dict(slot=i, order5=c[4], gate_order=c[5] if i % 2 else None)
                for i, c in enumerate(cases)]
        for i, (r, c) in enumerate(zip(eng.search_batch(jobs), cases)):
            check_result(r.r5, c[-1], (name, i, "batch"))
            assert r.found_stage == (5 if c[-1] else 0)
    # ret[10] and the RNG draws against the oracle's search_5lut where n <= 64
    eng = engines["default"]
    for tabs, tgt, mask, seed, *_ in cases:
        if len(tabs) > 64:
            continue
        o_rng = S.OrcRng.from_seed(seed)
        found, ret, _ = S.oracle_search(5, tabs, tgt, mask, [], o_rng)
        g_rng = Xorshift1024(seed)
        res = sb.search_5lut(eng, tabs, tgt, mask, [], g_rng)
        assert (res.found, res.ret) == (found, ret) and g_rng.draws == o_rng.draws


# ------------------------------------------------------------------------------------------------
# d: ranks past 2^32

def test_ranks_past_2_to_the_32(engines):
    """Input bits 0-7 excluded: the first allowed combination (8, 9, 10, 11, 12) has rank 2.4e9 at
    n = 300 and 2.0e10 (> 2^34) at n = 500.  Circuits planted on gates >= 8 and >= 256."""
    rs = np.random.RandomState(9393)
    inb = list(range(8))
    done = 0
    for i, (n, spec, gates) in enumerate([(300, 100, [8, 9, 11, 256, 299]),
                                          (300, "m2", [8, 10, 12, 257, 280]),
                                          (500, 65, [8, 9, 10, 300, 499]),
                                          (500, "m3", [8, 9, 12, 256, 257])]):
        tabs = S.synthetic_state(n, seed=9400 + i)
        mask = S.mux_mask(MUX[int(spec[1:])]) if isinstance(spec, str) else random_mask(rs, spec)
        tgt = E.planted5(tabs, gates, int(rs.randint(10)), *(int(x) for x in rs.choice(FUNCS, 2)))
        order = bytes(rs.permutation(256).astype(np.uint8))
        first = E.comb_rank(n, 5, [8, 9, 10, 11, 12])
        planted = E.comb_rank(n, 5, gates)
        assert first > 2**31 and (n < 500 or first > 2**34)
        key = E.search5_range(tabs, tgt, mask, inb, order, first, planted + 1, 200_000)
        assert key != NONE and key >> 12 > 2**31
        want = E.expected_result5(key, tabs, tgt, mask, order)
        for name in handles_for(n):
            form = form_of(name, n)
            eng = engines[name]
            eng.load(tabs, tgt, mask, inb)
            check_result(eng.search5(order), want, (n, name))
            note(key, nw_of(mask), form, rows=False)
            # the parts holding the planted combination (the others sweep on for minutes)
            orc = E.Search5Oracle(tabs, tgt, mask, inb, order, form == "head")
            for P in (2, 3, 7):
                for p in range(P):
                    w = orc.part_key(p, P, LIMIT)
                    if w is None:
                        continue
                    assert eng.search5_part(p, P, order) == w, (n, name, P, p)
                    COVER["parts"] += 1
                    done += 1
    assert done >= 12
    assert COVER["rank"] > 2**34


# ------------------------------------------------------------------------------------------------
# e: feasible counts

def test_feasible_counts(engines):
    """tuples_feasible = the oracle's count of feasible 5-combinations (inbits applied): on misses in
    every form and through node and batch, on two-kernel hits too (its sweep covers everything),
    and the parts' counts sum to the whole.  The fused form's count on a hit is the tuples its
    warps decomposed before they stopped, which depends on scheduling: not pinned."""
    rs = np.random.RandomState(9494)
    sbox = S.rijndael_sbox()
    cases = []
    for i, (n, spec, with0, hit) in enumerate([(14, "m2", True, False), (33, "m1", False, False),
                                               (40, 63, True, True), (52, 33, False, False),
                                               (53, "m3", True, False), (64, "m2", False, False),
                                               (48, 129, False, True), (24, 7, True, True),
                                               (14, "c", False, False), (20, "c", True, False),
                                               (24, "c", False, False)]):
        tabs = S.synthetic_state(n, seed=9500 + i)
        fixed = MUX[int(spec[1:])] if spec in ("m0", "m1", "m2", "m3") else []
        mask = S.mux_mask(fixed) if isinstance(spec, str) else random_mask(rs, spec)
        inb = sorted({b for b, _ in fixed} | ({0} if with0 else set()))
        if spec == "c":   # feasible combinations, none of which decomposes
            tabs, tgt, mask = _class_state(n, 0x116, 9500 + i)
        elif hit:
            gates = sorted(int(x) for x in rs.choice(np.arange(8, n), 5, replace=False))
            tgt = E.planted5(tabs, gates, int(rs.randint(10)), 0xCA, 0xE4)
        else:
            tgt = S.sbox_target(sbox, i % 8)
        order = bytes(rs.permutation(256).astype(np.uint8))
        key = E.search5_range(tabs, tgt, mask, inb, order, 0, comb(n, 5), 500_000)
        assert (key != NONE) == hit, (i, n)
        cases.append((tabs, tgt, mask, inb, order, key, E.feasible5(tabs, tgt, mask, inb)))
    assert sum(c[-1] > 0 for c in cases if c[5] == NONE) >= 3
    for name in ("default", "two", "fused"):
        eng = engines[name]
        for i, (tabs, tgt, mask, inb, order, key, feas) in enumerate(cases):
            n = len(tabs)
            two = form_of(name, n) == "two"
            eng.load(tabs, tgt, mask, inb)
            r = eng.search5(order)
            assert int(r.key) == key, (name, i)
            if key == NONE or two:
                assert int(r.tuples_feasible) == feas, (name, i, int(r.tuples_feasible), feas)
                parts = []
                for p in range(3):
                    k = eng.search5_part(p, 3, order)
                    parts.append(int(eng.finish5(k, order).tuples_feasible))
                assert sum(parts) == feas, (name, i, parts, feas)
            if key == NONE:
                eng.stage(2, tabs, tgt, mask, inb)
                node = eng.search_node(2, order5=order)
                assert int(node.r5.tuples_feasible) == feas and node.found_stage == 0
                eng.use(2)
        for i, c in enumerate(cases):
            eng.stage(i, *c[:4])
        res = eng.search_batch([dict(slot=i, order5=c[4]) for i, c in enumerate(cases)])
        for i, (r, c) in enumerate(zip(res, cases)):
            assert int(r.r5.key) == c[5]
            if c[5] == NONE or form_of(name, len(c[0])) == "two":
                assert int(r.r5.tuples_feasible) == c[-1], (name, "batch", i)


# ------------------------------------------------------------------------------------------------
# f: the two-kernel form's hit buffer overflows

HITS_CAP_TUPLES = (4 << 20) // 2   # kDefaultHitsCap words, two per recorded tuple
FORCED_CAP_TUPLES = 3 * (100_000 + 32 * 512) // 2   # SBG_HITS_CAP=1, clamped to 3 kPerPrefixMax
ROOMY_WORDS = 8 << 20   # holds C(52, 5) tuples of two words


def _class_state(n, f, seed):
    """A state whose gates are, on 16 masked positions (a 4-cube), copies of the 4 coordinates (or
    their complements), and a target f of the coordinates there.  A 5-combination is feasible iff
    it holds all 4 coordinates; for f = 0x116 none decomposes (checked by the oracle below)."""
    rs = np.random.RandomState(seed)
    pos = rs.choice(256, 16, replace=False)

    def table(vals):
        t = rs.randint(0, 2**32, 8).astype(np.uint64)
        t = (t[:4] << np.uint64(32)) | t[4:]
        for i, p in enumerate(pos):
            bit = np.uint64(1) << np.uint64(p & 63)
            t[p >> 6] = (t[p >> 6] | bit) if vals[i] else (t[p >> 6] & ~bit)
        return t
    cls = rs.permutation([i % 4 for i in range(n)])
    flips = rs.randint(0, 2, n)
    tabs = np.stack([table([((i >> c) & 1) ^ int(x) for i in range(16)]) for c, x in zip(cls, flips)])
    mask = np.zeros(4, dtype=np.uint64)
    for p in pos:
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return tabs, table([(f >> i) & 1 for i in range(16)]), mask


def _oracle7(tabs, tgt, mask, outer, middle):
    lst, _ = S.oracle_filter7(tabs, tgt, mask, [])
    key = E.decomp7_key(tabs, tgt, mask, lst, outer, middle)
    return E.expected_result7(key, lst, tabs, tgt, mask, outer, middle)


def _check_node(node, want5, want7, what):
    check_result(node.r5, want5, what + ("r5",))
    if want5 is not None:
        assert node.found_stage == 5, what
        return
    assert E.result7_fields(node.r7) == want7, what
    assert node.found_stage == 7, what


def test_overflow_fallback(engines):
    rs = np.random.RandomState(9595)
    cases = []
    # fresh default handles at n = 51, 52 under masks of 1 and 2 positions
    for i, (n, size) in enumerate([(51, 1), (52, 2)]):
        tabs = S.synthetic_state(n, seed=9600 + i)
        mask = random_mask(rs, size)
        tgt = S.sbox_target(S.rijndael_sbox(), i)
        cases.append(("default", tabs, tgt, mask))
    # fresh handles with the hit buffer forced to its minimum, n = 40-48: two hits, and one state
    # without any 5-LUT match whose node and batch chains must redo the 7-LUT stage
    for i, n in enumerate((41, 44)):
        tabs, tgt, mask = _class_state(n, 0x6996, 9700 + i)   # parity: decomposes
        cases.append(("capped", tabs, tgt, mask))
    tabs, tgt, mask = _class_state(40, 0x116, 9702)
    cases.append(("capped", tabs, tgt, mask))
    seen_miss = False
    for i, (kind, tabs, tgt, mask) in enumerate(cases):
        n = len(tabs)
        order = bytes(rs.permutation(256).astype(np.uint8))
        outer, middle = sb.shuffled_orders7(Xorshift1024(rs.bytes(128)))
        feas = E.feasible5(tabs, tgt, mask, [])
        assert feas > (HITS_CAP_TUPLES if kind == "default" else FORCED_CAP_TUPLES), (i, feas)
        key = E.search5_range(tabs, tgt, mask, [], order, 0, comb(n, 5), 100_000)
        want5 = E.expected_result5(key, tabs, tgt, mask, order)
        want7 = None if want5 is not None else _oracle7(tabs, tgt, mask, outer, middle)
        seen_miss |= want5 is None
        env = {} if kind == "default" else {"SBG_HITS_CAP": "1"}
        what = (kind, i, n)
        # Launches of search5 without a fallback: the fused form (k_begin, k_sweep) and the
        # two-kernel form on a buffer that holds every tuple (k_begin, k_sweep, k_decomp5).  A
        # fallback makes both: the two-kernel launches, then the fused ones.
        quiet = engines["fused"]
        quiet.load(tabs, tgt, mask, [])
        a = quiet.launches
        check_result(quiet.search5(order), want5, what + ("fused",))
        l_fused = quiet.launches - a
        roomy = _fresh(SBG_HITS_CAP=str(ROOMY_WORDS))
        try:
            roomy.load(tabs, tgt, mask, [])
            a = roomy.launches
            check_result(roomy.search5(order), want5, what + ("roomy",))
            l_two = roomy.launches - a
        finally:
            roomy.close()
        assert l_two == l_fused + 1, (what, l_two, l_fused)   # k_decomp5
        eng = _fresh(**env)
        try:
            eng.load(tabs, tgt, mask, [])
            a = eng.launches
            r = eng.search5(order)
            check_result(r, want5, what + ("search5",))
            assert eng.launches - a == l_two + l_fused, (what, eng.launches - a, l_two, l_fused)
            COVER["redo5"] += 1
            if want5 is None:
                assert int(r.tuples_feasible) == feas
        finally:
            eng.close()
        # The chains, against a handle whose 7-LUT stage plans with the same buffer but whose
        # search_5lut is fused: each job's chain makes the k_decomp5 launch more, and on a fallback
        # the fused search_5lut again.  A miss then redoes the 7-LUT stage step by step as well
        # (which the baseline also does when its own phase-1 buffer overflows).
        for path in ("node", "batch"):
            jobs = [dict(slot=s, order5=order, outer=outer, middle=middle) for s in (0, 1)]
            deltas = []
            for e_env in (dict(env, SBG_SEARCH5="fused"), env):
                e = _fresh(**e_env)
                try:
                    e.stage(0, tabs, tgt, mask, [])
                    e.stage(1, tabs, tgt, mask, [])
                    a = e.launches
                    if path == "node":
                        nodes = [e.search_node(**jobs[0])]
                    else:
                        nodes = e.search_batch(jobs)
                    for node in nodes:
                        _check_node(node, want5, want7, what + (path, e_env))
                    deltas.append(e.launches - a)
                finally:
                    e.close()
            redo = len(nodes) * l_two
            if want5 is not None:
                assert deltas[1] == deltas[0] + redo, (what, path, deltas, l_two)
            else:
                assert deltas[1] >= deltas[0] + redo, (what, path, deltas, l_two)
                COVER["redo7"] += 1
            print("overflow %s %s: launches %d with the fallback, %d fused" % (what, path,
                                                                             deltas[1], deltas[0]))
    assert seen_miss


def test_part_fallback_keeps_the_prefix_deal(engines):
    """The two-kernel form at n = 130 under a 1-position mask: every combination is feasible, so
    every part's hit buffer overflows and the part is redone in the fused form.  Its share must
    stay the one the prefix deal gives it (the other parts' shares may come from parts that did
    not overflow), not the chunk head's; a whole search may use the head."""
    rs = np.random.RandomState(9898)
    n = 130
    tabs = S.synthetic_state(n, seed=9899)
    tgt = S.sbox_target(S.rijndael_sbox(), 5)
    order = bytes(rs.permutation(256).astype(np.uint8))
    dense = random_mask(rs, 1)
    two, prefix = engines["two"], engines["prefix"]

    def counted(e, fn):
        a = e.launches
        v = fn()
        return v, e.launches - a
    # launches without a fallback: two kernels under a full mask (next to nothing feasible), and
    # the fused form
    two.load(tabs, tgt, S.mux_mask([]), [])
    _, l_two = counted(two, lambda: two.search5_part(1, 3, order))
    prefix.load(tabs, tgt, dense, [])
    _, l_fused = counted(prefix, lambda: prefix.search5_part(1, 3, order))
    orc = E.Search5Oracle(tabs, tgt, dense, [], order, False)
    head = E.Search5Oracle(tabs, tgt, dense, [], order, True)
    two.load(tabs, tgt, dense, [])
    differ = 0
    for P in (2, 3, 7):
        for p in range(P):
            want = orc.part_key(p, P, LIMIT)
            assert want is not None and want != NONE, (P, p)
            got, launches = counted(two, lambda: two.search5_part(p, P, order))
            assert got == want, (P, p, hex(got), hex(want))
            assert launches == l_two + l_fused, (P, p, launches, l_two, l_fused)
            differ += head.part_key(p, P, LIMIT) != want
            COVER["parts"] += 1
    assert differ >= 6   # the head's deal would have given other keys
    got, launches = counted(two, lambda: int(two.search5(order).key))
    assert got == orc.part_key(0, 1) and launches == l_two + l_fused


def test_coverage_report():
    """What the tests above met (printed; run after them)."""
    print("search_5lut oracle coverage: NW x form %s, (row, NW, form) met %d, rows at NW 1 / 8 "
          "per form %s, max pos_outer %d, max rank %d (2^%.1f), parts compared %d, part sets %s, "
          "search5 overflow redos %d, 7-LUT stage redos %d"
          % (sorted(COVER["nw"]), len(COVER["rows"]),
             {f: [len({r for r, w, g in COVER["rows"] if (w, g) == (nw, f)}) for nw in (1, 8)]
              for f in ("two", "prefix", "head")},
             COVER["pos"], COVER["rank"], np.log2(max(COVER["rank"], 1)), COVER["parts"],
             sorted(COVER["part_sets"], key=str), COVER["redo5"], COVER["redo7"]))
