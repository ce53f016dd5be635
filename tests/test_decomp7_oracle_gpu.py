"""GPU: search_7lut's phase 2 (k_decomp7, sbg_finish7) against the CPU oracle at every mask width.

Each list entry's own first key (decomp7_part(p, L)), every part's key of several shardings, every
ordering row as the first-match row, outer / middle positions at the end of the shuffled orders,
list indices past 2^16, and the full sbg_result through every entry path (sbg_search7,
search_node, search_batch, decomp7_part + finish7 on the finding and on another handle).  Every
comparison runs with the stage-1 filter on and off (SBG_DECOMP_FILTER).  The oracle's keys come
from orc_decomp7_key (tests/_enum_support.py), its results from expected_result7."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200.lut import pack_tuple7, unpack_tuple7
from sboxgates_b200.rng import Xorshift1024

pytestmark = pytest.mark.gpu

NONE = E.NONE
NS = [14, 40, 64, 96, 130, 257, 500]
FIXS = [[], [(7, 1)], [(6, 0), (2, 1)], [(5, 1), (6, 0), (7, 1)]]   # mux masks of depth 0-3
RANDOM_SIZES = [33, 65, 100, 129, 200, 255]
FUNCS = [0x96, 0xE8, 0xCA, 0xD8, 0x1B, 0x6A, 0xB4, 0x78, 0x3C, 0xA6]
ASYM = [0xCA, 0xD8, 0xE4, 0xB4, 0xA6, 0x1B, 0x72, 0x4E, 0x2D, 0x8E]   # no two inputs symmetric


@pytest.fixture(scope="module")
def engines():
    """A default engine and one with the stage-1 filter off."""
    mp = pytest.MonkeyPatch()
    out = {}
    try:
        for f in ("1", "0"):
            mp.setenv("SBG_DECOMP_FILTER", f)
            out[f] = sb.LutEngine(0)
    finally:
        mp.undo()
    yield out
    for e in out.values():
        e.close()


def random_mask(rs, size):
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, size, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def nw_of(mask):
    m = sum(bin(int(w)).count("1") for w in mask)
    return max(1, -(-m // 32))


def to_end(order, funcs, last):
    """The order with `funcs` moved to positions last, last - 1, ..."""
    o = list(order)
    for i, f in enumerate(funcs):
        j, t = o.index(f), last - i
        o[j], o[t] = o[t], o[j]
    return bytes(o)


def packed(tuples):
    return np.array([pack_tuple7(t) for t in tuples], dtype=np.uint64)


def check_result(res, want, what):
    got = E.result7_fields(res)
    assert want is not None, what
    for f, v in want.items():
        assert got[f] == v, (what, f, got[f], v)


COVER = {"nw": set(), "rows": set(), "stale": set(), "po": 0, "pm": 0, "idx": 0, "decided": 0}


def note(key, nw, stale=False):
    if key == NONE:
        return
    COVER["rows"].add((key >> 16) & 0x7F)
    COVER["po"] = max(COVER["po"], (key >> 8) & 0xFF)
    COVER["pm"] = max(COVER["pm"], key & 0xFF)
    COVER["idx"] = max(COVER["idx"], key >> 23)
    if stale:
        COVER["stale"].add(((key >> 16) & 0x7F, nw))


# ------------------------------------------------------------------------------------------------
# a + c: every entry's own key, every part's key

def _entry_cases():
    rs = np.random.RandomState(7070)
    masks = [("mux", f) for f in FIXS] + [("rand", s) for s in RANDOM_SIZES]
    for i, (kind, spec) in enumerate(masks * 2):
        n = NS[i % len(NS)]
        tabs = S.synthetic_state(n, seed=5100 + i)
        mask = S.mux_mask(spec) if kind == "mux" else random_mask(rs, spec)
        P = sorted(int(x) for x in rs.choice(np.arange(1, n), 7, replace=False))
        kind_t = i % 4
        flat = E.stale_pairs(rs, n, 2 if n >= 30 else 1, 256 if n >= 262 else 1)
        pairs = [flat[j:j + 2] for j in range(0, len(flat), 2)]
        if kind_t == 0:
            tgt = E.planted7(tabs, P, int(rs.randint(70)), *rs.choice(FUNCS, 3))
        elif kind_t == 1:
            tgt = S.lut_table(int(rs.choice(FUNCS)), tabs[P[0]], tabs[P[3]], tabs[P[6]])
        elif kind_t == 2:
            tgt = S.lut_table(0xCA, S.lut_table(0x96, tabs[P[1]], tabs[P[2]], tabs[P[4]]),
                              tabs[P[5]], tabs[P[6]])
        else:
            prev, cur = pairs[0]
            tgt = E.planted7(tabs, cur, int(rs.randint(4)), *rs.choice(FUNCS, 3), stale_gate=prev[1])
        tuples = {tuple(P)}
        others = [g for g in range(n) if g not in P]
        for j in range(10):   # neighbours sharing 5-6 gates
            t = list(P)
            for pos in rs.choice(7, 1 + j % 2, replace=False):
                t[pos] = int(rs.choice(others))
            if len(set(t)) == 7:
                tuples.add(tuple(sorted(t)))
        for prev, cur in pairs:
            tuples |= {tuple(prev), tuple(cur)}
        lst = np.array(sorted(tuples), dtype=np.uint16)
        outer, middle = sb.shuffled_orders7(Xorshift1024(rs.bytes(128)))
        yield tabs, tgt, mask, [0] if i % 3 == 0 else [], lst, outer, middle


def test_entry_and_part_keys_match_the_oracle(engines):
    cases = []
    for tabs, tgt, mask, inbits, lst, outer, middle in _entry_cases():
        keys = E.decomp7_entry_keys(tabs, tgt, mask, lst, outer, middle)
        COVER["decided"] += len(lst)
        cases.append((tabs, tgt, mask, inbits, lst, outer, middle, keys))
    assert sum(k != NONE for c in cases for k in c[-1]) >= 2 * len(cases)
    nws = set()
    for f, eng in engines.items():
        for i, (tabs, tgt, mask, inbits, lst, outer, middle, keys) in enumerate(cases):
            nws.add((nw_of(mask), f))
            eng.load(tabs, tgt, mask, inbits)
            eng.set_list7(packed(lst))
            L = len(lst)
            for p in range(L):
                got = eng.decomp7_part(p, L, outer, middle)
                assert got == keys[p], (f, i, p, hex(got), hex(keys[p]))
                note(got, nw_of(mask), E.stale_source(lst, p, (got >> 16) & 0x7F) is not None
                     if got != NONE else False)
            for P in (2, 3, 7, L + 3):
                want = E.part_keys(keys, P)
                for p in range(P):
                    got = eng.decomp7_part(p, P, outer, middle)
                    assert got == want[p], (f, i, P, p, hex(got), hex(want[p]))
    COVER["nw"] |= nws
    assert {nw for nw, _ in nws} >= {1, 2, 3, 4, 5, 7, 8}


# ------------------------------------------------------------------------------------------------
# b: every ordering row first, stale rows at NW 1 and 8, positions at the ends of the orders

def _row_cases():
    rs = np.random.RandomState(7171)
    sizes = [32, 64, 90, 128, 150, 192, 224, 256]   # NW 1..8
    specs = ([(k, sizes[k % 8]) for k in range(70)] + [(k, 256) for k in range(70)] * 2
             + [(11, 256), (11, 224)] * 6   # row 11's circuits often decompose on an earlier row
             + [(k, s) for k in range(4) for s in (32, 256) for _ in range(3)] + [(3, 32)] * 12)
    for i, (k, size) in enumerate(specs):
        n = NS[i % len(NS)]
        tabs = S.synthetic_state(n, seed=5300 + i)
        mask = random_mask(rs, size)
        fo, fm, fi = (int(x) for x in rs.choice(ASYM, 3))
        if i >= 222:   # a stale row: the target runs on the previous entry's outer tables
            prev, cur = E.stale_pairs(rs, n, 1, 256 if n >= 262 else 1)
            tgt = E.planted7(tabs, cur, k, fo, fm, fi, stale_gate=prev[1])
            lst = np.array([prev, cur], dtype=np.uint16)
        else:
            P = sorted(int(x) for x in rs.choice(n, 7, replace=False))
            tgt = E.planted7(tabs, P, k, fo, fm, fi)
            lst = np.array([P], dtype=np.uint16)
        outer, middle = sb.shuffled_orders7(Xorshift1024(rs.bytes(128)))
        if i % 2 == 0:   # the pair's member with bit 7 clear last, its complement before it
            rep = min(fo, 255 - fo)
            outer = to_end(outer, [rep, 255 - rep] if i % 4 == 0 else [255 - rep, rep], 255)
            middle = to_end(middle, [fm, 255 - fm], 255)
        yield tabs, tgt, mask, lst, outer, middle, k


@pytest.fixture(scope="module")
def row_cases():
    out = []
    for tabs, tgt, mask, lst, outer, middle, k in _row_cases():
        keys = E.decomp7_entry_keys(tabs, tgt, mask, lst, outer, middle)
        COVER["decided"] += len(lst)
        out.append((tabs, tgt, mask, lst, outer, middle, k, keys))
    return out


def test_row_cases_cover_every_row_and_the_position_extremes(row_cases):
    rows, stale, po, pm = set(), set(), 0, 0
    for tabs, tgt, mask, lst, outer, middle, k, keys in row_cases:
        for i, key in enumerate(keys):
            if key == NONE:
                continue
            r = (key >> 16) & 0x7F
            rows.add(r)
            po, pm = max(po, (key >> 8) & 0xFF), max(pm, key & 0xFF)
            if E.stale_source(lst, i, r) is not None:
                stale.add((r, nw_of(mask)))
    assert rows == set(range(70)), sorted(set(range(70)) - rows)
    assert {(r, nw) for r in range(4) for nw in (1, 8)} <= stale, sorted(stale)
    assert po >= 250 and pm >= 250, (po, pm)


def test_row_keys_and_results_match_the_oracle(engines, row_cases):
    for f, eng in engines.items():
        for i, (tabs, tgt, mask, lst, outer, middle, k, keys) in enumerate(row_cases):
            eng.load(tabs, tgt, mask, [])
            eng.set_list7(packed(lst))
            L = len(lst)
            for p in range(L):
                got = eng.decomp7_part(p, L, outer, middle)
                assert got == keys[p], (f, i, p, hex(got), hex(keys[p]))
            key = eng.decomp7_part(0, 1, outer, middle)
            assert key == min(keys), (f, i)
            if key != NONE:
                idx = key >> 23
                note(key, nw_of(mask), E.stale_source(lst, idx, (key >> 16) & 0x7F) is not None)
                want = E.expected_result7(key, lst, tabs, tgt, mask, outer, middle)
                check_result(eng.finish7(key, outer, middle), want, (f, i))


# ------------------------------------------------------------------------------------------------
# c: a real capped list, parts of 2-3 entries, indices past 2^16

def test_deep_parts_of_a_capped_list(engines):
    rs = np.random.RandomState(7272)
    n, nparts = 64, 40_000
    tabs = S.synthetic_state(n, seed=5500)
    mask = S.mux_mask([(5, 1), (6, 0), (7, 1)])
    eng = engines["1"]
    eng.load(tabs, S.sbox_target(S.rijndael_sbox(), 3), mask, [])
    base = eng.filter7_part(0, 1)
    assert len(base) == 100_000
    # a circuit planted on a deep entry of that list, which is then decided under the planted
    # target (phase 2 takes any ascending list)
    deep = 88_000
    P = unpack_tuple7(base[deep])
    tgt = E.planted7(tabs, P, 37, 0x96, 0xE8, 0xCA)
    outer, middle = sb.shuffled_orders7(Xorshift1024(rs.bytes(128)))
    for e in engines.values():
        e.load(tabs, tgt, mask, [])
        e.set_list7(base)
    lst = E.unpack_list(base)
    parts = sorted({deep % nparts} | {int(x) for x in rs.choice(20_000, 39, replace=False)})
    oracle = E._List7(tabs, tgt, mask, lst, outer, middle)
    with ThreadPoolExecutor(max_workers=E.workers()) as pool:
        want = list(pool.map(lambda p: oracle.key(p, nparts), parts))
    COVER["decided"] += sum(len(range(p, len(lst), nparts)) for p in parts)
    stale = sum(E.stale_source(lst, i, 0) is not None for p in parts
                for i in range(p, len(lst), nparts))
    print("deep parts: stale entries met %d" % stale)
    assert any(w != NONE and w >> 23 >= 80_000 for w in want)
    for f, e in engines.items():
        for p, w in zip(parts, want):
            got = e.decomp7_part(p, nparts, outer, middle)
            assert got == w, (f, p, hex(got), hex(w))
            note(got, 1)
        w = max(x for x in want if x != NONE)
        check_result(e.finish7(w, outer, middle),
                     E.expected_result7(w, lst, tabs, tgt, mask, outer, middle), f)


# ------------------------------------------------------------------------------------------------
# d: the result through every entry path

def _path_cases():
    rs = np.random.RandomState(7373)
    specs = [(14, 32), (40, 64), (64, 96), (96, 128), (130, 150), (40, 192), (64, 224), (130, 256),
             (24, 100), (96, 33)]
    for i, (n, size) in enumerate(specs):
        tabs = S.synthetic_state(n, seed=5700 + i)
        mask = random_mask(rs, size)
        P = [0, 1, 2, 3, 4, 5, 6 + int(rs.randint(6))]
        tgt = E.planted7(tabs, P, int(rs.randint(70)), *rs.choice(FUNCS, 3))
        yield tabs, tgt, mask, rs.bytes(128)


def test_results_through_every_entry_path(engines):
    cases = []
    for tabs, tgt, mask, seed in _path_cases():
        outer, middle = sb.shuffled_orders7(Xorshift1024(seed))
        lst = E.filter7_range(tabs, tgt, mask, [], 0, 64)   # the list's entries among the first ranks
        key = E.decomp7_key(tabs, tgt, mask, lst, outer, middle)
        assert key != NONE
        COVER["decided"] += (key >> 23) + 1
        want = E.expected_result7(key, lst, tabs, tgt, mask, outer, middle)
        cases.append((tabs, tgt, mask, seed, outer, middle, lst, key, want))
    for f, eng in engines.items():
        other = engines["0" if f == "1" else "1"]
        for i, (tabs, tgt, mask, seed, outer, middle, lst, key, want) in enumerate(cases):
            what = (f, i)
            eng.load(tabs, tgt, mask, [])
            full = eng.filter7_part(0, 1)
            assert np.array_equal(E.unpack_list(full[:len(lst)]), lst), what
            check_result(eng.search7(outer, middle), want, what + ("search7",))
            eng.stage(1, tabs, tgt, mask, [])
            check_result(eng.search_node(1, outer=outer, middle=middle).r7, want, what + ("node",))
            # decomp7_part over 3 parts, the winning part last, then finish7 on this handle (the
            # entries came with the key) and on a handle that found nothing (it reads them)
            eng.load(tabs, tgt, mask, [])
            eng.filter7_part(0, 1)
            win = (key >> 23) % 3
            keys = [eng.decomp7_part(p, 3, outer, middle) for p in [p for p in range(3) if p != win] + [win]]
            assert min(keys) == key == keys[-1], what
            check_result(eng.finish7(key, outer, middle), want, what + ("finish7 here",))
            other.load(tabs, tgt, mask, [])
            other.filter7_part(0, 1)
            other.decomp7_part((win + 1) % 3, 3, outer, middle)
            check_result(other.finish7(key, outer, middle), want, what + ("finish7 elsewhere",))
            note(key, nw_of(mask))
        # search_batch: all states staged, two waves of concurrent chains
        for i, c in enumerate(cases):
            eng.stage(i, c[0], c[1], c[2], [])
        res = eng.search_batch([dict(slot=i, outer=c[4], middle=c[5]) for i, c in enumerate(cases)])
        for i, (r, c) in enumerate(zip(res, cases)):
            check_result(r.r7, c[-1], (f, i, "batch"))
    # search_7lut (ret[10], RNG draws) against the oracle's whole search where n <= 40
    eng = engines["1"]
    for tabs, tgt, mask, seed, *_ in cases:
        if len(tabs) > 40:
            continue
        o_rng = S.OrcRng.from_seed(seed)
        found, ret, _ = S.oracle_search(7, tabs, tgt, mask, [], o_rng)
        g_rng = Xorshift1024(seed)
        res = sb.search_7lut(eng, tabs, tgt, mask, [], g_rng)
        assert found and (res.found, res.ret) == (found, ret)
        assert g_rng.draws == o_rng.draws


# ------------------------------------------------------------------------------------------------
# e: finish7 after the list changed

def _state_b(rs, first, outer, middle):
    """A state whose key is 0: its list's entry `first` realises the target on row 0 with the
    first functions of both orders."""
    n = 30
    tabs = S.synthetic_state(n, seed=5900)
    tgt = E.planted7(tabs, first, 0, outer[0], middle[0], 0xCA)
    return tabs, tgt, np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)


@pytest.mark.parametrize("change", ["set_list7", "use_problem", "filter7_part"])
def test_finish7_after_the_list_changed(engines, change):
    rs = np.random.RandomState(7474)
    outer, middle = sb.shuffled_orders7(Xorshift1024(rs.bytes(128)))
    b_first = [0, 1, 2, 3, 4, 5, 6]   # entry 0 of B's phase-1 list under a full mask
    tabs_b, tgt_b, mask_b = _state_b(rs, b_first, outer, middle)
    list_b = [b_first, [0, 1, 2, 3, 4, 5, 9], [2, 4, 8, 11, 13, 20, 21]]
    for f, eng in engines.items():
        # list A under an empty mask: its first entry matches at once, key 0
        tabs_a = S.synthetic_state(24, seed=5901)
        list_a = np.array([[3, 5, 9, 11, 12, 13, 14], [4, 6, 7, 8, 10, 15, 16]], dtype=np.uint16)
        eng.load(tabs_a, tgt_b, np.zeros(4, dtype=np.uint64), [])
        eng.set_list7(packed(list_a))
        assert eng.decomp7_part(0, 1, outer, middle) == 0
        if change == "set_list7":
            eng.load(tabs_b, tgt_b, mask_b, [])
            eng.set_list7(packed(list_b))
            lst = np.array(list_b, dtype=np.uint16)
        elif change == "use_problem":
            eng.stage(3, tabs_b, tgt_b, mask_b, [])
            eng.use(3)
            eng.set_list7(packed(list_b))
            lst = np.array(list_b, dtype=np.uint16)
        else:
            eng.load(tabs_b, tgt_b, mask_b, [])
            lst = E.unpack_list(eng.filter7_part(0, 1))
            assert list(lst[0]) == b_first
        want = E.expected_result7(0, lst, tabs_b, tgt_b, mask_b, outer, middle)
        check_result(eng.finish7(0, outer, middle), want, (f, change))


def test_coverage_report():
    """What the tests above met (printed; run after them)."""
    print("phase-2 oracle coverage: NW x filter %s, rows hit %d, stale (row, NW) %s, max po %d, "
          "max pm %d, max idx %d, entries decided by the oracle %d"
          % (sorted(COVER["nw"]), len(COVER["rows"]), sorted(COVER["stale"]), COVER["po"],
             COVER["pm"], COVER["idx"], COVER["decided"]))
