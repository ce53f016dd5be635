"""CPU: the host reference of the enumerations (tests/_enum_reference.py) against the oracle it
stands in for -- orc_solve_inner, orc_lut_ttable, expected_record, record_depths,
match_functions_allowed, match_group, the deal of Deal5 -- and the seeded generator of
test_enum_fuzz_gpu.py: deterministic, and covering what its coverage test asserts."""
import collections
from math import comb

import numpy as np
import pytest

import _enum_reference as R
import _enum_support as E
import _support as S
import sboxgates_b200 as sb
import test_enum_fuzz_gpu as FZ
from test_enum_depth_gpu import _nw

MASK_POSITIONS = (0, 1, 31, 32, 33, 255, 256)


def _mask(rs, count):
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, count, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def _triples(rs, count):
    """Random (x, y, z, target, mask) rows, a third of them degenerate: constant tables, equal or
    complementary inputs, an input equal to the target or its complement."""
    rnd = lambda: rs.randint(0, 2**63, (count, 4)).astype(np.uint64) * np.uint64(2) \
        + rs.randint(0, 2, (count, 4)).astype(np.uint64)   # noqa: E731
    x, y, z, tgt = rnd(), rnd(), rnd(), rnd()
    for j in range(count):
        kind = j % 9
        if kind == 1:
            x[j] = 0
        elif kind == 2:
            y[j] = R.ONES
        elif kind == 3:
            y[j] = x[j]
        elif kind == 4:
            z[j] = ~x[j]
        elif kind == 5:
            z[j] = tgt[j]
        elif kind == 6:
            x[j], y[j] = ~tgt[j], tgt[j]
    mask = np.stack([_mask(rs, MASK_POSITIONS[j % len(MASK_POSITIONS)]) for j in range(count)])
    return x, y, z, tgt, mask


def test_solve_inner_matches_the_oracle():
    rs = np.random.RandomState(1)
    x, y, z, tgt, mask = _triples(rs, 10_000)
    ok, fi, seen = R.solve_inner(x, y, z, tgt, mask)
    counts = collections.Counter()
    for j in range(len(x)):
        want = R.solve_inner_oracle(x[j], y[j], z[j], tgt[j], mask[j])
        got = (bool(ok[j]), int(fi[j]), int(seen[j])) if ok[j] else (False,)
        assert got == (want if want[0] else (False,)), j
        counts[want[0]] += 1
    assert counts[True] > 1000 and counts[False] > 1000


def test_lut_tables_match_the_oracle():
    rs = np.random.RandomState(2)
    x, y, z, _, _ = _triples(rs, 600)
    f = rs.randint(0, 256, 600)
    got = R.lut_tables(f, x, y, z)
    for j in range(600):
        assert np.array_equal(got[j], S.lut_table(int(f[j]), x[j], y[j], z[j])), j


def _small_state(width, seed, mask_count):
    rs = np.random.RandomState(seed)
    n = {3: 24, 5: 10, 7: 10}[width]
    tabs = S.synthetic_state(n, seed=seed)
    tgt, g = FZ._planted(rs, tabs, width, list(range(n)))
    tabs[int(rs.choice([x for x in range(n) if x not in g]))] = ~tgt   # a degenerate gate
    mask = S.mux_mask([(1, 1), (4, 0), (6, 1)]) if mask_count is None else _mask(rs, mask_count)
    order, outer, middle = E.orders(seed)
    orders = {3: (rs.permutation(n).astype(np.uint16),), 5: (order,), 7: (outer, middle)}[width]
    tuples = None
    if width == 7:
        full = E.filter7_range(tabs, tgt, mask, [], 0, comb(n, 7))
        tuples = full[:3]
    return tabs, tgt, mask, orders, tuples


@pytest.mark.parametrize("width", [3, 5, 7])
@pytest.mark.parametrize("mask_count", [None, 33, 200])
def test_records_match_expected_record(width, mask_count):
    tabs, tgt, mask, orders, tuples = _small_state(width, 40 + width, mask_count)
    ref = R.Reference(width, tabs, tgt, mask, [], orders, tuples)
    assert ref.total > 0
    step = max(1, len(ref.all) // 400)
    for rec in ref.all[::step]:
        key = int(rec["key"])
        if width == 3:
            i, k, m = sb.decode_key3(key)
            g = [int(orders[0][x]) for x in (i, k, m)]
            ok, fi, seen = R.solve_inner_oracle(*[tabs[x] for x in g], tgt, mask)
            assert ok and E.record_fields(rec) == (g, 0, 0, fi, seen), hex(key)
        else:
            want = E.expected_record(width, key, tabs, tgt, mask, orders[0],
                                     orders[1] if width == 7 else None,
                                     tuples[key >> 23] if width == 7 else None)
            assert want is not None and E.record_fields(rec) == want, hex(key)
        assert int(rec["width"]) == width and not rec["pad"].any()
        assert not rec["gates"][width:].any()
    assert R.check_realises(ref.all, tabs, tgt, mask) == len(ref.all)


def test_check_realises_rejects_a_wrong_field():
    tabs, tgt, mask, orders, tuples = _small_state(7, 47, None)
    ref = R.Reference(7, tabs, tgt, mask, [], orders, tuples)
    good = ref.all[:50].copy()
    R.check_realises(good, tabs, tgt, mask)
    for field, change in (("inner_seen", lambda v: v ^ 0x10), ("func_inner", lambda v: v ^ 0x01),
                          ("width", lambda v: 5), ("pad", lambda v: v + 1)):
        bad = good.copy()
        j = int(np.flatnonzero(bad["inner_seen"] & 1)[0]) if field == "func_inner" else 7
        bad[field][j] = change(bad[field][j])
        with pytest.raises(AssertionError):
            R.check_realises(bad, tabs, tgt, mask)


@pytest.mark.parametrize("width", [3, 5, 7])
def test_selection_matches_the_library_helpers(width):
    tabs, tgt, mask, orders, tuples = _small_state(width, 40 + width, None)
    ref = R.Reference(width, tabs, tgt, mask, [], orders, tuples)
    rs = np.random.RandomState(width)
    depth = rs.randint(0, 9, len(tabs)).astype(np.uint16)
    dep = E.record_depths(ref.all, depth)
    half = sorted(int(x) for x in rs.choice(256, 128, replace=False))
    sets = (half, sorted(sb.AFFINE_FUNCTIONS), sorted(sb.gate_functions(194)))
    ok = R.function_ok(ref.all, *sets)
    step = max(1, len(ref.all) // 300)
    for j in range(0, len(ref.all), step):
        rec = ref.all[j]
        assert dep[j] == sb.match_depth(rec, depth)
        assert ok[j] == sb.match_functions_allowed(rec, *sets)
    for grouping in (None, "shape", "tuple"):
        ids = R.group_ids(ref.all["key"], width, grouping)
        for j in range(0, len(ref.all), step):
            assert int(ids[j]) == sb.match_group(int(ref.all["key"][j]), width, grouping)
        bound = int(np.median(dep))
        ref.select(depth, bound, *sets, grouping=grouping, functions=True)
        keep = (dep <= bound) & ok
        sub = ref.all[keep]
        seen, want = set(), []
        for rec in sub:
            gid = sb.match_group(int(rec["key"]), width, grouping)
            if gid not in seen:
                seen.add(gid)
                want.append(rec)
        assert ref.recs.tobytes() == np.array(want, dtype=sb.MATCH_DTYPE).tobytes()
        assert np.array_equal(ref.hist, R.histogram(E.record_depths(ref.recs, depth)))
        # the shares partition the selection, and their block sums add up to it
        for nparts in (1, 2, 3, 5):
            parts = [ref.share(q, nparts) for q in range(nparts)]
            merged = np.sort(np.concatenate(parts), order="key")
            assert merged.tobytes() == ref.recs.tobytes()
            for q in range(nparts):
                assert int(ref.share_sums(q, nparts).sum()) == len(parts[q])


def test_ticket_items_follow_the_deal():
    """5-LUT: a key's 3-gate prefix is the deal item whose rank range (Deal5 without the fused
    head) holds the key's combination; 3-LUT: the position pair's lexicographic rank."""
    n = 13
    deal = E.Deal5(n, [], head=False)
    ranks = np.arange(comb(n, 5), dtype=np.uint64)
    items = R.ticket_items(5, ranks << np.uint64(12), n)
    for j in range(deal.blocks()):
        for lo, hi in deal.block_ranges(j):
            assert (items[lo:hi] // R.KDEAL == j).all(), j
    pairs = [(i, k) for i in range(n) for k in range(i + 1, n)]
    keys = np.array([i << 18 | k << 9 | (k + 1) for i, k in pairs], dtype=np.uint64)
    assert R.ticket_items(3, keys, n).tolist() == list(range(len(pairs)))
    assert R.item_count(3, n) == len(pairs) and R.item_count(5, n) == comb(n - 2, 3)


def test_generator_is_deterministic():
    for seed in FZ.SEEDS:
        for idx in (0, 7, FZ.CONFIGS - 1):
            a, b = FZ.Config(seed, idx), FZ.Config(seed, idx)
            assert a.tag() == b.tag()
            assert a.tables.tobytes() == b.tables.tobytes()
            assert a.target.tobytes() == b.target.tobytes() and a.mask.tobytes() == b.mask.tobytes()
            assert [bytes(o) for o in a.orders] == [bytes(o) for o in b.orders]
            assert a.gate_depth.tobytes() == b.gate_depth.tobytes()
            assert FZ.Config(seed, idx, 1).tag() != a.tag()


def test_generator_covers_the_matrix():
    """Per seed: every (width, NW, form) the kernels have; every pair of settings and all three
    with a restricted inner set at widths 5 and 7; shares with every form; degenerate tables;
    random masks whose last 32-bit word is partly padding at every width; 3-LUT states at
    n >= 255."""
    for seed in FZ.SEEDS:
        cfgs = FZ.configs(seed)
        forms = {(c.width, c.nw, c.form) for c in cfgs}
        assert forms == {(w, nw, f) for w in (3, 5, 7) for nw in FZ.NWS for f in FZ.FORMS
                         if not (w == 3 and f == "grouped")}, seed
        assert all(_nw(c.mask) == c.nw for c in cfgs)
        assert {c.form for c in cfgs if c.nparts > 1} == set(FZ.FORMS), seed
        assert any(c.degenerate for c in cfgs), seed
    cfgs = [c for seed in FZ.SEEDS for c in FZ.configs(seed)]
    for w in (5, 7):
        mine = [c for c in cfgs if c.width == w]
        g = lambda c: c.grouping is not None   # noqa: E731
        assert any(c.depth and c.functions for c in mine), w
        assert any(c.depth and g(c) for c in mine), w
        assert any(c.functions and g(c) for c in mine), w
        assert any(c.depth and c.inner_restricted and g(c) for c in mine), w
    for w in (3, 5, 7):
        padded = [c for c in cfgs if c.width == w and c.mask_spec.startswith("r")
                  and int(c.mask_spec[1:]) % 32 != 0]
        assert padded, w
    assert any(c.width == 3 and c.n >= 255 for c in cfgs)
    assert sum(bool(c.degenerate) for c in cfgs) >= 20
    assert {c.nparts for c in cfgs} == {1, 2, 3, 5}
    kinds = {k for c in cfgs if c.functions for k in c.roles}
    assert kinds == set(FZ.ROLE_KINDS)
