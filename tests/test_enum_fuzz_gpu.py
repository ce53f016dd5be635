"""GPU: seeded differential test of the enumerations against the host reference
(tests/_enum_reference.py), which builds every expected record from the CPU oracle's keys alone.

Each configuration draws a state (width, n, mask, excluded input bits, gate tables with injected
degenerate gates, target, and for width 7 a short list cut from the phase-1 list) and settings
(any subset of the depth filter, the function filter and a grouping; a sharding into 1, 2, 3 or 5
parts).  Then the total, feasible count, depth histogram, first K counted and count-free, pages,
picks and samples, and on global shares each share's total and block sums and the shares' summed
fetches and picks, are compared byte for byte with the reference.  The configurations are
stratified so that every seed meets every (width, words per table, kernel form); configurations
with more than 2^20 matches are drawn again.  test_coverage_report prints what the run met."""
import collections
import functools
from math import comb

import numpy as np
import pytest

import _enum_reference as R
import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import lut
from test_enum_depth_gpu import _nw

pytestmark = pytest.mark.gpu

SEEDS = (101, 202, 303)
CONFIGS = 40
NWS = (1, 2, 4, 8)
FORMS = ("plain", "filtered", "grouped")
MODES = ("count", "first", "free", "page", "pick", "sample", "share", "global")
MUX = {8: [], 4: [(3, 1)], 2: [(0, 0), (5, 1)], 1: [(1, 1), (4, 0), (6, 1)]}
# random mask sizes per words per table: the first (last) sizes of each give a partly padded last
# 32-bit word
RANDOM_POSITIONS = {1: [(1, 3), (31, 32)], 2: [(33, 33), (63, 64)], 4: [(65, 65), (127, 128)],
                    8: [(129, 129), (200, 256)]}
ROLE_KINDS = ("none", "half", "affine", "gates194", "single", "empty")
ROLE_P = (0.3, 0.2, 0.15, 0.15, 0.15, 0.05)
DEGENERATE = ("duplicate", "complement", "zero", "one", "target", "not_target")


@functools.lru_cache(maxsize=1)
def _sbox():
    return S.rijndael_sbox()


def _random_mask(rs, count):
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, count, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def _planted(rs, tabs, width, allowed):
    """A random width-3, 5 or 7 LUT circuit of allowed gates: (target, its gates)."""
    g = [int(x) for x in rs.choice(allowed, width, replace=False)]
    f = [int(x) for x in rs.randint(1, 255, 3)]
    if width == 3:
        return S.lut_table(f[0], *[tabs[x] for x in g]), g
    outer = S.lut_table(f[0], tabs[g[0]], tabs[g[1]], tabs[g[2]])
    mid = tabs[g[3]] if width == 5 else S.lut_table(f[1], tabs[g[3]], tabs[g[4]], tabs[g[5]])
    return S.lut_table(f[2], outer, mid, tabs[g[-1]]), g


class Config:
    """One drawn configuration.  width, NW and form stratum follow from (seed, idx); the rest is
    drawn from RandomState((seed, idx, attempt)), attempt > 0 after a redraw."""

    def __init__(self, seed, idx, attempt=0):
        self.seed, self.idx, self.attempt = seed, idx, attempt
        rs = self.rs = np.random.RandomState([seed, idx, attempt])
        j = idx // 3
        self.width = (3, 5, 7)[(idx + seed) % 3]
        self.nw = NWS[(j + seed) % 4]
        stratum = (j // 4 + seed) % 3
        w = self.width
        # state
        if w == 3:
            self.n = int(rs.randint(255, 501)) if self.nw == 1 and rs.rand() < 0.3 \
                else int(rs.randint(8, 65))
        else:
            self.n = int(rs.randint(7, 23)) if w == 5 else int(rs.randint(8, 15))
        n = self.n
        if rs.rand() < 0.4 or (w == 3 and n > 64):
            self.mask_spec = "mux%d" % {8: 0, 4: 1, 2: 2, 1: 3}[self.nw]
            self.mask = S.mux_mask(MUX[self.nw])
        else:
            lo, hi = RANDOM_POSITIONS[self.nw][int(rs.randint(2))]
            if w == 3 and n > 64:
                lo, hi = max(lo, 31), max(hi, 31)
            count = int(rs.randint(lo, hi + 1))
            self.mask_spec = "r%d" % count
            self.mask = _random_mask(rs, count)
        assert _nw(self.mask) == self.nw, (self.mask_spec, self.nw)
        size = int(rs.randint(0, 5))
        self.inbits = sorted(int(x) for x in rs.choice(8, size, replace=False))
        if size and rs.rand() < 0.4 and 0 not in self.inbits:
            self.inbits[0] = 0
            self.inbits = sorted(set(self.inbits))
        allowed = [g for g in range(n) if w == 3 or g not in self.inbits]
        tabs = S.synthetic_state(n, seed=int(rs.randint(1 << 30)))
        kind = rs.choice(["own", "other", "sbox", "random"], p=[0.7, 0.1, 0.1, 0.1])
        self.planted = []
        if kind == "own" or kind == "other":
            pw = w if kind == "own" else int(rs.choice([x for x in (3, 5, 7) if x != w]))
            if len(allowed) >= pw:
                tgt, self.planted = _planted(rs, tabs, pw, allowed)
            else:
                kind = "random"
        if kind == "sbox":
            tgt = S.sbox_target(_sbox(), int(rs.randint(8)))
        elif kind == "random":
            tgt = rs.randint(0, 2**63, 4).astype(np.uint64) * np.uint64(2) \
                + rs.randint(0, 2, 4).astype(np.uint64)
        self.target_kind = str(kind)
        # degenerate gates: past the input bits, never one the planted circuit uses
        self.degenerate = []
        free = [g for g in range(8, n) if g not in self.planted]
        if rs.rand() < 0.4 and free:
            for g in rs.choice(free, min(len(free), int(rs.randint(1, 5))), replace=False):
                d = str(rs.choice(DEGENERATE))
                src = int(rs.randint(n))
                tabs[g] = {"duplicate": tabs[src], "complement": ~tabs[src],
                           "zero": np.zeros(4, dtype=np.uint64), "one": np.full(4, R.ONES),
                           "target": tgt, "not_target": ~tgt}[d]
                self.degenerate.append((int(g), d))
        self.tables, self.target = tabs, tgt
        # orders
        self.orders = {3: (rs.permutation(n).astype(np.uint16),),
                       5: (bytes(rs.permutation(256).astype(np.uint8)),),
                       7: (bytes(rs.permutation(256).astype(np.uint8)),
                           bytes(rs.permutation(256).astype(np.uint8)))}[w]
        self.list_size = int(rs.randint(1, 5))
        # settings kinds: the stratum fixes the form; width 3 has no grouped form, so there its
        # stratum 2 installs a grouping (which width 3 ignores) over the filtered form
        self.depth = self.functions = False
        self.grouping = None
        if stratum == 1 or (stratum == 2 and w == 3):
            r = int(rs.randint(3))
            self.depth, self.functions = r != 1, r != 0
            if stratum == 2:
                self.grouping = str(rs.choice(["shape", "tuple"]))
        elif stratum == 2:
            self.grouping = str(rs.choice(["shape", "tuple"]))
            self.depth, self.functions = bool(rs.rand() < 0.6), bool(rs.rand() < 0.6)
        elif w == 3 and rs.rand() < 0.3:
            self.grouping = "tuple"
        self.roles = None
        if self.functions:
            self.roles = [str(rs.choice(ROLE_KINDS, p=ROLE_P)) for _ in range(3)]
            restricted_inner = self.depth and self.grouping is not None and rs.rand() < 0.7
            if restricted_inner and self.roles[2] == "none":
                self.roles[2] = str(rs.choice(["half", "affine", "gates194", "single"]))
            elif self.grouping is not None and w == 7 and rs.rand() < 0.6:
                # one middle function and every inner one: the grouped count's fast path, where
                # most list entries hold matches but none with that middle LUT
                self.roles[1], self.roles[2] = "single", "none"
            active = (0, 1, 2) if w == 7 else (0, 2) if w == 5 else (2,)
            if all(self.roles[r] == "none" for r in active):
                self.roles[active[int(rs.randint(len(active)))]] = "half"
        self.gate_depth = rs.randint(0, 9, n).astype(np.uint16)
        self.bound_kind = str(rs.choice(["quantile", "zero", "max"], p=[0.75, 0.1, 0.15]))
        self.nparts = int(rs.choice([1, 2, 3, 5], p=[0.3, 0.25, 0.25, 0.2]))

    @property
    def form(self):
        """The kernel form the settings select (sbg_api.cu: grouping at width 5 / 7 -> grouped,
        else any filter -> filtered, else plain)."""
        if self.grouping is not None and self.width != 3:
            return "grouped"
        return "filtered" if self.depth or self.functions else "plain"

    @property
    def inner_restricted(self):
        return self.functions and self.roles[2] != "none"

    def tag(self):
        return ("seed %d config %d attempt %d: width %d n %d mask %s inbits %s target %s degenerate "
                "%s depth %s functions %s grouping %s nparts %d" % (
                    self.seed, self.idx, self.attempt, self.width, self.n, self.mask_spec,
                    self.inbits, self.target_kind, self.degenerate, self.depth and self.bound_kind,
                    self.roles, self.grouping, self.nparts))

    def pick_list(self, full):
        """The 1-4 list entries (width 7) cut from the phase-1 list `full` ((count, 7)): the planted
        tuple's entry when there is one, the rest at random; in list order."""
        if len(full) == 0:
            return full
        rs = self.rs
        chosen = set(int(x) for x in rs.choice(len(full), min(self.list_size, len(full)),
                                               replace=False))
        if len(self.planted) == 7:
            hit = np.flatnonzero((full == np.array(sorted(self.planted))).all(axis=1))
            if hit.size:
                chosen = set(sorted(chosen)[:-1]) | {int(hit[0])}
        return full[sorted(chosen)]

    def settings(self, ref):
        """The concrete settings, some of them from the unfiltered reference records (a bound at a
        quantile of their depths, a single function taken from a match): a dict for apply()."""
        rs = self.rs
        out = dict(depth=None, bound=None, roles=(None, None, None), grouping=self.grouping)
        if self.depth:
            dep = E.record_depths(ref.all, self.gate_depth)
            if self.bound_kind == "zero":
                bound = 0
            elif self.bound_kind == "max" or len(dep) == 0:
                bound = sb.SBG_DEPTH_BINS - 1
            else:
                bound = int(np.quantile(dep, rs.rand()))
            out["depth"], out["bound"] = self.gate_depth, bound
        if self.functions:
            pick = ref.all[int(rs.randint(len(ref.all)))] if len(ref.all) else None
            out["roles"] = tuple(self._role(kind, r, pick) for r, kind in enumerate(self.roles))
        return out

    def _role(self, kind, r, pick):
        """One role's function set: None (all 256), a random half, the affine functions, AND / OR /
        XOR (gate_functions(194)), the one function a match has in that role, or empty."""
        if kind == "single" and pick is None:
            kind = "affine"
        if kind == "none":
            return None
        if kind == "half":
            return sorted(int(x) for x in self.rs.choice(256, 128, replace=False))
        if kind == "affine":
            return sorted(sb.AFFINE_FUNCTIONS)
        if kind == "gates194":
            return sorted(sb.gate_functions(194))
        if kind == "single":
            return [[int(pick["func_outer"]), int(pick["func_middle"]),
                     sb.allowed_fill(pick["func_inner"], pick["inner_seen"])][r]]
        return []


def configs(seed):
    return [Config(seed, i) for i in range(CONFIGS)]


# ------------------------------------------------------------------------------------------------

STATS = {}   # seed -> Counter of what its run met


def _apply(eng, cfg, st, tuples):
    eng.load(cfg.tables, cfg.target, cfg.mask, cfg.inbits)
    if cfg.width == 7:
        eng.set_list7(np.array([lut.pack_tuple7(t) for t in tuples], dtype=np.uint64))
    if st["depth"] is not None:
        eng.set_depth_filter(st["depth"], st["bound"])
    else:
        eng.clear_depth_filter()
    if any(s is not None for s in st["roles"]):
        eng.set_function_filter(*st["roles"])
    else:
        eng.clear_function_filter()
    eng.set_grouping(st["grouping"])


def _reset(eng):
    eng.set_grouping(None)
    eng.clear_function_filter()
    eng.clear_depth_filter()


def _run(eng, cfg, k, count=True, part=0, nparts=1):
    fn = {3: eng.enumerate3, 5: eng.enumerate5, 7: eng.enumerate7}[cfg.width]
    return fn(*cfg.orders, k, count, part, nparts)


class _Checker:
    """Byte-for-byte comparisons against the reference, counted."""

    def __init__(self, cfg, stats):
        self.cfg, self.stats, self.tag = cfg, stats, cfg.tag()

    def same(self, got, want, mode, what):
        assert got.dtype == sb.MATCH_DTYPE and len(got) == len(want), \
            (self.tag, what, len(got), len(want))
        if got.tobytes() != want.tobytes():
            bad = int(np.flatnonzero(got.view(np.uint64).reshape(len(got), -1)
                                     != want.view(np.uint64).reshape(len(want), -1))[0] // 4)
            raise AssertionError("%s: %s: record %d differs: got %s, want %s"
                                 % (self.tag, what, bad, got[bad], want[bad]))
        self.stats["records"] += len(got)
        if len(got):
            self.stats[(self.cfg.width, self.cfg.nw, self.cfg.form, mode)] += 1


def _cut(rs, total, seams):
    """(first, count) pages: the start, random ranks, ticket seams and the end."""
    pages = [(0, int(rs.randint(1, 200)))]
    for r in rs.randint(0, max(total, 1), 3):
        pages.append((int(r), int(rs.randint(1, 300))))
    for s in rs.choice(seams, min(len(seams), 3), replace=False) if len(seams) else []:
        pages.append((max(int(s) - int(rs.randint(0, 3)), 0), int(rs.randint(2, 40))))
    pages += [(max(total - 5, 0), 10), (total, 4)]
    return pages


def _run_config(engine, shares, cfg, stats):
    w = cfg.width
    tuples = None
    if w == 7:
        engine.load(cfg.tables, cfg.target, cfg.mask, cfg.inbits)
        full = E.unpack_list(engine.filter7_part(0, 1))
        want_list = E.filter7_range(cfg.tables, cfg.target, cfg.mask, cfg.inbits, 0,
                                    comb(cfg.n, 7))
        assert np.array_equal(full, want_list), (cfg.tag(), "phase-1 list")
        tuples = cfg.pick_list(full)
    total, keys, feasible = R.oracle_keys(w, cfg.tables, cfg.target, cfg.mask, cfg.inbits,
                                          cfg.orders, tuples)
    if keys is None:
        return False
    ref = R.Reference(w, cfg.tables, cfg.target, cfg.mask, cfg.inbits, cfg.orders, tuples,
                      keys=keys, feasible=feasible)
    st = cfg.settings(ref)
    o, m, i = st["roles"]
    ref.select(st["depth"], st["bound"], o, m, i, st["grouping"],
               functions=any(s is not None for s in st["roles"]))
    want, t = ref.recs, ref.total
    chk = _Checker(cfg, stats)
    tag = chk.tag
    rs = np.random.RandomState([cfg.seed, cfg.idx, cfg.attempt, 99])
    _apply(engine, cfg, st, tuples)
    # count and first K, counted and count-free
    for k in sorted({0, 1, int(rs.randint(0, t + 2)), t, t + 1}):
        e = _run(engine, cfg, k)
        assert (e.total, e.feasible) == (t, ref.feasible), (tag, k, e.total, t, e.feasible,
                                                            ref.feasible)
        chk.same(e.matches, want[:k], "first", "first %d" % k)
        if st["depth"] is not None:
            assert np.array_equal(engine.depth_counts(), ref.hist), (tag, "depth_counts")
        f = _run(engine, cfg, k, count=False)
        assert f.total is None, tag
        chk.same(f.matches, want[:k], "free", "count-free first %d" % k)
    stats[(w, cfg.nw, cfg.form, "count")] += 1
    # pages, picks and a sample on the cursor of a counted enumeration
    e = _run(engine, cfg, 0)
    for first, count in _cut(rs, t, ref.seams()):
        chk.same(engine.fetch_matches(first, count), want[first:first + count], "page",
                 "page (%d, %d)" % (first, count))
    if t:
        ranks = rs.randint(0, t, int(rs.randint(1, 400)))
        ranks = np.concatenate([ranks, ranks[:int(rs.randint(0, len(ranks) + 1))], [t - 1, 0]])
        rs.shuffle(ranks)
        chk.same(engine.pick_matches(ranks), want[ranks], "pick", "pick")
        r, got = sb.sample_matches(engine, e, min(t, int(rs.randint(1, 200))), seed=cfg.idx)
        chk.same(got, want[r.astype(np.int64)], "sample", "sample")
    if cfg.nparts > 1:
        _check_shares(shares[:cfg.nparts], cfg, st, tuples, ref, chk, rs)
    stats["configs"] += 1
    stats["matches"] += len(ref.all) > 0
    stats[("pair", cfg.depth, cfg.functions, cfg.grouping is not None and w != 3)] += 1
    if cfg.depth and cfg.inner_restricted and cfg.grouping is not None and w != 3:
        stats["all_three_inner"] += 1
    if cfg.degenerate and len(ref.all):
        stats["degenerate_with_matches"] += 1
    if w == 3 and cfg.n > 64 and len(ref.all):
        stats["large_n3_with_matches"] += 1
    return True


def _check_shares(engs, cfg, st, tuples, ref, chk, rs):
    P = len(engs)
    tag, want, t = chk.tag, ref.recs, ref.total
    counts = []
    for q, eng in enumerate(engs):
        _apply(eng, cfg, st, tuples)
        mine = ref.share(q, P)
        k = min(len(mine), int(rs.randint(0, 300)))
        e = _run(eng, cfg, k, True, q, P)
        assert e.total == len(mine), (tag, "share", q, P, e.total, len(mine))
        chk.same(e.matches, mine[:k], "share", "share %d/%d first %d" % (q, P, k))
        f = _run(eng, cfg, k, False, q, P)
        chk.same(f.matches, mine[:k], "share", "share %d/%d count-free first %d" % (q, P, k))
        e = _run(eng, cfg, 0, True, q, P)
        sums = eng.enum_block_sums()
        assert sums.tobytes() == ref.share_sums(q, P).tobytes(), (tag, "block sums", q, P)
        counts.append(len(sums))
    sums = np.zeros((P, max(max(counts), 1)), dtype=np.uint64)
    for q, eng in enumerate(engs):
        sums[q, :counts[q]] = ref.share_sums(q, P)
    assert [eng.enum_set_global(sums, counts) for eng in engs] == [t] * P, (tag, "global total")
    for first, count in _cut(rs, t, ref.seams())[:4]:
        got = sum(eng.fetch_matches(first, count).view(np.uint64) for eng in engs)
        chk.same(got.view(sb.MATCH_DTYPE).reshape(-1), want[first:first + count], "global",
                 "global page (%d, %d)" % (first, count))
    if t:
        ranks = rs.randint(0, t, int(rs.randint(1, 300)))
        got = sum(eng.pick_matches(ranks).view(np.uint64) for eng in engs)
        chk.same(got.view(sb.MATCH_DTYPE).reshape(-1), want[ranks], "global", "global pick")
        whole = sb.Enumeration(t, ref.feasible, want[:0])
        k = min(t, 50)
        parts = [sb.sample_matches(eng, whole, k, seed=cfg.idx) for eng in engs]
        got = sum(p[1].view(np.uint64) for p in parts)
        chk.same(got.view(sb.MATCH_DTYPE).reshape(-1), want[parts[0][0].astype(np.int64)],
                 "global", "global sample")
    for eng in engs:
        _reset(eng)


def _run_seed(engine, shares, seed):
    if seed in STATS:
        return STATS[seed]
    stats = collections.Counter()
    try:
        for idx in range(CONFIGS):
            for attempt in range(20):
                cfg = Config(seed, idx, attempt)
                if _run_config(engine, shares, cfg, stats):
                    break
                stats["redrawn"] += 1
            else:
                raise AssertionError("seed %d config %d: every draw exceeded %d matches"
                                     % (seed, idx, R.CAP))
    finally:
        _reset(engine)
    STATS[seed] = stats
    return stats


@pytest.fixture(scope="module")
def shares():
    engs = [sb.LutEngine(0) for _ in range(5)]
    yield engs
    for e in engs:
        e.close()


@pytest.mark.parametrize("seed", SEEDS)
def test_random_configurations_match_the_reference(engine, shares, seed):
    _run_seed(engine, shares, seed)


def test_coverage_report(engine, shares):
    total = collections.Counter()
    for seed in SEEDS:
        total.update(_run_seed(engine, shares, seed))
    cells = [(w, nw, f) for w in (3, 5, 7) for nw in NWS for f in FORMS
             if not (w == 3 and f == "grouped")]
    print("\nenumeration fuzz: %d configurations (%d redrawn above %d matches), %d records compared"
          % (total["configs"], total["redrawn"], R.CAP, total["records"]))
    for w, nw, f in cells:
        print("  width %d NW %d %-8s %s" % (w, nw, f, " ".join(
            "%s=%d" % (m, total[(w, nw, f, m)]) for m in MODES)))
    for key in sorted(k for k in total if isinstance(k, tuple) and k[0] == "pair"):
        print("  settings depth=%s functions=%s grouping=%s: %d" % (key[1], key[2], key[3],
                                                                     total[key]))
    for key in ("all_three_inner", "degenerate_with_matches", "large_n3_with_matches", "matches"):
        print("  %s: %d" % (key, total[key]))
    for w, nw, f in cells:
        for m in ("count", "first", "free", "page", "pick", "sample"):
            assert total[(w, nw, f, m)] > 0, (w, nw, f, m)
    for f in FORMS:
        assert sum(total[(w, nw, f, m)] for w in (3, 5, 7) for nw in NWS
                   for m in ("share", "global")) > 0, f
    for d, fn, g in ((True, True, False), (True, False, True), (False, True, True),
                     (True, True, True)):
        assert total[("pair", d, fn, g)] > 0, (d, fn, g)
    assert total["all_three_inner"] > 0
    assert total["degenerate_with_matches"] >= 10
    assert total["large_n3_with_matches"] > 0
    assert total["records"] >= 1_000_000
