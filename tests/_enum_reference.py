"""Test-side host reference of the enumerations (sbg_enum3 / sbg_enum5 / sbg_enum7): the exact
records, totals, depth histogram and deal-block sums an enumeration must give for any state and any
settings (depth filter, function filter, grouping), built from the CPU oracle's keys alone.

The oracle (tests/enum_oracle.c through _enum_support's thread pools) only says which keys match.
Everything else is rebuilt here, vectorised with numpy over 4 x u64 truth tables: each key is decoded
into its gates in reference order and its outer and middle functions, the outer and middle tables
are computed, and the inner LUT is solved cell by cell as orc_solve_inner does (a cell holding a
masked 1 and a masked 0 rejects the match; `ones` / `seen` give func_inner / inner_seen).  The
filters and the grouping are then applied to those records.  No record the library emits is used.

check_realises() needs no keys: it rebuilds any record's circuit from the record's fields alone.

TEST INFRASTRUCTURE -- nothing under sboxgates_b200/ imports this module.
"""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor
from itertools import combinations
from math import comb

import numpy as np

import _enum_support as E
import _support as S
from sboxgates_b200.native import MATCH_DTYPE

CAP = 1 << 20                  # largest total the references are built for
ONES = np.uint64(2**64 - 1)
KDEAL = E.source_constant("kDeal", "sbg_device.cuh")
SHIFT = {("shape", 5): 8, ("shape", 7): 16, ("tuple", 5): 12, ("tuple", 7): 23}


# ------------------------------------------------------------------------------------------------
# Truth tables, vectorised: arrays of shape (..., 4) uint64.

def _sel(t, bit):
    return t if bit else ~t


def lut_tables(func, a, b, c):
    """lut_table (state.c:202-230) row by row: func (N,) function numbers, a, b, c (N, 4)."""
    func = np.asarray(func, dtype=np.uint64)
    a, b, c = (np.asarray(x, dtype=np.uint64) for x in (a, b, c))
    out = np.zeros(np.broadcast_shapes(a.shape, b.shape, c.shape), dtype=np.uint64)
    for m in range(8):
        on = ((func >> np.uint64(m)) & np.uint64(1)).astype(bool)[..., None]
        out |= np.where(on, _sel(a, m & 4) & _sel(b, m & 2) & _sel(c, m & 1), np.uint64(0))
    return out


def solve_inner(x, y, z, target, mask):
    """orc_solve_inner row by row: (ok, func_inner, inner_seen), each (N,).  x, y, z, target and
    mask broadcast against each other ((N, 4) or (4,))."""
    x, y, z, target, mask = (np.asarray(t, dtype=np.uint64) for t in (x, y, z, target, mask))
    shape = np.broadcast_shapes(x.shape, y.shape, z.shape, target.shape, mask.shape)[:-1]
    ok = np.ones(shape, dtype=bool)
    fi = np.zeros(shape, dtype=np.uint8)
    seen = np.zeros(shape, dtype=np.uint8)
    for c in range(8):
        cell = _sel(x, c & 4) & _sel(y, c & 2) & _sel(z, c & 1) & mask
        one = np.any(cell & target, axis=-1)
        zero = np.any(cell & ~target, axis=-1)
        ok &= ~(one & zero)
        fi |= one.astype(np.uint8) << np.uint8(c)
        seen |= (one | zero).astype(np.uint8) << np.uint8(c)
    return ok, fi, seen


# ------------------------------------------------------------------------------------------------
# The oracle's keys.

def _enum7_entries(tables, target, mask, tuples, outer, middle, max_keys):
    """orc_enum7 one list entry at a time on the pool: (total, keys with full-list indices)."""
    lib = E.enum_oracle()
    tabs, tp = S._u64(tables)
    tgt, gp = S._u64(target)
    msk, mp = S._u64(mask)
    lst = np.ascontiguousarray(tuples, dtype=np.uint16).reshape(-1, 7)
    fo, fm = S._order(outer), S._order(middle)

    def run(i):
        keys = np.zeros(max(max_keys, 1), dtype=np.uint64)
        one = np.ascontiguousarray(lst[i:i + 1])
        total = int(lib.orc_enum7(tp, gp, mp, one.ctypes.data_as(E.u16p), 1, fo, fm, max_keys,
                                  keys.ctypes.data_as(E.u64p)))
        return total, keys[:min(total, max_keys)] + np.uint64(i << 23)
    with ThreadPoolExecutor(max_workers=E.workers()) as pool:
        parts = list(pool.map(run, range(lst.shape[0])))
    keys = np.concatenate([p[1] for p in parts]) if parts else np.zeros(0, dtype=np.uint64)
    return sum(p[0] for p in parts), keys


def oracle_keys(width, tables, target, mask, inbits, orders, tuples=None, cap=CAP):
    """(total, every key in ascending order or None if total > cap, feasible) of the unfiltered
    enumeration: orc_enum3_range / orc_enum5_range / orc_enum7 on the pools.  `orders` are the
    enumerate call's order arguments: (gate_order,), (func_order,) or (outer, middle).  feasible:
    the matches (width 3), the feasible 5-combinations (width 5), the list length (width 7)."""
    if width == 3:
        total, keys = E.enum3_range(tables, target, mask, orders[0], cap + 1)
        feasible = total
    elif width == 5:
        total, keys, feasible = E.enum5_range(tables, target, mask, inbits, orders[0], cap + 1)
    else:
        total, keys = _enum7_entries(tables, target, mask, tuples, orders[0], orders[1],
                                     min(cap + 1, 70 * 65536))
        feasible = len(tuples)
    if total > cap:
        return total, None, feasible
    return total, np.asarray(keys, dtype=np.uint64), feasible


# ------------------------------------------------------------------------------------------------
# Records.

_COMBS = {}


def _combs(n, t):
    """Every t-subset of 0..n-1 in lexicographic order (the oracle's ranks), as an array."""
    if (n, t) not in _COMBS:
        assert comb(n, t) <= 4_000_000, (n, t)
        _COMBS[(n, t)] = np.array(list(combinations(range(n), t)), dtype=np.int64).reshape(-1, t)
    return _COMBS[(n, t)]


def decode(width, keys, n, orders, tuples=None):
    """(gates (N, width) in reference order, func_outer (N,), func_middle (N,)) of keys: the 3-LUT
    position triple through the gate order, the 5-combination of the rank through ordering row k
    (orc_order5_row) and order[pos], the list entry through row k (orc_order7_row), outer[po] and
    middle[pm]."""
    keys = np.asarray(keys, dtype=np.uint64).astype(np.int64) if len(keys) else \
        np.zeros(0, dtype=np.int64)
    rows = np.arange(len(keys))[:, None]
    zero = np.zeros(len(keys), dtype=np.int64)
    if width == 3:
        go = np.asarray(orders[0], dtype=np.int64)
        pos = np.stack([keys >> 18, (keys >> 9) & 0x1FF, keys & 0x1FF], axis=1)
        return go[pos], zero, zero
    if width == 5:
        order = np.frombuffer(bytes(orders[0]), dtype=np.uint8).astype(np.int64)
        row5 = np.array(S.order5_rows(), dtype=np.int64)
        tup = _combs(n, 5)[keys >> 12]
        return tup[rows, row5[(keys >> 8) & 0xF]], order[keys & 0xFF], zero
    outer = np.frombuffer(bytes(orders[0]), dtype=np.uint8).astype(np.int64)
    middle = np.frombuffer(bytes(orders[1]), dtype=np.uint8).astype(np.int64)
    row7 = np.array(S.order7_rows(), dtype=np.int64)
    tup = np.asarray(tuples, dtype=np.int64).reshape(-1, 7)[keys >> 23]
    return tup[rows, row7[(keys >> 16) & 0x7F]], outer[(keys >> 8) & 0xFF], middle[keys & 0xFF]


def _inputs(width, tables, gates, fo, fm):
    """The inner LUT's three input tables of records given by their fields."""
    t = np.asarray(tables, dtype=np.uint64)
    g = [t[gates[:, i]] for i in range(width)]
    if width == 3:
        return g[0], g[1], g[2]
    x = lut_tables(fo, g[0], g[1], g[2])
    y = g[3] if width == 5 else lut_tables(fm, g[3], g[4], g[5])
    return x, y, g[-1]


def build_records(width, keys, tables, target, mask, orders, tuples=None):
    """The MATCH_DTYPE records of the matches `keys` (each must decompose): the fields decoded from
    the key, func_inner / inner_seen solved on the host."""
    n = len(tables)
    gates, fo, fm = decode(width, keys, n, orders, tuples)
    ok, fi, seen = solve_inner(*_inputs(width, tables, gates, fo, fm), target, mask)
    assert ok.all(), "oracle keys that do not decompose: %s" % [hex(int(k)) for k in
                                                                 np.asarray(keys)[~ok][:5]]
    recs = np.zeros(len(keys), dtype=MATCH_DTYPE)
    recs["key"] = keys
    recs["gates"][:, :width] = gates
    recs["func_outer"] = fo
    recs["func_middle"] = fm
    recs["func_inner"] = fi
    recs["inner_seen"] = seen
    recs["width"] = width
    return recs


def check_realises(recs, tables, target, mask, what=""):
    """Every record (of widths 3, 5 or 7; all-zero records of width 0 are skipped) rebuilt from its
    own fields: gates past the width, the functions the width has no LUT for and the pad are zero;
    the outer and middle LUTs over the record's gates, with func_inner as the inner LUT, equal the
    target on the mask; and func_inner / inner_seen are exactly the solved bits of those inputs.
    Returns the number of records checked."""
    recs = np.asarray(recs)
    widths = recs["width"].astype(np.int64)
    assert np.isin(widths, [0, 3, 5, 7]).all(), (what, sorted(set(widths.tolist())))
    zero = recs[widths == 0]
    assert not zero.view(np.uint64).any(), (what, "a width-0 record that is not all zero")
    for width in (3, 5, 7):
        r = recs[widths == width]
        if len(r) == 0:
            continue
        where = np.flatnonzero(widths == width)
        assert not r["gates"][:, width:].any(), (what, width, "gates past the width")
        assert not r["pad"].any(), (what, width, "pad")
        if width == 3:
            assert not r["func_outer"].any(), (what, "func_outer at width 3")
        if width < 7:
            assert not r["func_middle"].any(), (what, width, "func_middle below width 7")
        gates = r["gates"][:, :width].astype(np.int64)
        assert (gates < len(tables)).all(), (what, width, "gate out of range")
        x, y, z = _inputs(width, tables, gates, r["func_outer"].astype(np.int64),
                          r["func_middle"].astype(np.int64))
        fi = r["func_inner"]
        out = lut_tables(fi, x, y, z)
        bad = np.any((out ^ np.asarray(target, dtype=np.uint64)) & np.asarray(mask, dtype=np.uint64),
                     axis=1)
        assert not bad.any(), (what, width, "does not realise the target",
                               int(where[np.argmax(bad)]), hex(int(r["key"][np.argmax(bad)])))
        ok, sfi, sseen = solve_inner(x, y, z, target, mask)
        wrong = ~ok | (sfi != fi) | (sseen != r["inner_seen"])
        assert not wrong.any(), (what, width, "func_inner / inner_seen not the solved bits",
                                 int(where[np.argmax(wrong)]), hex(int(r["key"][np.argmax(wrong)])))
    return len(recs) - len(zero)


# ------------------------------------------------------------------------------------------------
# Settings: what a filter or grouping keeps.

def function_ok(recs, outer=None, middle=None, inner=None):
    """match_functions_allowed over an array of records (sets: None = all 256)."""
    width = recs["width"].astype(np.int64)
    ok = np.ones(len(recs), dtype=bool)
    if outer is not None:
        ok &= (width == 3) | np.isin(recs["func_outer"], np.asarray(list(outer), dtype=np.int64))
    if middle is not None:
        ok &= (width != 7) | np.isin(recs["func_middle"], np.asarray(list(middle), dtype=np.int64))
    if inner is not None:
        comp = np.zeros((256, 256), dtype=bool)    # [seen, ones]: some f of inner completes them
        s = np.arange(256)
        for f in inner:
            comp[s, int(f) & s] = True
        ok &= comp[recs["inner_seen"].astype(np.int64), recs["func_inner"].astype(np.int64)]
    return ok


def group_ids(keys, width, grouping):
    """match_group's id of every key."""
    keys = np.asarray(keys, dtype=np.uint64)
    if grouping is None or width == 3:
        return keys
    return keys >> np.uint64(SHIFT[(grouping, width)])


def group_first(recs, width, grouping):
    """Mask of the first record of each run of equal group ids (records in key order)."""
    keep = np.ones(len(recs), dtype=bool)
    if len(recs):
        ids = group_ids(recs["key"], width, grouping)
        keep[1:] = ids[1:] != ids[:-1]
    return keep


def histogram(depths):
    """The depth histogram as depth_counts gives it: cut after the last non-empty bin."""
    depths = np.asarray(depths, dtype=np.int64)
    if depths.size == 0:
        return np.zeros(0, dtype=np.uint64)
    return np.bincount(depths).astype(np.uint64)


# ------------------------------------------------------------------------------------------------
# Deal blocks: how a part's tickets are cut (sbg_api.cu run_enum: kDeal position pairs or 3-gate
# prefixes per block, one list entry per block; block j goes to part j mod P).

def ticket_items(width, keys, n):
    """The ticket item (position pair rank, 3-gate prefix rank or list index) of each key."""
    keys = np.asarray(keys, dtype=np.uint64).astype(np.int64)
    if width == 3:
        i, k = keys >> 18, (keys >> 9) & 0x1FF
        return i * (2 * n - i - 1) // 2 + (k - i - 1)
    if width == 5:
        c = _combs(n, 5)[keys >> 12]
        m = n - 2   # prefixes are 3-subsets of 0..n-3, lexicographic
        a, b, d = c[:, 0], c[:, 1], c[:, 2]
        tri = np.array([comb(m - x, 3) for x in range(m + 1)], dtype=np.int64)
        pair = np.array([[comb(m - x, 2) for x in range(m + 1)]], dtype=np.int64)[0]
        return (comb(m, 3) - tri[a]) + (pair[a + 1] - pair[b]) + (d - b - 1)
    return keys >> 23


def item_count(width, n, list_len=0):
    return comb(n, 2) if width == 3 else comb(n - 2, 3) if width == 5 else list_len


def block_size(width):
    return 1 if width == 7 else KDEAL


def deal_share(blocks, q, nparts):
    """sbg_api.cu deal_share: the deal blocks part q of nparts holds."""
    return (blocks - q + nparts - 1) // nparts if blocks > q else 0


class Reference:
    """The expected outcome of an enumeration of one state under given settings.

    all:      every unfiltered record, key order;
    recs:     the records the enumeration must give (filters, then grouping), key order;
    total, feasible, hist (depth histogram of recs);
    blocks:   the deal block of each of recs; share(q, P) / share_sums(q, P) per part."""

    def __init__(self, width, tables, target, mask, inbits, orders, tuples=None, keys=None,
                 feasible=None):
        self.width, self.n = width, len(tables)
        self.tables, self.target, self.mask = tables, target, mask
        self.inbits, self.orders, self.tuples = list(inbits), orders, tuples
        if keys is None:
            _, keys, feasible = oracle_keys(width, tables, target, mask, inbits, orders, tuples)
            assert keys is not None, "more than %d matches" % CAP
        self.keys = keys
        self.all = build_records(width, keys, tables, target, mask, orders, tuples)
        self.plain_feasible = feasible
        self.items = ticket_items(width, keys, self.n)
        self.select()

    def select(self, depth=None, bound=None, outer=None, middle=None, inner=None, grouping=None,
               functions=False):
        """Applies settings: depth filter (gate depths, bound) if depth is not None, the function
        filter (outer, middle, inner) if `functions`, and a grouping."""
        ok = np.ones(len(self.all), dtype=bool)
        self.depths = None
        if depth is not None:
            self.depths = E.record_depths(self.all, depth)
            ok &= self.depths <= bound
        depth_ok = ok.copy()
        if functions:
            ok &= function_ok(self.all, outer, middle, inner)
        idx = np.flatnonzero(ok)
        sub = self.all[idx]
        if grouping is not None and self.width != 3:
            idx = idx[group_first(sub, self.width, grouping)]
        self.idx = idx
        self.recs = self.all[idx]
        self.total = len(idx)
        self.hist = histogram(self.depths[idx]) if depth is not None else None
        self.feasible = self._feasible(depth, bound, depth_ok)
        self.blocks = self.items[idx] // block_size(self.width)
        return self

    def _feasible(self, depth, bound, depth_ok):
        if self.width == 7:
            return len(self.tuples)
        if self.width == 3:
            return int(depth_ok.sum())
        if depth is None:
            return self.plain_feasible
        return E.feasible5_under_bound(self.tables, self.target, self.mask, self.inbits, depth,
                                       bound)

    def nblocks(self):
        items = item_count(self.width, self.n, 0 if self.tuples is None else len(self.tuples))
        return -(-items // block_size(self.width))

    def share(self, q, nparts):
        """The records of part q of nparts, key order."""
        return self.recs[self.blocks % nparts == q]

    def share_sums(self, q, nparts):
        """The match count of each of part q's deal blocks, in its local block order."""
        mine = self.blocks[self.blocks % nparts == q]
        return np.bincount(mine // nparts, minlength=deal_share(self.nblocks(), q, nparts)) \
            .astype(np.uint64)

    def seams(self):
        """Ranks in recs where the ticket item changes (a ticket's first match)."""
        it = self.items[self.idx]
        return np.flatnonzero(np.diff(it) != 0) + 1 if len(it) > 1 else np.zeros(0, dtype=np.int64)


def solve_inner_oracle(x, y, z, target, mask):
    """orc_solve_inner on one triple: (ok, func, seen)."""
    arrs = [S._u64(t) for t in (x, y, z, target, mask)]
    fi, seen = C.c_uint8(), C.c_uint8()
    ok = S.oracle_lib().orc_solve_inner(*[a[1] for a in arrs], C.byref(fi), C.byref(seen))
    return bool(ok), int(fi.value), int(seen.value)
