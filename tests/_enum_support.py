"""Test-side helpers of the enumeration tests: the CPU enumeration oracle (tests/enum_oracle.c,
compiled with oracle/sbg_oracle.c into a temporary directory on first use), its ctypes bindings,
the seeded states the tests share, and an independent check of one enumerated record.

TEST INFRASTRUCTURE -- nothing under sboxgates_b200/ imports this module.
"""
import ctypes as C
import os
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

import _support as S

HERE = os.path.dirname(os.path.abspath(__file__))
u64p, u16p, u8p, i8p = S.u64p, S.u16p, S.u8p, S.i8p
NONE = 2**64 - 1   # no match (SBG_KEY_NONE, UINT64_MAX)

_lib = None


def enum_oracle():
    """Loads the enumeration oracle, compiling it first (once per process, outside the tree)."""
    global _lib
    if _lib is not None:
        return _lib
    out = os.path.join(tempfile.mkdtemp(prefix="sbg_enum_oracle_"), "libenumoracle.so")
    cc = os.environ.get("CC", "gcc")
    subprocess.run([cc, "-O2", "-fPIC", "-shared", "-I", S.ORACLE_DIR, "-o", out,
                    os.path.join(HERE, "enum_oracle.c"), os.path.join(S.ORACLE_DIR, "sbg_oracle.c")],
                   check=True, capture_output=True)
    lib = C.CDLL(out)
    lib.orc_enum5.restype = C.c_uint64
    lib.orc_enum5.argtypes = [u64p, C.c_int, u64p, u64p, i8p, u8p, C.c_uint64, u64p, u64p]
    lib.orc_enum7.restype = C.c_uint64
    lib.orc_enum7.argtypes = [u64p, u64p, u64p, u16p, C.c_int, u8p, u8p, C.c_uint64, u64p]
    lib.orc_enum5_range.restype = C.c_uint64
    lib.orc_enum5_range.argtypes = [u64p, C.c_int, u64p, u64p, i8p, u8p, C.c_int64, C.c_int64,
                                    C.c_uint64, u64p, u64p]
    lib.orc_search5_range.restype = C.c_uint64
    lib.orc_search5_range.argtypes = [u64p, C.c_int, u64p, u64p, i8p, u8p, C.c_int64, C.c_int64]
    lib.orc_feasible5_range.restype = C.c_uint64
    lib.orc_feasible5_range.argtypes = [u64p, C.c_int, u64p, u64p, i8p, C.c_int64, C.c_int64]
    lib.orc_filter7_range.restype = C.c_int64
    lib.orc_filter7_range.argtypes = [u64p, C.c_int, u64p, u64p, i8p, C.c_int64, C.c_int64, u16p,
                                      C.c_int64]
    lib.orc_check7_list.restype = C.c_int64
    lib.orc_check7_list.argtypes = [u64p, u64p, u64p, u16p, C.c_int64, C.POINTER(C.c_int64)]
    lib.orc_scan3_key.restype = C.c_uint64
    lib.orc_scan3_key.argtypes = [u64p, C.c_int, u64p, u64p, u16p, C.c_int64, C.c_int64]
    lib.orc_enum3_range.restype = C.c_uint64
    lib.orc_enum3_range.argtypes = [u64p, C.c_int, u64p, u64p, u16p, C.c_int64, C.c_int64,
                                    C.c_uint64, u64p]
    _lib = lib
    return lib


# ------------------------------------------------------------------------------------------------
# Rank-range forms: a space of combinations cut into pieces of consecutive ranks, the pieces run on
# a thread pool (the ctypes calls release the interpreter lock), the results merged.

def workers():
    return max(1, min(8, os.cpu_count() or 1))


def pieces(lo, hi, size):
    """[lo, hi) cut into consecutive ranges of at most `size` ranks."""
    return [(a, min(hi, a + size)) for a in range(lo, hi, max(1, size))]


def _problem(tables, target, mask, inbits):
    tables, tp = S._u64(tables)
    target, gp = S._u64(target)
    mask, mp = S._u64(mask)
    ib = S.inbits_array(inbits)
    return (tables, target, mask, ib), (tp, tables.shape[0], gp, mp, ib.ctypes.data_as(i8p))


def filter7_range(tables, target, mask, inbits, lo, hi, piece=None):
    """The feasible 7-combinations (inbits applied) of ranks [lo, hi), in order, as a (count, 7)
    uint16 array: orc_filter7_range over pieces, concatenated."""
    lib = enum_oracle()
    _keep, args = _problem(tables, target, mask, inbits)

    def run(r):
        out = np.zeros((r[1] - r[0], 7), dtype=np.uint16)
        cnt = lib.orc_filter7_range(*args, r[0], r[1], out.ctypes.data_as(u16p), out.shape[0])
        return out[:cnt]
    rs = pieces(lo, hi, piece or max(1, -(-(hi - lo) // workers())))
    with ThreadPoolExecutor(max_workers=workers()) as pool:
        parts = list(pool.map(run, rs))
    return np.concatenate(parts) if parts else np.zeros((0, 7), dtype=np.uint16)


def check7_list(tables, target, mask, tuples):
    """(entries of a (count, 7) list that check_n_lut_possible(7) rejects, index of the first)."""
    lib = enum_oracle()
    _keep, args = _problem(tables, target, mask, [])
    lst = np.ascontiguousarray(tuples, dtype=np.uint16).reshape(-1, 7)
    step = max(1, -(-lst.shape[0] // workers()))

    def run(a):
        first = C.c_int64()
        sub = lst[a:a + step]
        bad = lib.orc_check7_list(args[0], args[2], args[3], sub.ctypes.data_as(u16p), sub.shape[0],
                                  C.byref(first))
        return int(bad), (a + first.value if bad else -1)
    with ThreadPoolExecutor(max_workers=workers()) as pool:
        res = list(pool.map(run, range(0, lst.shape[0], step)))
    firsts = [f for _, f in res if f >= 0]
    return sum(b for b, _ in res), (min(firsts) if firsts else -1)


def search5_range(tables, target, mask, inbits, order, lo, hi, piece):
    """orc_search5_key's key restricted to ranks [lo, hi): the pieces run a batch (one per worker)
    at a time, and the search stops after the first batch that holds a match."""
    lib = enum_oracle()
    _keep, args = _problem(tables, target, mask, inbits)
    fo = S._order(order)
    rs = pieces(lo, hi, piece)
    w = workers()
    with ThreadPoolExecutor(max_workers=w) as pool:
        for b in range(0, len(rs), w):
            keys = list(pool.map(lambda r: int(lib.orc_search5_range(*args, fo, r[0], r[1])),
                                 rs[b:b + w]))
            if min(keys) != NONE:
                return min(keys)
    return NONE


def enum5_range(tables, target, mask, inbits, order, max_keys, lo=0, hi=None, piece=None):
    """(total, first max_keys keys, feasible) of search_5lut's matches of ranks [lo, hi) (default:
    all of C(n,5)): orc_enum5_range over pieces, totals summed, key lists concatenated."""
    lib = enum_oracle()
    _keep, args = _problem(tables, target, mask, inbits)
    fo = S._order(order)
    if hi is None:
        hi = int(S.oracle_lib().orc_n_choose_k(args[1], 5))

    def run(r):
        keys = np.zeros(max(max_keys, 1), dtype=np.uint64)
        feasible = C.c_uint64()
        total = lib.orc_enum5_range(*args, fo, r[0], r[1], max_keys, keys.ctypes.data_as(u64p),
                                    C.byref(feasible))
        return int(total), [int(k) for k in keys[:min(total, max_keys)]], int(feasible.value)
    rs = pieces(lo, hi, piece or max(1, -(-(hi - lo) // (4 * workers()))))
    with ThreadPoolExecutor(max_workers=workers()) as pool:
        parts = list(pool.map(run, rs))
    keys = [k for p in parts for k in p[1]][:max_keys]
    return sum(p[0] for p in parts), keys, sum(p[2] for p in parts)


def scan3_key(tables, target, mask, order, lo=0, hi=None, piece=None):
    """lut_search's 3-LUT scan (lut.c:501-523) over the gate order `order`: the key i<<18 | k<<9 | m
    of its first realising position triple, or NONE; minimum over pieces of orc_scan3_key."""
    lib = enum_oracle()
    _keep, args = _problem(tables, target, mask, [])
    n = args[1]
    go = np.ascontiguousarray(order, dtype=np.uint16)
    if hi is None:
        hi = n * (n - 1) * (n - 2) // 6
    rs = pieces(lo, hi, piece or max(1, -(-(hi - lo) // (4 * workers()))))
    with ThreadPoolExecutor(max_workers=workers()) as pool:
        keys = list(pool.map(lambda r: int(lib.orc_scan3_key(args[0], n, args[2], args[3],
                                                             go.ctypes.data_as(u16p), r[0], r[1])),
                             rs))
    return min(keys) if keys else NONE


def enum3_range(tables, target, mask, order, max_keys, lo=0, hi=None, piece=None):
    """(total, first max_keys keys) of the 3-LUT scan's matches among the position triples of ranks
    [lo, hi) (default: all of C(n,3)): orc_enum3_range over pieces, totals summed, key lists
    concatenated.  Every match is a feasible triple, so the total is also the feasible count."""
    lib = enum_oracle()
    _keep, args = _problem(tables, target, mask, [])
    n = args[1]
    go = np.ascontiguousarray(order, dtype=np.uint16)
    if hi is None:
        hi = n * (n - 1) * (n - 2) // 6

    def run(r):
        keys = np.zeros(max(max_keys, 1), dtype=np.uint64)
        total = lib.orc_enum3_range(args[0], n, args[2], args[3], go.ctypes.data_as(u16p), r[0],
                                    r[1], max_keys, keys.ctypes.data_as(u64p))
        return int(total), [int(k) for k in keys[:min(total, max_keys)]]
    rs = pieces(lo, hi, piece or max(1, -(-(hi - lo) // (4 * workers()))))
    with ThreadPoolExecutor(max_workers=workers()) as pool:
        parts = list(pool.map(run, rs))
    keys = [k for p in parts for k in p[1]][:max_keys]
    return sum(p[0] for p in parts), keys


# ------------------------------------------------------------------------------------------------
# search_7lut's phase 2 on the host: orc_decomp7_key over pieces of a list, per entry and per part,
# and the sbg_result fields a key must come with.

class _List7:
    """The pointers orc_decomp7_key takes for one (state, list, orders), marshalled once."""

    def __init__(self, tables, target, mask, tuples, outer, middle):
        self.tables, self.tp = S._u64(tables)
        self.target, self.gp = S._u64(target)
        self.mask, self.mp = S._u64(mask)
        self.lst = np.ascontiguousarray(tuples, dtype=np.uint16).reshape(-1, 7)
        self.outer, self.middle = S._order(outer), S._order(middle)

    def key(self, part, nparts, lo=0, hi=None):
        """orc_decomp7_key(part, nparts) of entries [lo, hi) (hi <= the list's length), full-list
        indices.  The list handed over starts at entry lo - 1, whose row 69 leaves the outer cache
        that entry lo begins with; entry lo - 1 itself is not decided."""
        hi = self.lst.shape[0] if hi is None else hi
        base = max(lo - 1, 0)
        sub = self.lst[base:hi]
        first = lo - base + (part - lo) % nparts   # the first entry >= lo of index part (mod nparts)
        key = int(S.oracle_lib().orc_decomp7_key(self.tp, self.gp, self.mp,
                                                 sub.ctypes.data_as(u16p), sub.shape[0],
                                                 self.outer, self.middle, first, nparts))
        return key if key == NONE else key + (base << 23)


def decomp7_range(tables, target, mask, tuples, outer, middle, lo, hi):
    """The oracle's first key over list entries [lo, hi) with full-list indices (orc_decomp7_key of
    the whole list restricted to those entries; the outer cache on entry to lo comes from lo - 1)."""
    lst = _List7(tables, target, mask, tuples, outer, middle)
    hi = min(hi, lst.lst.shape[0])
    return NONE if lo >= hi else lst.key(0, 1, lo, hi)


def decomp7_key(tables, target, mask, tuples, outer, middle, piece=8):
    """orc_decomp7_key of the whole list: slices of `piece` entries, a batch (one per worker) at a
    time in list order, stopping after the first batch that holds a match."""
    lst = _List7(tables, target, mask, tuples, outer, middle)
    rs = pieces(0, lst.lst.shape[0], piece)
    w = workers()
    with ThreadPoolExecutor(max_workers=w) as pool:
        for b in range(0, len(rs), w):
            keys = list(pool.map(lambda r: lst.key(0, 1, r[0], r[1]), rs[b:b + w]))
            if min(keys) != NONE:
                return min(keys)
    return NONE


def decomp7_entry_keys(tables, target, mask, tuples, outer, middle):
    """Every entry's own first key: orc_decomp7_key(part=p, nparts=len(list)) for each p (the
    entry's predecessor still sets its outer cache), on the pool."""
    lst = _List7(tables, target, mask, tuples, outer, middle)
    count = lst.lst.shape[0]
    with ThreadPoolExecutor(max_workers=workers()) as pool:
        return list(pool.map(lambda p: lst.key(p, count), range(count)))


def part_keys(entry_keys, nparts):
    """Part p's key of decomp7_part(p, nparts) from the entries' own keys: the minimum over the
    entries of index p (mod nparts) (NONE for an empty part)."""
    return [min(entry_keys[p::nparts], default=NONE) for p in range(nparts)]


def planted7(tables, gates, k, fo, fm, fi, stale_gate=None):
    """Target fi(fo(outer), fm(middle), last) on ordering row k of the 7 gates; the outer LUT reads
    stale_gate in place of its first input when given (what a stale-cache row computes)."""
    row = S.order7_rows()[k]
    g = [int(gates[row[i]]) for i in range(7)]
    a = g[0] if stale_gate is None else stale_gate
    return S.lut_table(int(fi), S.lut_table(int(fo), tables[a], tables[g[1]], tables[g[2]]),
                       S.lut_table(int(fm), tables[g[3]], tables[g[4]], tables[g[5]]), tables[g[6]])


def stale_pairs(rs, n, count, lo=1):
    """count pairs (0, a1..a4, t1, t2) < (0, t1, t2, ...) that follow each other in list order, the
    a's of each pair above the t1 of the pair before and the first a at least lo: the second entry
    of a pair runs rows 0-3 on the outer tables the first one's row 69 left (gates a1, t1, t2)."""
    out, floor = [], lo
    for j in range(count):
        room = (n - 6 - floor - 4) // (count - j)   # values left for this pair's a's and t1
        assert room >= 1, (n, count, lo)
        t1 = floor + 4 + int(rs.randint(room))
        head = sorted(int(x) for x in rs.choice(np.arange(floor, t1), 4, replace=False))
        rest = sorted(int(x) for x in rs.choice(np.arange(t1 + 2, n), 4, replace=False))
        out += [[0] + head + [t1, t1 + 1], [0, t1, t1 + 1] + rest]
        floor = t1 + 1
    return out


def stale_source(tuples, idx, k):
    """The gate the reference's outer cache holds in place of row k's first gate at entry idx, or
    None: rows 0-3 (outer = first three gates) of an entry whose first gate is 0 keep the outer
    tables of the previous entry's row 69 (outer = its gates 1, 5, 6) when that entry ends in this
    one's gates 1 and 2 (the cache key drops the first gate)."""
    if idx == 0 or k >= 4:
        return None
    t, prev = tuples[idx], tuples[idx - 1]
    if t[0] == 0 and prev[5] == t[1] and prev[6] == t[2]:
        return int(prev[1])
    return None


def expected_result7(key, tuples, tables, target, mask, outer, middle):
    """The sbg_result fields (a dict) the 7-LUT key `key` over the list `tuples` must come with, from
    the oracle's ordering rows and inner solver; None for SBG_KEY_NONE or a key that does not
    decompose."""
    if key == NONE:
        return None
    idx, k, po, pm = key >> 23, (key >> 16) & 0x7F, (key >> 8) & 0xFF, key & 0xFF
    lst = np.asarray(tuples, dtype=np.uint16).reshape(-1, 7)
    row = S.order7_rows()[k]
    gates = [int(lst[idx][row[i]]) for i in range(7)]
    fo, fm = int(outer[po]), int(middle[pm])
    sub = stale_source(lst, idx, k)
    a = gates[0] if sub is None else sub
    t1 = S.lut_table(fo, tables[a], tables[gates[1]], tables[gates[2]])
    t2 = S.lut_table(fm, tables[gates[3]], tables[gates[4]], tables[gates[5]])
    arrs = [S._u64(x) for x in (t1, t2, tables[gates[6]], target, mask)]
    fi, seen = C.c_uint8(), C.c_uint8()
    if not S.oracle_lib().orc_solve_inner(*[x[1] for x in arrs], C.byref(fi), C.byref(seen)):
        return None
    return dict(found=1, key=key, index=idx, ordering=k, pos_outer=po, pos_middle=pm,
                func_outer=fo, func_middle=fm, func_inner=int(fi.value),
                inner_seen=int(seen.value), gates=gates, stale_outer=int(sub is not None))


def result7_fields(res):
    """The fields of an sbg_result (SbgResult) that expected_result7 gives, as a dict."""
    out = {f: int(getattr(res, f)) for f in ("found", "key", "index", "ordering", "pos_outer",
                                              "pos_middle", "func_outer", "func_middle",
                                              "func_inner", "inner_seen", "stale_outer")}
    out["gates"] = [int(g) for g in res.gates[:7]]
    return out


# ------------------------------------------------------------------------------------------------
# search_5lut on the host: one combination's key, the keys of the library's shares of a sharded
# search, the feasible count and the sbg_result fields a 5-LUT key must come with.

def search5_tuple_key(tables, target, mask, inbits, order, rank):
    """The key of combination `rank` alone (orc_search5_range over [rank, rank + 1)), or NONE."""
    lib = enum_oracle()
    _keep, args = _problem(tables, target, mask, inbits)
    return int(lib.orc_search5_range(*args, S._order(order), rank, rank + 1))


def feasible5(tables, target, mask, inbits, lo=0, hi=None, piece=None):
    """The feasible 5-combinations (inbits applied) of ranks [lo, hi) (default: all of C(n,5)):
    orc_feasible5_range over pieces on the pool, summed."""
    lib = enum_oracle()
    _keep, args = _problem(tables, target, mask, inbits)
    if hi is None:
        hi = int(S.oracle_lib().orc_n_choose_k(args[1], 5))
    rs = pieces(lo, hi, piece or max(1, -(-(hi - lo) // (4 * workers()))))
    with ThreadPoolExecutor(max_workers=workers()) as pool:
        return sum(pool.map(lambda r: int(lib.orc_feasible5_range(*args, r[0], r[1])), rs))


def planted5(tabs, gates, k, fo, fi):
    """Target fi(fo(outer triple), inner pair) on ordering row k of the 5 gates (in the order of
    `gates`, which is the combination's when they ascend)."""
    row = S.order5_rows()[k]
    g = [int(gates[row[i]]) for i in range(5)]
    return S.lut_table(int(fi), S.lut_table(int(fo), tabs[g[0]], tabs[g[1]], tabs[g[2]]),
                       tabs[g[3]], tabs[g[4]])


def expected_result5(key, tables, target, mask, order):
    """The sbg_result fields (a dict) the 5-LUT key `key` must come with, from the oracle's ordering
    rows and inner solver; None for SBG_KEY_NONE or a key that does not decompose."""
    if key == NONE:
        return None
    rank, k, pos = key >> 12, (key >> 8) & 0xF, key & 0xFF
    comb = nth_comb(len(tables), 5, rank)
    row = S.order5_rows()[k]
    gates = [comb[row[i]] for i in range(5)]
    fo = int(order[pos])
    t1 = S.lut_table(fo, tables[gates[0]], tables[gates[1]], tables[gates[2]])
    arrs = [S._u64(x) for x in (t1, tables[gates[3]], tables[gates[4]], target, mask)]
    fi, seen = C.c_uint8(), C.c_uint8()
    if not S.oracle_lib().orc_solve_inner(*[x[1] for x in arrs], C.byref(fi), C.byref(seen)):
        return None
    return dict(found=1, key=key, index=rank, ordering=k, pos_outer=pos, pos_middle=0,
                func_outer=fo, func_middle=0, func_inner=int(fi.value), inner_seen=int(seen.value),
                gates=gates, stale_outer=0)


def result5_fields(res):
    """The fields of an sbg_result that expected_result5 gives, as a dict."""
    out = result7_fields(res)
    out["gates"] = out["gates"][:5]
    return out


def source_constant(name, filename):
    """A `constexpr uint64_t name = <int>;` of the library's source (sboxgates_b200/csrc)."""
    import re
    text = open(os.path.join(S.ROOT, "sboxgates_b200", "csrc", filename)).read()
    m = re.search(r"constexpr uint64_t %s = (\d+);" % name, text)
    assert m is not None, "cannot read %s from %s: update source_constant" % (name, filename)
    return int(m.group(1))


class Deal5:
    """How search_5lut's sweep (k_sweep) cuts C(n,5) into items and deals them to the parts of a
    sharded search, as rank ranges.

    An item is a 3-gate prefix (a 3-subset of {0..n-3}, lexicographic), whose 5-combinations form
    one contiguous rank range.  With the fused head (fused form, n >= 128) the first items are
    (allowed-gate prefix, chunk of 32 (d,e) pairs) items over the first prefixes made of allowed
    gates only, and the prefix items start at the first allowed prefix the head does not cover
    (t_offset); sbg_plan_tickets gives the head's items, its chunks per prefix and t_offset.  The
    head items and the prefix items are each dealt in blocks of kDeal consecutive items, block j to
    part j mod P.  Every head item lies below t_offset, so a part's blocks in the order head blocks,
    prefix blocks are in ascending rank order."""

    def __init__(self, n, inbits, head):
        from sboxgates_b200 import native
        self.n = n
        self.kdeal = source_constant("kDeal", "sbg_device.cuh")
        self.total = int(S.oracle_lib().orc_n_choose_k(n - 2, 3))
        excl = sorted({int(b) for b in inbits if 0 <= b < 8})
        self.items, self.chunks, self.t_offset = 0, 1, 0
        if head:
            out = (C.c_uint64 * 4)()
            rc = native.load_library().sbg_plan_tickets(
                5, 3, n, sum(1 << b for b in excl), 1, source_constant("kHeadWaves5", "sbg_api.cu"),
                out)
            assert rc == 0, (n, excl)
            self.items, self.chunks, self.t_offset = int(out[0]), int(out[1]), int(out[2])
        self.allowed = [g for g in range(n) if g not in excl]
        self.head_blocks = -(-self.items // self.kdeal)
        self.prefix_blocks = -(-(self.total - self.t_offset) // self.kdeal)

    def _base(self, pre):
        """(rank of the prefix's first combination, its number of combinations)."""
        r = self.n - pre[2] - 1
        return comb_rank(self.n, 5, list(pre) + [pre[2] + 1, pre[2] + 2]), r * (r - 1) // 2

    def block_ranges(self, j):
        """The rank ranges [lo, hi) of block j of the dealt order (head blocks first), ascending."""
        out = []
        if j < self.head_blocks:
            for i in range(j * self.kdeal, min((j + 1) * self.kdeal, self.items)):
                t, c = divmod(i, self.chunks)
                idx = nth_comb(len(self.allowed) - 2, 3, t)
                base, q = self._base([self.allowed[x] for x in idx])
                lo, hi = base + 32 * c, base + min(32 * c + 32, q)
                if lo >= hi:
                    continue
                if out and out[-1][1] == lo:
                    out[-1] = (out[-1][0], hi)
                else:
                    out.append((lo, hi))
            return out
        j -= self.head_blocks
        first = self.t_offset + j * self.kdeal
        last = min(first + self.kdeal, self.total) - 1
        lo, _ = self._base(nth_comb(self.n - 2, 3, first))
        base, q = self._base(nth_comb(self.n - 2, 3, last))
        return [(lo, base + q)]

    def blocks(self):
        return self.head_blocks + self.prefix_blocks

    def part_blocks(self, part, nparts, skip_excluded=True):
        """The blocks of part `part` of `nparts`, in ascending rank order.  Prefix blocks that end
        before the first prefix of allowed gates hold no allowed combination; skip_excluded leaves
        them out (with input bits 0-7 excluded at n = 500 they are 68,000 blocks)."""
        first = 0
        if skip_excluded and len(self.allowed) >= 5:
            lead = comb_rank(self.n - 2, 3, self.allowed[:3])
            first = max(0, (lead - self.t_offset) // self.kdeal)
        start = first + (part - first) % nparts
        return ([j for j in range(part, self.head_blocks, nparts)]
                + [self.head_blocks + j for j in range(start, self.prefix_blocks, nparts)])


class Search5Oracle:
    """The oracle's first keys of one search_5lut problem per dealt block, computed on demand and
    kept, so that the keys of several shardings come from one walk."""

    def __init__(self, tables, target, mask, inbits, order, head):
        self.n = len(tables)
        self.deal = Deal5(self.n, inbits, head)
        self.keep, self.args = _problem(tables, target, mask, inbits)
        self.order = S._order(order)
        self.keys = {}
        self.walked = 0   # combinations the oracle has decided or rejected

    def block_key(self, j):
        if j not in self.keys:
            key = NONE
            for lo, hi in self.deal.block_ranges(j):
                key = int(enum_oracle().orc_search5_range(*self.args, self.order, lo, hi))
                self.walked += hi - lo
                if key != NONE:
                    break
            self.keys[j] = key
        return self.keys[j]

    def part_key(self, part, nparts, limit=None):
        """The key of part `part` of `nparts`: its blocks a batch (one per worker) at a time in rank
        order, stopping after the first batch that holds a match.  None if its blocks spanning
        `limit` combinations held no match and more are left."""
        blocks = self.deal.part_blocks(part, nparts)
        w = workers()
        spanned = 0
        with ThreadPoolExecutor(max_workers=w) as pool:
            for b in range(0, len(blocks), w):
                if limit is not None and spanned >= limit:
                    return None
                batch = blocks[b:b + w]
                keys = list(pool.map(self.block_key, batch))
                if min(keys) != NONE:
                    return min(keys)
                spanned += sum(hi - lo for j in batch for lo, hi in self.deal.block_ranges(j))
        return NONE


def part_keys5(tables, target, mask, inbits, order, part, nparts, head):
    """The key of the library's share `part` of `nparts` of a sharded search_5lut (Deal5)."""
    return Search5Oracle(tables, target, mask, inbits, order, head).part_key(part, nparts)


def comb_rank(n, t, comb):
    """Lexicographic rank of a t-subset of {0..n-1} (orc_combination_rank)."""
    c = (C.c_uint16 * t)(*[int(x) for x in comb])
    return int(S.oracle_lib().orc_combination_rank(n, t, c))


def nth_comb(n, t, rank):
    c = (C.c_uint16 * t)()
    S.oracle_lib().orc_nth_combination(int(rank), n, t, c)
    return [int(x) for x in c]


def oracle_enum5(tables, target, mask, inbits, order, max_keys):
    """(total, first max_keys keys, feasible combinations) of search_5lut's matches."""
    lib = enum_oracle()
    tables, tp = S._u64(tables)
    target, gp = S._u64(target)
    mask, mp = S._u64(mask)
    ib = S.inbits_array(inbits)
    keys = np.zeros(max(max_keys, 1), dtype=np.uint64)
    feasible = C.c_uint64()
    total = lib.orc_enum5(tp, tables.shape[0], gp, mp, ib.ctypes.data_as(i8p), S._order(order),
                          max_keys, keys.ctypes.data_as(u64p), C.byref(feasible))
    return int(total), [int(k) for k in keys[:min(total, max_keys)]], int(feasible.value)


def oracle_enum7(tables, target, mask, tuples, outer, middle, max_keys):
    """(total, first max_keys keys) of search_7lut's matches over the list `tuples` ((count, 7))."""
    lib = enum_oracle()
    tables, tp = S._u64(tables)
    target, gp = S._u64(target)
    mask, mp = S._u64(mask)
    lst = np.ascontiguousarray(tuples, dtype=np.uint16).reshape(-1, 7)
    keys = np.zeros(max(max_keys, 1), dtype=np.uint64)
    total = lib.orc_enum7(tp, gp, mp, lst.ctypes.data_as(u16p), lst.shape[0], S._order(outer),
                          S._order(middle), max_keys, keys.ctypes.data_as(u64p))
    return int(total), [int(k) for k in keys[:min(total, max_keys)]]


def unpack_list(packed):
    """The library's packed 63-bit list entries -> (count, 7) gate numbers."""
    p = np.asarray(packed, dtype=np.uint64)
    return np.stack([((p >> np.uint64(9 * (6 - i))) & np.uint64(0x1FF)).astype(np.uint16)
                     for i in range(7)], axis=1).reshape(-1, 7)


def orders(seed):
    """A 5-LUT order and a 7-LUT (outer, middle) pair from seeded shuffles."""
    rs = np.random.RandomState(seed)
    return (bytes(rs.permutation(256).astype(np.uint8)), bytes(rs.permutation(256).astype(np.uint8)),
            bytes(rs.permutation(256).astype(np.uint8)))


def expected_record(which, key, tables, target, mask, order, middle=None, tuple7=None):
    """What the record of `key` must hold, rebuilt on the host with the CPU oracle: (gates,
    func_outer, func_middle, func_inner, inner_seen); None if the key does not decompose."""
    lib = S.oracle_lib()
    if which == 5:
        rank, k, pos = key >> 12, (key >> 8) & 0xF, key & 0xFF
        comb = (C.c_uint16 * 5)()
        lib.orc_nth_combination(rank, tables.shape[0], 5, comb)
        row = S.order5_rows()[k]
        gates = [int(comb[row[i]]) for i in range(5)]
        fo, fm = order[pos], 0
        t1 = S.lut_table(fo, tables[gates[0]], tables[gates[1]], tables[gates[2]])
        t2 = tables[gates[3]]
    else:
        k, po, pm = (key >> 16) & 0x7F, (key >> 8) & 0xFF, key & 0xFF
        row = S.order7_rows()[k]
        gates = [int(tuple7[row[i]]) for i in range(7)]
        fo, fm = order[po], middle[pm]
        t1 = S.lut_table(fo, tables[gates[0]], tables[gates[1]], tables[gates[2]])
        t2 = S.lut_table(fm, tables[gates[3]], tables[gates[4]], tables[gates[5]])
    arrs = [S._u64(x) for x in (t1, t2, tables[gates[-1]], target, mask)]
    fi, seen = C.c_uint8(), C.c_uint8()
    if not lib.orc_solve_inner(*[a[1] for a in arrs], C.byref(fi), C.byref(seen)):
        return None
    return gates, int(fo), int(fm), int(fi.value), int(seen.value)


def record_fields(rec):
    width = int(rec["width"])
    return ([int(g) for g in rec["gates"][:width]], int(rec["func_outer"]), int(rec["func_middle"]),
            int(rec["func_inner"]), int(rec["inner_seen"]))


# ------------------------------------------------------------------------------------------------
# The depth filter on the host: what a filtered enumeration must keep, from the unfiltered records.

def record_depths(recs, depth):
    """match_depth of every record (all of one width), vectorised."""
    if len(recs) == 0:
        return np.zeros(0, dtype=np.int64)
    w = int(recs["width"][0])
    d = np.asarray(depth, dtype=np.int64)[recs["gates"][:, :w].astype(np.int64)]
    if w == 3:
        return 1 + d.max(axis=1)
    if w == 5:
        return 1 + np.maximum(1 + d[:, :3].max(axis=1), d[:, 3:].max(axis=1))
    return 1 + np.maximum(np.maximum(1 + d[:, :3].max(axis=1), 1 + d[:, 3:6].max(axis=1)), d[:, 6])


def bound_admits(d, bound, width):
    """Whether a gate set of depths d ((..., width)) has an ordering of depth <= bound, by the
    shortcut the filtered kernels prune with: no gate of depth >= bound, and at most two (width 5)
    or one (width 7) of depth bound - 1; width 3 has one ordering, of depth 1 + the deepest gate."""
    d = np.asarray(d, dtype=np.int64)
    fits = np.all(d < bound, axis=-1)
    if width == 3:
        return fits
    return fits & (np.sum(d >= bound - 1, axis=-1) <= {5: 2, 7: 1}[width])


def feasible5_under_bound(tabs, target, mask, inbits, depth, bound):
    """The feasible 5-combinations of the state with an ordering of depth <= bound, by brute force
    over all of C(n, 5): a combination is feasible iff no masked position of target 1 and masked
    position of target 0 share its gates' 5-bit pattern; combinations holding an excluded input
    bit do not count."""
    from itertools import combinations
    n = len(tabs)
    pos = np.arange(256)
    bits = np.stack([(np.asarray(t, dtype=np.uint64)[pos >> 6] >> (pos & 63).astype(np.uint64))
                     & np.uint64(1) for t in tabs]).astype(np.int64)                    # (n, 256)
    tg = (np.asarray(target, dtype=np.uint64)[pos >> 6] >> (pos & 63).astype(np.uint64)) & np.uint64(1)
    mk = (np.asarray(mask, dtype=np.uint64)[pos >> 6] >> (pos & 63).astype(np.uint64)) & np.uint64(1)
    p1, p0 = np.flatnonzero((mk == 1) & (tg == 1)), np.flatnonzero((mk == 1) & (tg == 0))
    combs = np.array(list(combinations(range(n), 5)), dtype=np.int64).reshape(-1, 5)
    combs = combs[~np.isin(combs, list(inbits)).any(axis=1)]
    combs = combs[bound_admits(np.asarray(depth, dtype=np.int64)[combs], bound, 5)]
    if len(combs) == 0:
        return 0
    pattern = sum(bits[combs[:, i]] << i for i in range(5))                         # (C, 256)
    rows = np.arange(len(combs))[:, None]
    ones = np.zeros((len(combs), 32), dtype=bool)
    zeros = np.zeros((len(combs), 32), dtype=bool)
    ones[rows, pattern[:, p1]] = True
    zeros[rows, pattern[:, p0]] = True
    return int(np.sum(~np.any(ones & zeros, axis=1)))
