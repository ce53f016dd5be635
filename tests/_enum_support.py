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
