"""Test-side helpers of the enumeration tests: the CPU enumeration oracle (tests/enum_oracle.c,
compiled with oracle/sbg_oracle.c into a temporary directory on first use), its ctypes bindings,
the seeded states the tests share, and an independent check of one enumerated record.

TEST INFRASTRUCTURE -- nothing under sboxgates_b200/ imports this module.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import _support as S

HERE = os.path.dirname(os.path.abspath(__file__))
u64p, u16p, u8p, i8p = S.u64p, S.u16p, S.u8p, S.i8p

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
    _lib = lib
    return lib


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
