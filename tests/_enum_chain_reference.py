"""Test-side reference of the 7-LUT chain enumeration (sbg_enum7_chain), built from the CPU oracle
alone: the feasible 7-combinations of the whole space (orc_filter7_range, inbits applied, as for
sbg_enum7_all), every chain match of them from tests/enum_chain_oracle.c (direct evaluation and
orc_solve_inner), each key's tuple index replaced by the combination's rank among all C(n,7), and
one record per match assembled from the oracle's solved inner function.

TEST INFRASTRUCTURE -- nothing under sboxgates_b200/ imports this module.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import _enum7_all_reference as W
import _support as S
from sboxgates_b200 import MATCH_DTYPE

HERE = os.path.dirname(os.path.abspath(__file__))
CHAIN_ROWS = 210
LOW24 = np.uint64((1 << 24) - 1)
_lib = None


def chain_oracle():
    """Loads the chain oracle, compiling it first (once per process, outside the tree)."""
    global _lib
    if _lib is not None:
        return _lib
    out = os.path.join(tempfile.mkdtemp(prefix="sbg_chain_oracle_"), "libchainoracle.so")
    cc = os.environ.get("CC", "gcc")
    subprocess.run([cc, "-O2", "-fPIC", "-shared", "-I", S.ORACLE_DIR, "-o", out,
                    os.path.join(HERE, "enum_chain_oracle.c"),
                    os.path.join(S.ORACLE_DIR, "sbg_oracle.c")], check=True, capture_output=True)
    lib = C.CDLL(out)
    lib.orc_chain_row.restype = None
    lib.orc_chain_row.argtypes = [C.c_int, C.POINTER(C.c_int)]
    lib.orc_enum7_chain.restype = C.c_uint64
    lib.orc_enum7_chain.argtypes = [S.u64p, S.u64p, S.u64p, S.u16p, C.c_int64, S.u8p, S.u8p,
                                    C.c_uint64, S.u64p, S.u8p, S.u8p]
    _lib = lib
    return lib


def oracle_row(k):
    row = (C.c_int * 7)()
    chain_oracle().orc_chain_row(k, row)
    return [int(x) for x in row]


ROWS = None


def rows():
    global ROWS
    if ROWS is None:
        ROWS = np.array([oracle_row(k) for k in range(CHAIN_ROWS)], dtype=np.int64)
    return ROWS


def chain_matches(tables, target, mask, tuples, orders, cap=1 << 22):
    """Every chain match of `tuples` ((count, 7) uint16, ascending gates): (keys with the tuple's
    index as high field, solved inner bits, seen cells); None if there are more than cap."""
    lib = chain_oracle()
    tables = np.ascontiguousarray(tables, dtype=np.uint64)
    target = np.ascontiguousarray(target, dtype=np.uint64)
    mask = np.ascontiguousarray(mask, dtype=np.uint64)
    tuples = np.ascontiguousarray(tuples, dtype=np.uint16).reshape(-1, 7)
    keys = np.zeros(cap, dtype=np.uint64)
    inner = np.zeros(cap, dtype=np.uint8)
    seen = np.zeros(cap, dtype=np.uint8)
    o = [np.frombuffer(bytes(x), dtype=np.uint8).copy() for x in orders]
    total = lib.orc_enum7_chain(tables.ctypes.data_as(S.u64p), target.ctypes.data_as(S.u64p),
                                mask.ctypes.data_as(S.u64p), tuples.ctypes.data_as(S.u16p),
                                len(tuples), o[0].ctypes.data_as(S.u8p),
                                o[1].ctypes.data_as(S.u8p), cap, keys.ctypes.data_as(S.u64p),
                                inner.ctypes.data_as(S.u8p), seen.ctypes.data_as(S.u8p))
    if total > cap:
        return None
    return keys[:total], inner[:total], seen[:total]


def chain_reference(tables, target, mask, inbits, orders, cap=1 << 22):
    """(feasible combinations, every chain match as MATCH_DTYPE records in key order) of a state;
    None if it has more than cap matches."""
    n = len(tables)
    feas = W.feasible_tuples(tables, target, mask, inbits)
    found = chain_matches(tables, target, mask, feas, orders, cap)
    if found is None:
        return None
    keys, inner, seen = found
    recs = np.zeros(len(keys), dtype=MATCH_DTYPE)
    if len(keys) == 0:
        return feas, recs
    idx = (keys >> np.uint64(24)).astype(np.int64)
    ranks = W.lex_ranks(feas, n).astype(np.uint64)
    recs["key"] = (ranks[idx] << np.uint64(24)) | (keys & LOW24)
    k = ((keys >> np.uint64(16)) & np.uint64(0xFF)).astype(np.int64)
    recs["gates"] = np.take_along_axis(feas.astype(np.int64)[idx], rows()[k], axis=1)
    o = [np.frombuffer(bytes(x), dtype=np.uint8) for x in orders]
    recs["func_outer"] = o[0][((keys >> np.uint64(8)) & np.uint64(0xFF)).astype(np.int64)]
    recs["func_middle"] = o[1][(keys & np.uint64(0xFF)).astype(np.int64)]
    recs["func_inner"] = inner
    recs["inner_seen"] = seen
    recs["width"] = 7
    recs["shape"] = 1
    return feas, recs


def chain_depths(recs, depth):
    """The depth of each chain record: 1 + max(1 + max(1 + max(Da, Db, Dc), Dd, De), Df, Dg)."""
    d = np.asarray(depth, dtype=np.int64)[recs["gates"].astype(np.int64)]
    return 1 + np.maximum(np.maximum(1 + np.maximum(1 + d[:, :3].max(axis=1), d[:, 3:5].max(axis=1)),
                                     d[:, 5]), d[:, 6])


def rebuild_ok(rec, tables, target, mask, fill):
    """Whether L1, L2 and L3 = fill (which must agree with the record's solved bits) realise the
    target under the mask."""
    g = [tables[int(x)] for x in rec["gates"]]
    if (int(fill) & int(rec["inner_seen"])) != int(rec["func_inner"]):
        return False
    x1 = S.lut_table(int(rec["func_outer"]), g[0], g[1], g[2])
    x2 = S.lut_table(int(rec["func_middle"]), x1, g[3], g[4])
    out = S.lut_table(int(fill), x2, g[5], g[6])
    return bool(np.all(((out ^ np.asarray(target, dtype=np.uint64)) & mask) == 0))
