"""Test-side reference of the shared-input two-LUT enumeration (sbg_enum4_shared), built from the
CPU oracle alone: every match of a state from tests/enum_shared_oracle.c (every 4-combination,
inbits and check_n_lut_possible(4) applied, then direct evaluation and orc_solve_inner), one
record per match assembled from the oracle's solved inner function.  Also the recorded
search_5lut calls that found nothing (tests/golden/run_*.bin) and the function order each drew.

TEST INFRASTRUCTURE -- nothing under sboxgates_b200/ imports this module.
"""
import ctypes as C
import glob
import os
import subprocess
import tempfile

import numpy as np

import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import MATCH_DTYPE
from sboxgates_b200.rng import Xorshift1024

HERE = os.path.dirname(os.path.abspath(__file__))
SHARED_ROWS = 12
KEY_NONE = 2**64 - 1
_lib = None


def shared_oracle():
    """Loads the shared-input oracle, compiling it first (once per process, outside the tree)."""
    global _lib
    if _lib is not None:
        return _lib
    out = os.path.join(tempfile.mkdtemp(prefix="sbg_shared_oracle_"), "libsharedoracle.so")
    cc = os.environ.get("CC", "gcc")
    subprocess.run([cc, "-O2", "-fPIC", "-shared", "-I", S.ORACLE_DIR, "-o", out,
                    os.path.join(HERE, "enum_shared_oracle.c"),
                    os.path.join(S.ORACLE_DIR, "sbg_oracle.c")], check=True, capture_output=True)
    lib = C.CDLL(out)
    lib.orc_shared_row.restype = None
    lib.orc_shared_row.argtypes = [C.c_int, C.POINTER(C.c_int)]
    lib.orc_enum4_shared.restype = C.c_uint64
    lib.orc_enum4_shared.argtypes = [S.u64p, C.c_int, S.u64p, S.u64p, C.POINTER(C.c_int8), S.u8p,
                                     C.c_uint64, S.u64p, S.u8p, S.u8p, S.u64p]
    _lib = lib
    return lib


def oracle_row(k):
    row = (C.c_int * 5)()
    shared_oracle().orc_shared_row(k, row)
    return [int(x) for x in row]


def rows():
    return np.array([oracle_row(k) for k in range(SHARED_ROWS)], dtype=np.int64)


def _inbits8(inbits):
    ib = np.full(8, -1, dtype=np.int8)
    for i, b in enumerate(inbits):
        ib[i] = b
    return ib


def shared_matches(tables, target, mask, inbits, order, cap=1 << 22):
    """(feasible 4-combinations, keys, L2's solved bits, seen cells) of every match, by the oracle;
    keys / bits beyond cap are not returned (the count is: len(keys) < total then)."""
    lib = shared_oracle()
    tables = np.ascontiguousarray(tables, dtype=np.uint64)
    target = np.ascontiguousarray(target, dtype=np.uint64)
    mask = np.ascontiguousarray(mask, dtype=np.uint64)
    ib = _inbits8(inbits)
    o = np.frombuffer(bytes(order), dtype=np.uint8).copy()
    keys = np.zeros(max(cap, 1), dtype=np.uint64)
    inner = np.zeros(max(cap, 1), dtype=np.uint8)
    seen = np.zeros(max(cap, 1), dtype=np.uint8)
    feas = C.c_uint64()
    total = lib.orc_enum4_shared(tables.ctypes.data_as(S.u64p), len(tables),
                                 target.ctypes.data_as(S.u64p), mask.ctypes.data_as(S.u64p),
                                 ib.ctypes.data_as(C.POINTER(C.c_int8)), o.ctypes.data_as(S.u8p),
                                 cap, keys.ctypes.data_as(S.u64p), inner.ctypes.data_as(S.u8p),
                                 seen.ctypes.data_as(S.u8p), C.byref(feas))
    m = min(int(total), cap)
    return int(feas.value), int(total), keys[:m], inner[:m], seen[:m]


def shared_reference(tables, target, mask, inbits, order, cap=1 << 22):
    """(feasible combinations, every match as MATCH_DTYPE records in key order) of a state; None
    if it has more than cap matches."""
    n = len(tables)
    feas, total, keys, inner, seen = shared_matches(tables, target, mask, inbits, order, cap)
    if total > cap:
        return None
    recs = np.zeros(len(keys), dtype=MATCH_DTYPE)
    if len(keys) == 0:
        return feas, recs
    ranks = (keys >> np.uint64(12)).astype(np.int64)
    combs = np.array([combination(int(r), n, 4) for r in ranks], dtype=np.int64).reshape(-1, 4)
    k = ((keys >> np.uint64(8)) & np.uint64(0xF)).astype(np.int64)
    g5 = np.take_along_axis(combs, rows()[k], axis=1)
    recs["key"] = keys
    recs["gates"][:, :5] = g5
    o = np.frombuffer(bytes(order), dtype=np.uint8)
    recs["func_outer"] = o[(keys & np.uint64(0xFF)).astype(np.int64)]
    recs["func_inner"] = inner
    recs["inner_seen"] = seen
    recs["width"] = 4
    recs["shape"] = 2
    return feas, recs


def combination(rank, n, t):
    """The combination of lexicographic rank `rank` among C(n, t)."""
    out, x = [], 0
    from math import comb
    for pos in range(t):
        while True:
            c = comb(n - x - 1, t - pos - 1)
            if rank < c:
                break
            rank -= c
            x += 1
        out.append(x)
        x += 1
    return out


def combination_rank(c, n):
    from math import comb
    t, r, prev = len(c), 0, -1
    for pos, x in enumerate(c):
        for y in range(prev + 1, x):
            r += comb(n - y - 1, t - pos - 1)
        prev = x
    return r


def shared_depths(recs, depth):
    """The depth of each record: 1 + max(1 + max(Da, Db, Dc), Du, Dv)."""
    d = np.asarray(depth, dtype=np.int64)[recs["gates"][:, :5].astype(np.int64)]
    return 1 + np.maximum(1 + d[:, :3].max(axis=1), d[:, 3:5].max(axis=1))


def rebuild_ok(f1, f2, gates, tables, target, mask):
    """Whether L1 = f1 over gates[0..2] and L2 = f2 over (L1, gates[3], gates[4]) realise the target
    under the mask."""
    g = [tables[int(x)] for x in gates]
    x1 = S.lut_table(int(f1), g[0], g[1], g[2])
    out = S.lut_table(int(f2), x1, g[3], g[4])
    return not np.any((out ^ np.asarray(target, dtype=np.uint64)) & np.asarray(mask, dtype=np.uint64))


def unmatched_calls():
    """[(run file, record index, Record)] of every recorded search_5lut call that found nothing."""
    out = []
    for path in sorted(glob.glob(os.path.join(S.GOLDEN, "run_*.bin"))):
        for i, rec in enumerate(S.read_records(path)):
            if rec.which == 5 and not rec.found:
                out.append((os.path.basename(path), i, rec))
    return out


def call_order(rec):
    """The function order search_5lut drew at the recorded call."""
    return sb.shuffled_order(Xorshift1024.from_state(rec.rng_s, rec.rng_p))


def oracle_first(rec):
    """(matches, first key or KEY_NONE, L2's solved bits, seen cells, feasible) of a recorded
    call's state under its order."""
    feas, total, keys, inner, seen = shared_matches(rec.tables, rec.target, rec.mask,
                                                    rec.inbits_list(), call_order(rec), cap=1)
    if total == 0:
        return 0, KEY_NONE, 0, 0, feas
    return total, int(keys[0]), int(inner[0]), int(seen[0]), feas
