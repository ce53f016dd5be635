"""Test-side helpers of the 3-LUT enumeration tests: the CPU oracle orc_enum3_range
(tests/enum3_oracle.c, compiled with oracle/sbg_oracle.c into a temporary directory on first use)
and its piece-parallel wrapper.

TEST INFRASTRUCTURE -- nothing under sboxgates_b200/ imports this module.
"""
import ctypes as C
import os
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

import _enum_support as E
import _support as S

HERE = os.path.dirname(os.path.abspath(__file__))
u64p, u16p = S.u64p, S.u16p

_lib = None


def enum3_oracle():
    """Loads the 3-LUT enumeration oracle, compiling it first (once per process, outside the
    tree)."""
    global _lib
    if _lib is not None:
        return _lib
    out = os.path.join(tempfile.mkdtemp(prefix="sbg_enum3_oracle_"), "libenum3oracle.so")
    cc = os.environ.get("CC", "gcc")
    subprocess.run([cc, "-O2", "-fPIC", "-shared", "-I", S.ORACLE_DIR, "-o", out,
                    os.path.join(HERE, "enum3_oracle.c"), os.path.join(S.ORACLE_DIR, "sbg_oracle.c")],
                   check=True, capture_output=True)
    lib = C.CDLL(out)
    lib.orc_enum3_range.restype = C.c_uint64
    lib.orc_enum3_range.argtypes = [u64p, C.c_int, u64p, u64p, u16p, C.c_int64, C.c_int64,
                                    C.c_uint64, u64p]
    _lib = lib
    return lib


def enum3_range(tables, target, mask, order, max_keys, lo=0, hi=None, piece=None):
    """(total, first max_keys keys) of the 3-LUT scan's matches among the position triples of ranks
    [lo, hi) (default: all of C(n,3)): orc_enum3_range over pieces on a thread pool, totals summed,
    key lists concatenated.  Every match is a feasible triple, so the total is also the feasible
    count."""
    lib = enum3_oracle()
    tables, tp = S._u64(tables)
    target, gp = S._u64(target)
    mask, mp = S._u64(mask)
    n = tables.shape[0]
    go = np.ascontiguousarray(order, dtype=np.uint16)
    if hi is None:
        hi = n * (n - 1) * (n - 2) // 6

    def run(r):
        keys = np.zeros(max(max_keys, 1), dtype=np.uint64)
        total = lib.orc_enum3_range(tp, n, gp, mp, go.ctypes.data_as(u16p), r[0], r[1], max_keys,
                                    keys.ctypes.data_as(u64p))
        return int(total), [int(k) for k in keys[:min(total, max_keys)]]
    rs = E.pieces(lo, hi, piece or max(1, -(-(hi - lo) // (4 * E.workers()))))
    with ThreadPoolExecutor(max_workers=E.workers()) as pool:
        parts = list(pool.map(run, rs))
    keys = [k for p in parts for k in p[1]][:max_keys]
    return sum(p[0] for p in parts), keys
