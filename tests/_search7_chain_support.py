"""Test-side helpers of the first-chain search (sbg_search7_chain): the recorded search_7lut calls
that found nothing (tests/golden/run_*.bin), the function orders their recorded RNG gives, and the
CPU oracle's first chain key over each call's 7-LUT list (orc_filter7_range with inbits applied,
below the list cap at these sizes) from tests/enum_chain_oracle.c.

TEST INFRASTRUCTURE -- nothing under sboxgates_b200/ imports this module.
"""
import glob
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

import _enum7_all_reference as W
import _enum_chain_reference as CR
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200.rng import Xorshift1024

KEY_NONE = 2**64 - 1


def unmatched_calls():
    """[(run file, record index, Record)] of every recorded search_7lut call that found nothing."""
    out = []
    for path in sorted(glob.glob(os.path.join(S.GOLDEN, "run_*.bin"))):
        for i, rec in enumerate(S.read_records(path)):
            if rec.which == 7 and not rec.found:
                out.append((os.path.basename(path), i, rec))
    return out


def call_orders(rec):
    """The outer and middle orders search_7lut drew at the recorded call."""
    return sb.shuffled_orders7(Xorshift1024.from_state(rec.rng_s, rec.rng_p))


def oracle_first(tables, target, mask, tuples, orders):
    """(matches, first key idx<<24 | k<<16 | po<<8 | pm or KEY_NONE, L3's solved bits, seen cells)
    of the chain over `tuples` ((count, 7) uint16, list order), by the chain oracle."""
    lib = CR.chain_oracle()
    tables = np.ascontiguousarray(tables, dtype=np.uint64)
    target = np.ascontiguousarray(target, dtype=np.uint64)
    mask = np.ascontiguousarray(mask, dtype=np.uint64)
    tup = np.ascontiguousarray(tuples, dtype=np.uint16).reshape(-1, 7)
    o = [np.frombuffer(bytes(x), dtype=np.uint8).copy() for x in orders]
    key = np.zeros(1, dtype=np.uint64)
    inner = np.zeros(1, dtype=np.uint8)
    seen = np.zeros(1, dtype=np.uint8)
    total = lib.orc_enum7_chain(tables.ctypes.data_as(S.u64p), target.ctypes.data_as(S.u64p),
                                mask.ctypes.data_as(S.u64p), tup.ctypes.data_as(S.u16p), len(tup),
                                o[0].ctypes.data_as(S.u8p), o[1].ctypes.data_as(S.u8p), 1,
                                key.ctypes.data_as(S.u64p), inner.ctypes.data_as(S.u8p),
                                seen.ctypes.data_as(S.u8p))
    if total == 0:
        return 0, KEY_NONE, 0, 0
    return int(total), int(key[0]), int(inner[0]), int(seen[0])


def _record_first(rec):
    feas = W.feasible_tuples(rec.tables, rec.target, rec.mask, rec.inbits_list())
    assert len(feas) < sb.lut.SBG_LIST_CAP
    return oracle_first(rec.tables, rec.target, rec.mask, feas, call_orders(rec))


_FIRSTS = None


def recorded_firsts():
    """[(run file, record index, Record, oracle_first(...))] over every unmatched recorded call,
    computed once per process on a thread pool (the oracle releases the GIL)."""
    global _FIRSTS
    if _FIRSTS is None:
        calls = unmatched_calls()
        CR.chain_oracle()
        with ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
            firsts = list(ex.map(lambda c: _record_first(c[2]), calls))
        _FIRSTS = [c + (f,) for c, f in zip(calls, firsts)]
    return _FIRSTS


def rebuild_ok(luts, tables, target, mask):
    """Whether three LUTs in lut_search's form [(L1, a, b, c), (L2, ("new", 0), d, e),
    (L3, ("new", 1), f, g)] realise the target under the mask."""
    (f1, a, b, c), (f2, n0, d, e), (f3, n1, f, g) = luts
    assert n0 == ("new", 0) and n1 == ("new", 1)
    x1 = S.lut_table(f1, tables[a], tables[b], tables[c])
    x2 = S.lut_table(f2, x1, tables[d], tables[e])
    out = S.lut_table(f3, x2, tables[f], tables[g])
    return not np.any((out ^ np.asarray(target, dtype=np.uint64)) & np.asarray(mask, dtype=np.uint64))


def result_luts(res, rng_or_fill):
    """An SbgResult of search7_chain -> lut_search's form of its three LUTs."""
    return [(f,) + ins for f, ins in sb.chain_result_luts(res, rng_or_fill)]
