#!/usr/bin/env python3
"""Randomised differential test on the GPU (minutes, not part of pytest): for random states / masks /
excluded bits it checks that
  * every phase-1 form (position-major with 4- and 5-gate prefixes, packed and unpacked, with and
    without programmatic dependent launch) returns the same hit list, equal to the CPU oracle's where
    that is affordable;
  * sharded phase 1 (3 parts) merges to the same list;
  * search_5lut: fused kernel == two kernels == 3 parts, and == oracle for small n;
  * search_7lut: one-call path == step-by-step path == 4 parts.
usage: stress_gpu.py [cases] [seed]"""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200.rng import Xorshift1024


def engine(**env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return sb.LutEngine(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


cases = int(sys.argv[1]) if len(sys.argv) > 1 else 60
rs = np.random.RandomState(int(sys.argv[2]) if len(sys.argv) > 2 else 1)
engines = {"pm4": engine(SBG_PM_PREFIX=4), "pm5": engine(SBG_PM_PREFIX=5), "plain": engine(),
           "pm4_unpacked": engine(SBG_PM_PREFIX=4, SBG_PACKED=0)}
engines["plain"].set_timing(True)   # timed launches are stream-ordered, without programmatic dependent launch
e5 = {"fused": engine(SBG_SEARCH5="fused"), "two": engine(SBG_SEARCH5="two")}
e7_plain = engine(SBG_DECOMP_FILTER=0)   # phase 2 without the lane-parallel stage-1 filter
sbox = S.rijndael_sbox()
t_start = time.time()
stats = {"cases": 0, "oracle_lists": 0, "oracle_searches": 0, "hits": 0, "found5": 0, "found7": 0}
for ci in range(cases):
    n = int(rs.choice([7, 8, 9, 11, 14, 17, 20, 24, 28, 31, 32, 33, 36, 40, 47, 48, 56, 63, 64, 65, 72]))
    tabs = S.synthetic_state(n, seed=int(rs.randint(1 << 30)), num_inputs=min(8, n))
    kind = rs.randint(0, 3)
    if kind == 0:
        depth = int(rs.randint(0, 5))
        fixed = [(int(b), int(rs.randint(0, 2))) for b in rs.choice(8, depth, replace=False)]
        mask = S.mux_mask(fixed)
        inb = [b for b, _ in fixed if b < n]
    else:
        pc = int(rs.choice([5, 8, 13, 21, 32, 33, 50, 64, 65, 100, 128, 129, 200]))
        mask = np.zeros(4, dtype=np.uint64)
        for p in rs.choice(256, pc, replace=False):
            mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
        inb = [int(x) for x in rs.choice(min(8, n), int(rs.randint(0, 3)), replace=False)]
    tgt = S.sbox_target(sbox, int(rs.randint(0, 8))) if rs.randint(0, 2) else \
        S.lut_table(int(rs.randint(1, 255)), tabs[rs.randint(n)], tabs[rs.randint(n)], tabs[rs.randint(n)])
    lists = {}
    for name, eng in engines.items():
        eng.load(tabs, tgt, mask, inb)
        lists[name] = eng.filter7_part(0, 1)
    ref = lists["pm4"]
    for name, l in lists.items():
        assert np.array_equal(l, ref), (ci, n, name, len(l), len(ref))
    eng = engines["pm4"] if n < 64 else engines["pm5"]
    parts = np.sort(np.concatenate([eng.filter7_part(p, 3) for p in range(3)]))[:100000]
    assert np.array_equal(parts, ref), (ci, n, "parts")
    if n <= 24:
        want, _ = S.oracle_filter7(tabs, tgt, mask, inb)
        assert [sb.lut.unpack_tuple7(p) for p in ref] == want.tolist(), (ci, n, "oracle list")
        stats["oracle_lists"] += 1
    stats["hits"] += len(ref)
    # search_5lut
    seed = rs.bytes(128)
    order = sb.shuffled_order(Xorshift1024(seed))
    keys = []
    for name, eng5 in e5.items():
        eng5.load(tabs, tgt, mask, inb)
        keys.append(eng5.search5_part(0, 1, order))
    e5["two"].load(tabs, tgt, mask, inb)
    keys.append(min(e5["two"].search5_part(p, 3, order) for p in range(3)))
    assert len(set(keys)) == 1, (ci, n, "search5 keys", keys)
    stats["found5"] += keys[0] != sb.lut.SBG_KEY_NONE
    if n <= 16:
        assert S.oracle_search5_key(tabs, tgt, mask, inb, order) == keys[0], (ci, n, "oracle key5")
    # search_7lut
    outer, middle = sb.shuffled_orders7(Xorshift1024(seed))
    eng.load(tabs, tgt, mask, inb)
    whole = eng.search7(outer, middle)
    cnt = eng.filter7_keep_local()
    k1 = eng.decomp7_part(0, 1, outer, middle)
    k4 = min(eng.decomp7_part(p, 4, outer, middle) for p in range(4))
    e7_plain.load(tabs, tgt, mask, inb)
    plain = e7_plain.search7(outer, middle)
    assert whole.key == k1 == k4 == plain.key, (ci, n, "search7 keys", whole.key, k1, k4, plain.key)
    stats["found7"] += bool(whole.found)
    if n <= 13 and (whole.found or cnt <= 6):
        tuples = np.array([sb.lut.unpack_tuple7(p) for p in ref], dtype=np.uint16).reshape(-1, 7)
        assert S.oracle_decomp7_key(tabs, tgt, mask, tuples, outer, middle) == k1 or \
            (k1 == sb.lut.SBG_KEY_NONE and S.oracle_decomp7_key(tabs, tgt, mask, tuples, outer, middle) == (1 << 64) - 1), (ci, n)
        stats["oracle_searches"] += 1
    stats["cases"] += 1
print("stress ok:", stats, "%.1f s" % (time.time() - t_start))
