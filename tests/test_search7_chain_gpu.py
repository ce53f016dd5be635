"""GPU: the first-chain search (sbg_search7_chain, LutEngine.search7_chain) and the opt-in chain
stage of lut_search and of the drop-in (SBG_LUT_CHAIN=1).

- Every recorded search_7lut call that found nothing: found and key as the CPU chain oracle gives
  them over the call's list and recorded orders; every found chain rebuilds the target.
- Seeded states at every table width (256 / 128 / 64 / 32 positions), n up to 64, with and without
  excluded input bits, against the first record of the count-free chain enumeration; a dense state
  whose list is cut at 100,000 against the tuple-grouped enumeration restricted to the list.
- Planted chains at n = 96 and 160 (beyond the enumeration's n <= 64).
- Handle state: list reuse (no phase 1), rebuild after restaging, searches unchanged, the cursor
  ends, the work counters, bad arguments.
- lut_search(chain=True) on the recorded nodes; the drop-in on des_s1 under both seeds."""
import ctypes as C
import json
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import _search7_chain_support as CS
import _support as S
import bench
import sboxgates_b200 as sb
from sboxgates_b200 import lut, native
from test_dropin_gpu import _run, _verify
from test_enum_depth_gpu import _nw
from test_handle_calls_gpu import result_fields

pytestmark = pytest.mark.gpu

SBG_ERR_ARG, SBG_ERR_STATE = -1, -4
FULL = np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)
LOW24 = (1 << 24) - 1


def _orders(rs):
    return bytes(rs.permutation(256).astype(np.uint8)), bytes(rs.permutation(256).astype(np.uint8))


def _chain_target(rs, tabs, gates):
    f = [int(x) for x in rs.randint(1, 255, 3)]
    x1 = S.lut_table(f[0], *tabs[gates[:3]])
    return S.lut_table(f[2], S.lut_table(f[1], x1, tabs[gates[3]], tabs[gates[4]]),
                       tabs[gates[5]], tabs[gates[6]])


def _check_found(res, tables, target, mask):
    luts = CS.result_luts(res, sb.allowed_fill(res.func_inner, res.inner_seen))
    assert CS.rebuild_ok(luts, tables, target, mask), (hex(res.key), luts)
    assert res.index == res.key >> 24 and res.ordering == (res.key >> 16) & 0xFF
    assert (res.pos_outer, res.pos_middle) == ((res.key >> 8) & 0xFF, res.key & 0xFF)
    assert res.stale_outer == 0 and res.index < res.tuples_feasible


# ------------------------------------------------------------------------------------------------
# The recorded nodes.

def test_recorded_unmatched_calls_match_the_oracle(engine):
    firsts = CS.recorded_firsts()
    assert len(firsts) == 83
    found = 0
    for name, i, rec, (total, key, fi, seen) in firsts:
        outer, middle = CS.call_orders(rec)
        engine.load(rec.tables, rec.target, rec.mask, rec.inbits_list())
        res = engine.search7_chain(outer, middle)
        assert (bool(res.found), int(res.key)) == (total > 0, key), (name, i)
        if res.found:
            found += 1
            assert (res.func_outer, res.func_middle) == (outer[res.pos_outer],
                                                         middle[res.pos_middle])
            assert (res.func_inner, res.inner_seen) == (fi, seen)
            _check_found(res, rec.tables, rec.target, rec.mask)
    assert found == 6


# ------------------------------------------------------------------------------------------------
# Against the chain enumeration.

def _list(engine):
    """The installed list of the loaded problem, as (count, 7) gate arrays (phase 1 runs here)."""
    return np.array([lut.unpack_tuple7(p) for p in engine.filter7_part(0, 1)],
                    dtype=np.int64).reshape(-1, 7)


@pytest.mark.parametrize("depth", range(4))
def test_first_match_equals_the_enumeration(engine, depth):
    rs = np.random.RandomState(100 + depth)
    seen_found = seen_none = 0
    for trial in range(8):
        n = int(rs.choice([9, 12, 16, 24, 40, 64]))
        tabs = bench._state(n, int(rs.randint(1 << 30)))
        fixed = [(int(b), int(rs.randint(2))) for b in rs.choice(8, depth, replace=False)]
        mask = S.mux_mask(fixed)
        assert _nw(mask) == (8, 4, 2, 1)[depth]
        inbits = [b for b, _ in fixed] if trial % 2 else []
        allowed = [g for g in range(n) if g not in inbits]
        if trial % 3 != 2:
            tgt = _chain_target(rs, tabs, sorted(int(x) for x in rs.choice(allowed, 7, replace=False)))
        else:
            tgt = bench._rijndael_bit(int(rs.randint(8)))
        outer, middle = _orders(rs)
        engine.load(tabs, tgt, mask, inbits)
        lst = _list(engine)
        if len(lst) >= sb.lut.SBG_LIST_CAP:
            continue
        res = engine.search7_chain(outer, middle)
        e = engine.enumerate7_chain(outer, middle, 1, count=False)
        tag = (depth, trial, n, inbits)
        assert res.tuples_feasible == len(lst)
        if len(e.matches) == 0:
            assert not res.found and res.key == CS.KEY_NONE, tag
            seen_none += 1
            continue
        m = e.matches[0]
        combo = sorted(int(g) for g in m["gates"])
        idx = int(np.nonzero((lst == combo).all(axis=1))[0][0])
        assert res.found and res.key == (idx << 24) | (int(m["key"]) & LOW24), tag
        assert list(res.gates) == [int(g) for g in m["gates"]]
        assert (res.func_outer, res.func_middle, res.func_inner, res.inner_seen) == \
            (m["func_outer"], m["func_middle"], m["func_inner"], m["inner_seen"])
        _check_found(res, tabs, tgt, mask)
        seen_found += 1
    assert seen_found >= 2


def test_capped_list_equals_the_grouped_enumeration_on_the_list(engine):
    """A dense state whose list is cut at 100,000: the first chain is the smallest chain key among
    the list's combinations, from the tuple-grouped chain enumeration (one record per gate set, its
    smallest key) restricted to the ranks of list entries."""
    n = 48
    tabs = S.synthetic_state(n, seed=48)
    fixed = [(0, 1), (5, 0), (3, 1)]
    mask, inbits = S.mux_mask(fixed), [0, 5, 3]
    tgt = S.sbox_target(S.rijndael_sbox(), 0)
    outer, middle = _orders(np.random.RandomState(48))
    engine.load(tabs, tgt, mask, inbits)
    lst = _list(engine)
    assert len(lst) == sb.lut.SBG_LIST_CAP
    res = engine.search7_chain(outer, middle)
    ranks = CS.W.lex_ranks(lst, n)
    where = {int(r): i for i, r in enumerate(ranks)}
    try:
        engine.set_grouping("tuple")
        groups = engine.enumerate7_chain(outer, middle, 64, count=False)
    finally:
        engine.set_grouping(None)
    keys = [(where[int(k) >> 24] << 24) | (int(k) & LOW24) for k in groups.matches["key"]
            if int(k) >> 24 in where]
    assert keys, "no chain on the list"
    assert res.found and res.key == min(keys)
    _check_found(res, tabs, tgt, mask)
    assert res.tuples_feasible == sb.lut.SBG_LIST_CAP


@pytest.mark.parametrize("n", [96, 160])
def test_planted_chain_beyond_64_gates(engine, n):
    rs = np.random.RandomState(n)
    tabs = bench._state(n, n)
    late = sorted(int(x) for x in rs.choice(range(n - 24, n), 7, replace=False))
    tgt = _chain_target(rs, tabs, [late[i] for i in rs.permutation(7)])
    outer, middle = _orders(rs)
    engine.load(tabs, tgt, FULL, [])
    res = engine.search7_chain(outer, middle)
    assert 0 < res.tuples_feasible < sb.lut.SBG_LIST_CAP
    assert res.found
    _check_found(res, tabs, tgt, FULL)
    assert sorted(int(g) for g in res.gates) <= late


# ------------------------------------------------------------------------------------------------
# Handle state.

def _state14():
    rs = np.random.RandomState(14)
    tabs = S.synthetic_state(14, seed=1414)
    tgt = _chain_target(rs, tabs, [2, 4, 6, 8, 9, 11, 13])
    return tabs, tgt, S.mux_mask([(2, 1)]), [0], _orders(rs)


def test_handle_state(engine):
    tabs, tgt, mask, inb, (outer, middle) = _state14()
    engine.load(tabs, tgt, mask, inb)
    r1 = engine.search7(outer, middle)
    e1 = engine.enumerate7(outer, middle, 100)
    # after search7: the installed list, no phase 1
    before = engine.launches
    c1 = engine.search7_chain(outer, middle)
    reuse = engine.launches - before
    assert c1.found
    _check_found(c1, tabs, tgt, mask)
    assert (c1.tuples_feasible, c1.tuples_swept) == (r1.tuples_feasible, r1.tuples_swept)
    # the same state staged anew: phase 1 again, the same answer and counters
    engine.load(tabs, ~tgt, mask, inb)
    engine.load(tabs, tgt, mask, inb)
    before = engine.launches
    c2 = engine.search7_chain(outer, middle)
    rebuilt = engine.launches - before
    assert rebuilt > reuse
    assert result_fields(c1, 7) == result_fields(c2, 7)
    before = engine.launches
    engine.search7_chain(outer, middle)
    assert engine.launches - before == reuse
    # the searches and the list enumeration see what they saw before
    f = engine.finish7(r1.key, outer, middle)
    r2 = engine.search7(outer, middle)
    assert result_fields(r1, 7) == result_fields(f, 7) == result_fields(r2, 7)
    e2 = engine.enumerate7(outer, middle, 100)
    assert (e1.total, e1.matches.tobytes()) == (e2.total, e2.matches.tobytes())
    # another problem: its own list and answer
    tgt2 = S.sbox_target(S.rijndael_sbox(), 3)
    engine.load(tabs, tgt2, mask, inb)
    c3 = engine.search7_chain(outer, middle)
    feas = CS.W.feasible_tuples(tabs, tgt2, mask, inb)
    total, key, _, _ = CS.oracle_first(tabs, tgt2, mask, feas, (outer, middle))
    assert (bool(c3.found), int(c3.key), c3.tuples_feasible) == (total > 0, key, len(feas))
    # the call ends the cursor
    engine.enumerate7(outer, middle, 10)
    engine.fetch_matches(0, 1)
    engine.search7_chain(outer, middle)
    with pytest.raises(RuntimeError):
        engine.fetch_matches(0, 1)


def test_settings_are_not_read(engine):
    tabs, tgt, mask, inb, (outer, middle) = _state14()
    engine.load(tabs, tgt, mask, inb)
    plain = engine.search7_chain(outer, middle)
    try:
        engine.set_depth_filter(np.full(14, 50, dtype=np.uint16), 3)
        engine.set_function_filter([0], [0], [0])
        engine.set_grouping("tuple")
        assert result_fields(engine.search7_chain(outer, middle), 7) == result_fields(plain, 7)
    finally:
        engine.set_grouping(None)
        engine.clear_function_filter()
        engine.clear_depth_filter()


def test_bad_arguments(engine):
    lib = native.load_library()
    order = (C.c_uint8 * 256)(*range(256))
    bad = (C.c_uint8 * 256)(*([0] + list(range(255))))
    res = native.SbgResult()
    fresh = sb.LutEngine(0)
    try:
        assert lib.sbg_search7_chain(fresh._h, order, order, C.byref(res)) == SBG_ERR_STATE
    finally:
        fresh.close()
    engine.load(bench._state(6, 6), bench._rijndael_bit(0), FULL, [])
    assert lib.sbg_search7_chain(engine._h, order, order, C.byref(res)) == SBG_ERR_ARG
    engine.load(bench._state(12, 12), bench._rijndael_bit(0), FULL, [])
    assert lib.sbg_search7_chain(engine._h, bad, order, C.byref(res)) == SBG_ERR_ARG
    assert lib.sbg_search7_chain(engine._h, order, bad, C.byref(res)) == SBG_ERR_ARG
    assert lib.sbg_search7_chain(engine._h, order, order, None) == SBG_ERR_ARG
    assert lib.sbg_search7_chain(engine._h, order, order, C.byref(res)) == 0


# ------------------------------------------------------------------------------------------------
# lut_search(chain=True).

def test_lut_search_chain_stage_on_recorded_nodes(engine):
    chains = 0
    for name, i, rec, (total, key, fi, seen) in CS.recorded_firsts():
        tabs, inb = rec.tables, rec.inbits_list()
        order = list(range(rec.n))
        seed = np.random.RandomState(i).bytes(128)
        base_rng, rng = sb.Xorshift1024(seed), sb.Xorshift1024(seed)
        base = sb.lut_search(engine, tabs, rec.target, rec.mask, inb, order, base_rng)
        got = sb.lut_search(engine, tabs, rec.target, rec.mask, inb, order, rng, chain=True)
        assert base.stage == 0 and base.shape == "tree", (name, i)
        if total == 0:
            assert (got.stage, got.luts, got.shape) == (0, [], "tree"), (name, i)
            assert rng.draws == base_rng.draws == 768
            assert rng.next() == base_rng.next()
            continue
        chains += 1
        assert got.stage == 7 and got.shape == "chain", (name, i)
        assert CS.rebuild_ok(got.luts, tabs, rec.target, rec.mask)
        # the chain over the orders lut_search drew, with L3 filled by the next draw
        ahead = sb.Xorshift1024(seed)
        sb.shuffled_order(ahead)
        outer, middle = sb.shuffled_orders7(ahead)
        engine.load(tabs, rec.target, rec.mask, inb)
        res = engine.search7_chain(outer, middle)
        assert got.luts == CS.result_luts(res, ahead)
        assert rng.draws == 256 + 512 + (res.inner_seen != 0xFF)
        assert rng.next() == ahead.next()
    assert chains == 6


# ------------------------------------------------------------------------------------------------
# The drop-in.

# The drop-in is linked here from this tree's node-shim archive (sboxgates_b200/csrc/Makefile's
# `dropin` recipe, into a temporary directory): the chain stage lives in the shim, which is linked
# statically, so a binary under oracle/_ref/ linked before the shim changed would not have it.
PKG = os.path.join(S.ROOT, "sboxgates_b200")
SHIM = os.path.join(PKG, "libsbg_lutshim_node.a")
HOST_OBJS = [os.path.join(S.REF_DIR, f) for f in (
    "boolfunc.pic.o", "convert_graph.pic.o", "state.pic.o", "xml_mini.pic.o", "lut.node.o",
    "sboxgates.host.o")]
needs_objs = pytest.mark.skipif(
    not all(os.path.exists(p) for p in HOST_OBJS + [SHIM, os.path.join(S.REF_DIR, "sboxes")]),
    reason="the reference's host objects under oracle/_ref/ or the node shim are not built")


@pytest.fixture(scope="module")
def dropin_exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("dropin") / "sboxgates_gpu")
    subprocess.run([os.environ.get("CC", "gcc"), "-march=x86-64-v3", "-O2", "-g",
                    "-I", os.path.join(S.ORACLE_DIR, "stubs"),
                    "-I", os.path.join(PKG, "csrc", "xmlmini"), "-DSBGREF_WRAP_FOPEN",
                    os.path.join(S.ORACLE_DIR, "ref_glue.c")] + HOST_OBJS +
                   ["-Wl,--whole-archive", SHIM, "-Wl,--no-whole-archive", "-L" + PKG,
                    "-lsboxgates_b200", "-Wl,-rpath," + PKG, "-lstdc++", "-lpthread",
                    "-Wl,--wrap=fopen", "-o", out], check=True, capture_output=True)
    return out


def _chain_nodes(err):
    m = re.search(r"7-LUT chain (\d+)", err)
    assert m, err[-2000:]
    return int(m.group(1))


@needs_objs
@pytest.mark.parametrize("seed", ["seed1", "seed2"])
def test_dropin_chain_stage_on_des_s1(dropin_exe, seed):
    extra = {"SBG_LUT_CHAIN": "1"}
    with tempfile.TemporaryDirectory() as tmp:
        got, secs, err = _run(dropin_exe, "des_s1.txt", ["-l", "-o", "0"], seed, tmp,
                              extra_env=extra)
        assert got
        graph = _verify(tmp, got[-1], "des_s1.txt", [0])
        assert graph.num_luts == int(got[-1].split("-")[1])
    assert _chain_nodes(err) >= 1
    assert "7-LUT chain stage:" in err
    import torch
    if torch.cuda.device_count() >= 2:
        sharded = dict(extra, SBG_GPUS="2", SBG_SHARD_MIN5="0", SBG_SHARD_MIN7="0",
                       SBG_SHARD_MIN_LIST="0")
        with tempfile.TemporaryDirectory() as tmp:
            got2, _, err2 = _run(dropin_exe, "des_s1.txt", ["-l", "-o", "0"], seed, tmp,
                                 extra_env=sharded)
        assert got2 == got and "sharded search phases" in err2
    # without the variable: the reference's files, and no chain column
    names = json.load(open(os.path.join(S.GOLDEN, "xml_names.json")))
    with tempfile.TemporaryDirectory() as tmp:
        plain, _, err0 = _run(dropin_exe, "des_s1.txt", ["-l", "-o", "0"], seed, tmp)
    assert plain == names["des_s1.txt -l -o 0 %s" % seed]
    assert "7-LUT chain" not in err0
