"""CPU: the first-chain search's interface (sbg_search7_chain) without a device -- the header and
the binding, lut_search's chain switch, chain_result_luts on hand-made results, and the CPU oracle's
first chain key on every recorded search_7lut call that found nothing (the fixture the GPU tests
compare against)."""
import ctypes as C
import inspect
import os
import re
import subprocess

import numpy as np
import pytest

import _search7_chain_support as CS
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native


def test_header_declares_the_call(tmp_path):
    header = open(os.path.join(S.ROOT, "include", "sboxgates_b200.h")).read()
    assert re.search(r"\bint sbg_search7_chain\(sbg_handle \*h, const uint8_t \*outer_order",
                     header)
    # sbg_result::ordering holds the chain row; the call ends the cursor
    assert re.search(r"int32_t ordering;.{0,120}sbg_search7_chain:\s+the chain row, 0\.\.209",
                     header, re.S)
    lifetime = header[header.index("Cursor lifetime"):header.index("Without a cursor")]
    assert "sbg_search7_chain" in lifetime.split("keep it")[0]
    # the declaration compiles against the documented argument types
    src = tmp_path / "decl.c"
    src.write_text('#include "sboxgates_b200.h"\n'
                   "int (*fn)(sbg_handle *, const uint8_t *, const uint8_t *, sbg_result *) = "
                   "sbg_search7_chain;\n"
                   "int key_none_is_max[SBG_KEY_NONE == UINT64_MAX ? 1 : -1];\n")
    subprocess.run([os.environ.get("CC", "gcc"), "-Werror", "-I", os.path.join(S.ROOT, "include"),
                    "-c", str(src), "-o", str(tmp_path / "decl.o")], check=True,
                   capture_output=True)


def test_ctypes_signature():
    restype, args = native.SIGNATURES["sbg_search7_chain"]
    assert restype is C.c_int
    assert args == [C.c_void_p, native.u8p, native.u8p, C.POINTER(native.SbgResult)]
    assert native.SIGNATURES["sbg_search7_chain"] == native.SIGNATURES["sbg_search7"]


def test_lut_search_chain_switch():
    params = inspect.signature(sb.lut_search).parameters
    assert list(params)[-1] == "chain" and params["chain"].default is False
    assert sb.LutSearchResult(0).shape == "tree"
    assert sb.LutSearchResult(7, [], None, "chain").shape == "chain"
    assert callable(sb.LutEngine.search7_chain)


def _result(gates, f1, f2, tables, target, mask):
    res = native.SbgResult()
    x1 = S.lut_table(f1, *tables[gates[:3]])
    x2 = S.lut_table(f2, x1, tables[gates[3]], tables[gates[4]])
    ok, fi, seen = sb.solve_inner(x2, tables[gates[5]], tables[gates[6]], target, mask)
    assert ok
    res.found, res.func_outer, res.func_middle = 1, f1, f2
    res.func_inner, res.inner_seen = fi, seen
    for i, g in enumerate(gates):
        res.gates[i] = g
    return res


def test_chain_result_luts_rebuild_the_target():
    tabs = S.synthetic_state(16, seed=21)
    rs = np.random.RandomState(3)
    for trial in range(20):
        gates = [int(x) for x in rs.choice(16, 7, replace=False)]
        f = [int(x) for x in rs.randint(1, 255, 3)]
        x1 = S.lut_table(f[0], *tabs[gates[:3]])
        tgt = S.lut_table(f[2], S.lut_table(f[1], x1, tabs[gates[3]], tabs[gates[4]]),
                          tabs[gates[5]], tabs[gates[6]])
        mask = S.mux_mask([(int(b), int(rs.randint(2))) for b in rs.choice(8, trial % 4,
                                                                          replace=False)])
        res = _result(gates, f[0], f[1], tabs, tgt, mask)
        rng = sb.Xorshift1024(rs.bytes(128))
        ref = rng.copy()
        luts = CS.result_luts(res, rng)
        assert luts[0] == (f[0], gates[0], gates[1], gates[2])
        assert luts[1] == (f[1], ("new", 0), gates[3], gates[4])
        assert luts[2][1:] == (("new", 1), gates[5], gates[6])
        # one draw iff a cell of L3 is unseen, as get_lut_function fills
        assert rng.draws - ref.draws == (0 if res.inner_seen == 0xFF else 1)
        assert CS.rebuild_ok(luts, tabs, tgt, mask)
        # a fill that disagrees with the solved bits is refused; the smallest agreeing one rebuilds
        fill = sb.allowed_fill(res.func_inner, res.inner_seen)
        assert CS.rebuild_ok(CS.result_luts(res, fill), tabs, tgt, mask)
        if res.inner_seen:
            with pytest.raises(ValueError):
                sb.chain_result_luts(res, res.func_inner ^ (res.inner_seen & -res.inner_seen))
    res.found = 0
    with pytest.raises(ValueError):
        sb.chain_result_luts(res, 0)


def test_recorded_unmatched_calls_and_their_first_chains():
    """The 83 recorded search_7lut calls that found nothing: exactly 6 have a chain over their list,
    the 2nd, 3rd and 4th such call of des_s1.txt -l -o 0 under each seed, and every first key
    decodes to a chain that rebuilds the target."""
    firsts = CS.recorded_firsts()
    assert len(firsts) == 83
    found = [(name, i) for name, i, rec, f in firsts if f[0] > 0]
    assert found == [("run_des_s1_seed1.bin", 39), ("run_des_s1_seed1.bin", 62),
                     ("run_des_s1_seed1.bin", 86), ("run_des_s1_seed2.bin", 39),
                     ("run_des_s1_seed2.bin", 62), ("run_des_s1_seed2.bin", 86)]
    keys = {(name, i): f[1] for name, i, rec, f in firsts if f[0] > 0}
    assert keys[("run_des_s1_seed1.bin", 39)] == 0x14783405
    assert keys[("run_des_s1_seed1.bin", 62)] == 0xEACABB5
    assert keys[("run_des_s1_seed1.bin", 86)] == 0xE5B0428
    for name, i, rec, (total, key, fi, seen) in firsts:
        if total == 0:
            assert key == CS.KEY_NONE
            continue
        feas = CS.W.feasible_tuples(rec.tables, rec.target, rec.mask, rec.inbits_list())
        idx, k, po, pm = sb.decode_key7_chain(key)
        gates = [int(feas[idx][p]) for p in sb.chain_row(k)]
        outer, middle = CS.call_orders(rec)
        res = _result(gates, outer[po], middle[pm], rec.tables, rec.target, rec.mask)
        assert (res.func_inner, res.inner_seen) == (fi, seen)
        assert CS.rebuild_ok(CS.result_luts(res, sb.allowed_fill(fi, seen)), rec.tables,
                             rec.target, rec.mask)
