"""CPU: the shared-input two-LUT enumeration's interface (sbg_enum4_shared / sbg_search4_shared)
without a device -- the header and the bindings, the row table, the key and record layout, depths
and grouping ids on hand-built records, and the test-side oracle (tests/enum_shared_oracle.c)
against a direct numpy restatement on small states and on the recorded search_5lut calls that
found nothing."""
import itertools
import os
import re
import subprocess
from collections import Counter

import numpy as np
import pytest

import _enum_shared_reference as R
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import lut, native


def test_header_declares_shared_and_native_binds_it(tmp_path):
    header = open(os.path.join(S.ROOT, "include", "sboxgates_b200.h")).read()
    for name in ("sbg_enum4_shared", "sbg_search4_shared", "sbg_shared_row"):
        assert re.search(r"\bint %s\(" % name, header)
        assert name in native.SIGNATURES
    src = tmp_path / "shape.c"
    src.write_text('#include <stdio.h>\n#include "sboxgates_b200.h"\n'
                   'int main(void) {\n  printf("%d\\n", SBG_SHAPE_SHARED);\n  return 0;\n}\n')
    exe = tmp_path / "shape"
    subprocess.run([os.environ.get("CC", "gcc"), "-I", os.path.join(S.ROOT, "include"), str(src),
                    "-o", str(exe)], check=True, capture_output=True)
    shared = int(subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout)
    assert shared == native.SBG_SHAPE_SHARED == sb.SBG_SHAPE_SHARED == 2
    # the cursor's lifetime paragraph names the new calls
    assert "sbg_search4_shared" in header[header.index("Cursor lifetime"):]


def test_shared_rows_against_definition():
    rows = [sb.shared_row(k) for k in range(12)]
    expect = []
    for j in range(4):
        l1 = [p for p in range(4) if p != j]
        for q in range(3):
            expect.append(l1 + sorted((l1[q], j)))
    assert rows == expect
    assert [R.oracle_row(k) for k in range(12)] == rows
    # every row reads all four positions, one of L1's twice
    for r in rows:
        assert sorted(set(r)) == [0, 1, 2, 3] and len(set(r[:3]) & set(r[3:])) == 1
    for bad in (-1, 12):
        with pytest.raises(ValueError):
            sb.shared_row(bad)


def _record(key, gates, fo, fi, seen):
    r = np.zeros(1, dtype=sb.MATCH_DTYPE)[0]
    r["key"], r["gates"][:5], r["func_outer"] = key, gates, fo
    r["func_inner"], r["inner_seen"], r["width"], r["shape"] = fi, seen, 4, native.SBG_SHAPE_SHARED
    return r


def test_key_record_depth_and_groups():
    # C(500, 4) < 2^32: the rank, row and position read as a 5-LUT key
    from math import comb
    assert comb(500, 4) < 2**32
    key = (comb(500, 4) - 1) << 12 | 11 << 8 | 255
    assert sb.decode_key5(key) == (comb(500, 4) - 1, 11, 255)
    rec = _record(key, [2, 3, 4, 1, 3], 21, 0x0F, 0xFF)
    depth = np.zeros(8, dtype=np.int64)
    depth[[1, 2, 3, 4]] = [5, 1, 2, 0]
    # 1 + max(1 + max(D2, D3, D4), D1, D3): D1 = 5 counts once
    assert sb.match_depth(rec, depth) == 6
    assert R.shared_depths(np.array([rec]), depth)[0] == 6
    assert sb.match_group(key, 4, "shape", shape="shared") == key >> 8
    assert sb.match_group(key, 4, "tuple", shape="shared") == key >> 12
    assert sb.match_group(key, 4, None, shape="shared") == key
    for w, sh in ((4, "tree"), (5, "shared"), (7, "shared")):
        with pytest.raises(ValueError):
            sb.match_group(key, w, "shape", shape=sh)
    # the record reads as a 5-LUT record: ret = [L1, L2, a, b, c, u, v, 0, 0, 0]
    assert sb.match_to_ret(rec, sb.Xorshift1024(b"\x01" * 128)) == [21, 0x0F, 2, 3, 4, 1, 3, 0, 0, 0]


def _direct(tables, target, mask, inbits, order):
    """Every match by a numpy restatement of the definition: per 4-combination, row and L1, L2 is
    solvable iff no cell (x1, u, v) holds a masked 1 and a masked 0."""
    n = len(tables)
    bits = np.unpackbits(np.asarray(tables, dtype="<u8").view(np.uint8), bitorder="little")
    bits = bits.reshape(n, 256).astype(bool)
    tb = np.unpackbits(np.asarray(target, dtype="<u8").view(np.uint8), bitorder="little")
    mb = np.unpackbits(np.asarray(mask, dtype="<u8").view(np.uint8), bitorder="little")
    on, off = (mb & tb).astype(bool), (mb & ~tb & 1).astype(bool)
    funcs = np.array([[(f >> c) & 1 for c in range(8)] for f in bytes(order)], dtype=bool)
    keys, feasible = [], 0
    for rank, c in enumerate(itertools.combinations(range(n), 4)):
        if any(g in inbits for g in c):
            continue
        cell4 = sum(bits[g].astype(int) << (3 - i) for i, g in enumerate(c))
        if any((on & (cell4 == v)).any() and (off & (cell4 == v)).any() for v in range(16)):
            continue
        feasible += 1
        for k in range(12):
            g5 = [c[p] for p in sb.shared_row(k)]
            cell1 = (bits[g5[0]].astype(int) << 2) | (bits[g5[1]].astype(int) << 1) | bits[g5[2]]
            x1 = funcs[:, cell1]                                   # (256 po, 256 positions)
            cell2 = (x1.astype(int) << 2) | (bits[g5[3]].astype(int) << 1) | bits[g5[4]]
            ok = np.ones(256, dtype=bool)
            for v in range(8):
                ok &= ~(((cell2 == v) & on).any(axis=1) & ((cell2 == v) & off).any(axis=1))
            keys += [rank << 12 | k << 8 | po for po in np.flatnonzero(ok)]
    return feasible, keys


@pytest.mark.parametrize("n,seed,positions,inbits", [(6, 1, 16, []), (7, 2, 24, [0]),
                                                     (8, 3, 12, [1, 5]), (9, 4, 32, [])])
def test_oracle_against_direct_restatement(n, seed, positions, inbits):
    rng = np.random.RandomState(seed)
    tables = S.synthetic_state(n, seed=seed)
    target = S.lut_table(int(rng.randint(256)), tables[n - 1], tables[n - 2], tables[1]) \
        ^ np.uint64(int(rng.randint(2)))
    mask = np.zeros(4, dtype=np.uint64)
    for p in rng.choice(256, positions, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    order = sb.shuffled_order(sb.Xorshift1024(rng.bytes(128)))
    feas, keys = _direct(tables, target, mask, inbits, order)
    ofeas, total, okeys, inner, seen = R.shared_matches(tables, target, mask, inbits, order)
    assert (ofeas, total, [int(k) for k in okeys]) == (feas, len(keys), keys)
    assert total > 0
    # and every record rebuilds
    _, recs = R.shared_reference(tables, target, mask, inbits, order)
    for rec in recs[:: max(1, len(recs) // 50)]:
        # the solved bits with zeros in the unseen cells complete L2
        assert R.rebuild_ok(rec["func_outer"], rec["func_inner"], rec["gates"][:5], tables, target,
                            mask)


def test_recorded_unmatched_search5_calls():
    """Which of the recorded search_5lut calls that found nothing have a shared-input circuit, and
    the hand-checked witness of crypto1_fc seed 1 (n = 5, gates {1, 2, 3, 4}, L1 = 21 over
    (2, 3, 4), L2 over (x1, 1, 3))."""
    calls = R.unmatched_calls()
    per_run, with_match = Counter(), Counter()
    witness = False
    for name, _, rec in calls:
        per_run[name] += 1
        feas, total, keys, _, _ = R.shared_matches(rec.tables, rec.target, rec.mask,
                                                    rec.inbits_list(), R.call_order(rec),
                                                    cap=1 << 20)
        if total:
            with_match[name] += 1
        if name == "run_crypto1_fc_seed1.bin" and rec.n == 5:
            order = R.call_order(rec)
            for key in keys:
                key = int(key)
                if key >> 12 == 4 and (key >> 8) & 15 == 1 and order[key & 255] == 21:
                    witness = True
        if rec.n <= 8:   # small enough for the restatement
            assert _direct(rec.tables, rec.target, rec.mask, rec.inbits_list(),
                           R.call_order(rec)) == (feas, [int(k) for k in keys])
    assert witness
    assert sum(per_run.values()) == 192
    assert dict(per_run) == {"run_crypto1_fc_seed1.bin": 7, "run_crypto1_fc_seed2.bin": 6,
                             "run_des_s1_seed1.bin": 48, "run_des_s1_seed2.bin": 48,
                             "run_rijndael_seed1.bin": 46, "run_sodark_seed1.bin": 37}
    assert dict(with_match) == {"run_crypto1_fc_seed1.bin": 3, "run_crypto1_fc_seed2.bin": 3,
                                "run_des_s1_seed1.bin": 14, "run_des_s1_seed2.bin": 14,
                                "run_rijndael_seed1.bin": 10, "run_sodark_seed1.bin": 15}


def test_lut_search_signature_and_shim_switch():
    import inspect
    assert inspect.signature(sb.lut_search).parameters["shared"].default is False
    shim = open(os.path.join(S.ROOT, "sboxgates_b200", "csrc", "lut_shim.c")).read()
    assert 'getenv("SBG_LUT_SHARED")' in shim and "sbg_search4_shared" in shim
    assert lut.LutEngine.enumerate4_shared and lut.LutEngine.search4_shared
