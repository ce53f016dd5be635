"""GPU: the CUDA path (through the C ABI) against the reference's golden outputs and the oracle."""
import glob
import os

import numpy as np
import pytest

import _support as S
import sboxgates_b200 as sb
from sboxgates_b200.rng import Xorshift1024

pytestmark = pytest.mark.gpu

FULL = np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)


def _run_gpu(engine, rec_or_case, rng):
    which, tables, target, mask, inbits = rec_or_case
    fn = sb.search_5lut if which == 5 else sb.search_7lut
    return fn(engine, tables, target, mask, inbits, rng)


def _replay(engine, path, limit_ns=None):
    n = 0
    for rec in S.read_records(path):
        rng = Xorshift1024.from_state(rec.rng_s, rec.rng_p)
        res = _run_gpu(engine, (rec.which, rec.tables, rec.target, rec.mask, rec.inbits_list()), rng)
        assert res.found == rec.found, (path, n)
        assert res.ret == rec.ret, (path, n, res.ret, rec.ret)
        assert rng.draws == rec.draws, (path, n)
        n += 1
    return n


def test_reference_cases(engine):
    """Synthetic + edge cases answered by the reference's own object code (incl. stale-cache)."""
    assert _replay(engine, os.path.join(S.GOLDEN, "ref_cases.bin")) >= 60


@pytest.mark.parametrize("name", ["run_crypto1_fa_seed1.bin", "run_crypto1_fb_seed1.bin",
                                  "run_crypto1_fc_seed1.bin", "run_crypto1_fc_seed2.bin",
                                  "run_des_s1_seed1.bin", "run_des_s1_seed2.bin",
                                  "run_rijndael_seed1.bin", "run_sodark_seed1.bin"])
def test_recorded_reference_runs(engine, name):
    """Every search call of seeded reference runs, including the ones that took the reference
    minutes: same found / ret[10] / RNG draw count."""
    path = os.path.join(S.GOLDEN, name)
    assert os.path.exists(path), "golden fixture missing: run oracle/gen_golden.py"
    if os.path.getsize(path) == 0:
        assert _scan_reference_graph(engine, name) > 0
    else:
        assert _replay(engine, path) > 0


def _words(table):
    return np.array([(table >> (64 * w)) & (2**64 - 1) for w in range(4)], dtype=np.uint64)


def _scan_reference_graph(engine, name):
    """A run whose recording is empty never reached search_5lut: every LUT of the graph it wrote
    came from a 3-LUT scan over the gates before it (lut.c:501-523).  The stored graph must be the
    file that run wrote (xml_names.json) and compute its S-box bit, and for each of its LUTs the
    GPU's scan over the preceding gates, in a shuffled order, must return the first triple that
    realises the LUT's table, with the CPU oracle's function and RNG draws.  Returns the LUT count."""
    import json
    from sboxgates_b200 import graph as G
    sbox_name, seed = name[len("run_"):-len(".bin")].rsplit("_", 1)
    want = json.load(open(os.path.join(S.GOLDEN, "xml_names.json")))["%s.txt -l %s" % (sbox_name,
                                                                                        seed)]
    paths = glob.glob(os.path.join(S.GOLDEN, "graphs", sbox_name + "_*.xml"))
    assert [os.path.basename(p)[len(sbox_name) + 1:] for p in paths] == want
    graph = G.load_graph(paths[0])
    sbox, _ = G.load_sbox(os.path.join(S.GOLDEN, "sboxes", sbox_name + ".txt"))
    assert G.verify_graph(graph, sbox, require_bits=[0]) == [0]
    rs = np.random.RandomState(len(graph.gates))
    luts = 0
    for idx, gate in enumerate(graph.gates):
        if gate.type != "LUT":
            continue
        tabs = np.stack([_words(g.table) for g in graph.gates[:idx]])
        tgt = _words(gate.table)
        order = [int(x) for x in rs.permutation(idx)]
        seed_bytes = rs.bytes(128)
        o_rng, g_rng = S.OrcRng.from_seed(seed_bytes), Xorshift1024(seed_bytes)
        first = None
        for i in range(idx):
            for k in range(i + 1, idx):
                for m in range(k + 1, idx):
                    trip = [tabs[order[i]], tabs[order[k]], tabs[order[m]]]
                    if first is None and S.oracle_check(3, tgt, FULL, trip):
                        ok, func = S.oracle_get_lut_function(*trip, tgt, FULL, o_rng)
                        if ok:
                            first = (func, order[i], order[k], order[m])
        got = sb.lut_search(engine, tabs, tgt, FULL, [], order, g_rng, allow5=False, allow7=False)
        assert got.stage == 3 and got.luts[0] == first, (name, idx, got.luts, first)
        assert g_rng.draws == o_rng.draws
        luts += 1
    assert luts == graph.num_luts
    return luts


def test_random_vs_oracle(engine):
    """Seeded random states against the CPU oracle at sizes it finishes in seconds."""
    sbox = S.rijndael_sbox()
    rs = np.random.RandomState(42)
    for i in range(40):
        n = int(rs.choice([7, 8, 9, 10, 11, 12, 13]))
        tabs = S.synthetic_state(n, seed=900 + i, num_inputs=min(8, n))
        fixed = [(int(b), int(rs.randint(0, 2))) for b in rs.choice(8, int(rs.randint(0, 4)),
                                                                    replace=False)]
        mask = S.mux_mask(fixed)
        inb = [b for b, _ in fixed if b < n]
        tgt = S.sbox_target(sbox, int(rs.randint(0, 8)))
        for which in (5, 7):
            seed = rs.bytes(128)
            o_rng = S.OrcRng.from_seed(seed)
            g_rng = Xorshift1024(seed)
            found, ret, st = S.oracle_search(which, tabs, tgt, mask, inb, o_rng)
            if which == 7 and st.tuples_feasible > 12 and not found:
                continue  # oracle too slow; covered by properties below
            res = _run_gpu(engine, (which, tabs, tgt, mask, inb), g_rng)
            assert (res.found, res.ret) == (found, ret), (i, which, n, fixed)
            assert g_rng.draws == o_rng.draws
            if which == 7:
                assert res.tuples_feasible == st.tuples_feasible


def test_phase2_filter_forms_agree_with_the_oracle(monkeypatch):
    """Phase 2 decides most (tuple, outer triple) pairs with a filter that gives every outer triple
    of a tuple a lane of its own (conflict graph of the 8 outer patterns, 2-colourable or not) and
    the rest with the warp-cooperative ballot form; SBG_DECOMP_FILTER=0 leaves everything to the
    ballot form.  Either way results must equal the CPU oracle's on recorded reference calls (incl.
    the stale-cache cases) and on random states."""
    for mode in ("0", "1"):
        eng = _fresh_engine(monkeypatch, SBG_DECOMP_FILTER=mode)
        n_cases = _replay(eng, os.path.join(S.GOLDEN, "ref_cases.bin"))
        assert n_cases >= 60
        assert _replay(eng, os.path.join(S.GOLDEN, "run_sodark_seed1.bin")) > 0
        sbox = S.rijndael_sbox()
        rs = np.random.RandomState(4242)
        for i in range(25):
            n = int(rs.choice([9, 10, 11, 12, 13]))
            tabs = S.synthetic_state(n, seed=5000 + i)
            fixed = [(int(b), int(rs.randint(0, 2))) for b in rs.choice(8, int(rs.randint(1, 5)),
                                                                        replace=False)]
            mask, inb = S.mux_mask(fixed), [b for b, _ in fixed if b < n]
            tgt = S.sbox_target(sbox, int(rs.randint(0, 8)))
            seed = rs.bytes(128)
            o_rng = S.OrcRng.from_seed(seed)
            found, ret, st = S.oracle_search(7, tabs, tgt, mask, inb, o_rng)
            if st.tuples_feasible > 40 and not found:
                continue   # too slow for the oracle
            res = sb.search_7lut(eng, tabs, tgt, mask, inb, Xorshift1024(seed))
            assert (res.found, res.ret) == (found, ret), (mode, i, n, fixed)
        eng.close()


def test_filter7_list_matches_oracle(engine):
    sbox = S.rijndael_sbox()
    for i, (n, fixed) in enumerate([(12, [(0, 1), (3, 0)]), (14, [(1, 1), (2, 1), (6, 0)]),
                                    (16, [(5, 0)]), (11, [(0, 0), (1, 0), (2, 0), (3, 0)])]):
        tabs = S.synthetic_state(n, seed=50 + i)
        mask = S.mux_mask(fixed)
        inb = [b for b, _ in fixed]
        tgt = S.sbox_target(sbox, i)
        want, _ = S.oracle_filter7(tabs, tgt, mask, inb)
        engine.load(tabs, tgt, mask, inb)
        got = engine.filter7_part(0, 1)
        assert [sb.lut.unpack_tuple7(p) for p in got] == want.tolist()


def _verify_result(which, tabs, tgt, mask, res):
    """The reference's own acceptance test of a result (lut.c:573-576, 617-621)."""
    r = res.ret
    if which == 5:
        t_outer = S.lut_table(r[0], tabs[r[2]], tabs[r[3]], tabs[r[4]])
        t_inner = S.lut_table(r[1], t_outer, tabs[r[5]], tabs[r[6]])
    else:
        t_outer = S.lut_table(r[0], tabs[r[3]], tabs[r[4]], tabs[r[5]])
        t_mid = S.lut_table(r[1], tabs[r[6]], tabs[r[7]], tabs[r[8]])
        t_inner = S.lut_table(r[2], t_outer, t_mid, tabs[r[9]])
    assert not np.any((t_inner ^ tgt) & mask)


def test_large_states_properties(engine):
    """At sizes the oracle cannot reach: planted circuits must be found, results must verify, the
    answer must not depend on mask compression (an all-ones mask with a masked-equivalent target)
    or on how the work is split into parts."""
    rs = np.random.RandomState(77)
    for n in (40, 64, 96):
        tabs = S.synthetic_state(n, seed=n)
        g5 = [int(x) for x in rs.choice(n, 5, replace=False)]
        t_outer = S.lut_table(0x6A, tabs[g5[0]], tabs[g5[1]], tabs[g5[2]])
        tgt = S.lut_table(0xC5, t_outer, tabs[g5[3]], tabs[g5[4]])
        seed = rs.bytes(128)
        res = sb.search_5lut(engine, tabs, tgt, FULL, [], Xorshift1024(seed))
        assert res.found
        _verify_result(5, tabs, tgt, FULL, res)
        # minimality: the planted combination cannot precede the reported one
        assert sorted(res.gates) <= sorted(g5)
        # split into 3 parts -> same key
        order = sb.shuffled_order(Xorshift1024(seed))
        engine.load(tabs, tgt, FULL, [])
        keys = [engine.search5_part(p, 3, order) for p in range(3)]
        assert min(keys) == res.key


def test_planted_7lut_large(engine):
    rs = np.random.RandomState(78)
    for n in (24, 32):
        tabs = S.synthetic_state(n, seed=1000 + n)
        g7 = [int(x) for x in rs.choice(n, 7, replace=False)]
        t_outer = S.lut_table(0x96, tabs[g7[0]], tabs[g7[1]], tabs[g7[2]])
        t_mid = S.lut_table(0xE8, tabs[g7[3]], tabs[g7[4]], tabs[g7[5]])
        tgt = S.lut_table(0xCA, t_outer, t_mid, tabs[g7[6]])
        seed = rs.bytes(128)
        res = sb.search_7lut(engine, tabs, tgt, FULL, [], Xorshift1024(seed))
        assert res.found
        _verify_result(7, tabs, tgt, FULL, res)
        assert sorted(res.gates) <= sorted(g7)
        # sharded: per-part lists merge to the same list, per-part keys to the same minimum
        outer, middle = sb.shuffled_orders7(Xorshift1024(seed))
        engine.load(tabs, tgt, FULL, [])
        whole = engine.filter7_part(0, 1)
        parts = [engine.filter7_part(p, 4) for p in range(4)]
        merged = np.sort(np.concatenate(parts))[:100000]
        assert merged.tolist() == whole.tolist()
        engine.set_list7(np.concatenate(parts[::-1]))
        keys = [engine.decomp7_part(p, 4, outer, middle) for p in range(4)]
        assert min(keys) == res.key


def _fresh_engine(monkeypatch, **env):
    """A new handle created under the given environment (the library reads its tuning knobs when a
    handle is created / on first use)."""
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))
    return sb.LutEngine(0)


def test_paths_agree(engine):
    """The one-call search (sbg_search7: on-device sort, single synchronisation) and the
    step-by-step one (filter part -> list -> decomposition part -> finish) return the same result;
    so do short lists (on-device bitonic sort) and long ones (radix sort)."""
    sbox = S.rijndael_sbox()
    rs = np.random.RandomState(5)
    for n, fixed in [(14, [(0, 1)]), (20, [(1, 0), (6, 1)]), (28, [(0, 0), (2, 1), (5, 0)]),
                     (36, [(3, 1), (4, 1), (7, 0)]), (33, [])]:
        tabs = S.synthetic_state(n, seed=700 + n)
        mask = S.mux_mask(fixed)
        inb = [b for b, _ in fixed]
        tgt = S.sbox_target(sbox, int(rs.randint(0, 8)))
        seed = rs.bytes(128)
        outer, middle = sb.shuffled_orders7(Xorshift1024(seed))
        engine.load(tabs, tgt, mask, inb)
        whole = engine.search7(outer, middle)
        count = engine.filter7_keep_local()
        key = engine.decomp7_part(0, 1, outer, middle)
        step = engine.finish7(key, outer, middle)
        assert (whole.found, whole.key, list(whole.gates), whole.func_inner, whole.inner_seen) == \
            (step.found, step.key, list(step.gates), step.func_inner, step.inner_seen)
        assert whole.tuples_feasible == count


def test_launch_modes_agree(engine):
    """The kernels of a chain are launched with programmatic dependent launch (each starts while its
    predecessor drains); with SBG_TIMING=1 they are plainly stream-ordered, with events between them;
    SBG_PACKED=0 keeps phase 1 on one part per accumulator register throughout.  A single search_7lut
    cuts phase 1's 4-gate prefixes into weighted tickets (groups of pairs); two chains of a batch share
    the device and take two whole prefixes per ticket instead.  Hit lists, search results and -- for
    sweeps that run to the end -- the T-unit counts must be identical in all modes, and each chain of
    the batch must return the single call's search_7lut result."""
    import subprocess
    import sys
    code = (
        "import sys, numpy as np; sys.path[:0]=[%r, %r]\n"
        "import _support as S, sboxgates_b200 as sb\n"
        "eng = sb.LutEngine(0); sbox = S.rijndael_sbox(); out = []\n"
        "for n, fixed in [(18, []), (24, [(0,1)]), (30, [(1,0),(4,1)]), (40, [(2,1),(3,0),(6,1)]), (44, [(5, 1)])]:\n"
        "    tabs, tgt, mask, inb = S.synthetic_state(n, seed=n), S.sbox_target(sbox, n %% 8), S.mux_mask(fixed), [b for b, _ in fixed]\n"
        "    eng.load(tabs, tgt, mask, inb)\n"
        "    out.append(eng.filter7_part(0, 1).tolist())\n"
        "    seed = np.random.RandomState(n).bytes(128)\n"
        "    for fn in (sb.search_5lut, sb.search_7lut):\n"
        "        r = fn(eng, tabs, tgt, mask, inb, sb.Xorshift1024(seed)); out.append([int(r.found), -1 if (r.found or r.tuples_feasible >= 100000) else int(r.tuples_swept)] + [int(x) for x in r.ret])\n"
        "    outer, middle = sb.shuffled_orders7(sb.Xorshift1024(seed))\n"
        "    eng.stage(0, tabs, tgt, mask, inb); eng.stage(1, tabs, tgt, mask, inb)\n"
        "    for slot, b in enumerate(eng.search_batch([dict(slot=s, outer=outer, middle=middle) for s in (0, 1)])):\n"
        "        got = (bool(b.r7.found), int(b.r7.key), int(b.r7.tuples_feasible), -1 if out[-1][1] < 0 else int(b.r7.tuples_swept))\n"
        "        assert got == (r.found, r.key, r.tuples_feasible, out[-1][1]), (n, slot, got, r)\n"
        "import json; print(json.dumps(out))\n" % (S.ROOT, os.path.join(S.ROOT, "tests")))
    outs = {}
    for mode, env in (("pdl", {}), ("timed", {"SBG_TIMING": "1"}), ("unpacked", {"SBG_PACKED": "0"})):
        res = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env),
                             capture_output=True, text=True)
        assert res.returncode == 0, (mode, res.stderr[-3000:])
        outs[mode] = res.stdout.strip().splitlines()[-1]
    assert len(set(outs.values())) == 1, sorted(outs)
    import json
    assert sum(len(x) for x in json.loads(outs["pdl"])[0::3]) > 0


def test_hit_buffer_overflow_is_retried(monkeypatch):
    """With a tiny hit buffer phase 1 overflows; the bounded-parallelism retry must still deliver
    the exact list (first SBG_LIST_CAP feasible tuples in lexicographic order)."""
    import subprocess
    import sys
    code = (
        "import sys, numpy as np; sys.path[:0]=[%r, %r]\n"
        "import _support as S, sboxgates_b200 as sb\n"
        "eng = sb.LutEngine(0); sbox = S.rijndael_sbox()\n"
        "tabs = S.synthetic_state(48, seed=48); mask = S.mux_mask([(0,1),(5,0),(3,1)])\n"
        "eng.load(tabs, S.sbox_target(sbox, 0), mask, [0,5,3])\n"
        "lst = eng.filter7_part(0, 1)\n"
        "parts = np.sort(np.concatenate([eng.filter7_part(p, 3) for p in range(3)]))[:100000]\n"
        "import hashlib; print(len(lst), hashlib.sha1(lst.tobytes()).hexdigest(), hashlib.sha1(parts.tobytes()).hexdigest())\n"
        % (S.ROOT, os.path.join(S.ROOT, "tests")))
    outs = []
    for cap in ("", "200000"):
        env = dict(os.environ)
        if cap:
            env["SBG_HITS_CAP"] = cap
        res = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True,
                             check=True)
        outs.append(res.stdout.strip().splitlines()[-1])
    assert outs[0] == outs[1]
    n_hits, whole_hash, parts_hash = outs[0].split()
    assert int(n_hits) == 100000          # the case really hits the cap
    assert whole_hash == parts_hash       # three parts (some of them retried) merge to the same list


def test_chunked_and_prefix_forms_agree():
    """Phase 1 hands its work out as (prefix, chunk) items over the allowed gates (head, or everything
    in the overflow retry) and as batches of whole prefixes; SBG_HEAD = 0 / 1 / 2 forces no head / a
    head / chunk items throughout.  Lists -- whole and merged from 3 parts -- must be identical, on
    dense states (small masks: the cap is reached inside the first prefixes, low gates excluded) and
    on a sparse one; the dense 5-gate-prefix case is also checked against the oracle's first entries."""
    import json
    import subprocess
    import sys
    code = (
        "import sys, hashlib, json, numpy as np; sys.path[:0]=[%r, %r]\n"
        "import _support as S, sboxgates_b200 as sb\n"
        "eng = sb.LutEngine(0); sbox = S.rijndael_sbox(); out = []\n"
        "cases = [(56, [(0,1),(5,0),(3,1)]), (72, [(0,1),(5,0),(3,1),(6,1)]), (50, [(2,1),(7,0)]),\n"
        "         (130, [(1,1),(2,0),(4,1),(7,1)]), (130, [(0,0),(1,1),(3,1)])]\n"
        "for n, fixed in cases:\n"
        "    eng.load(S.synthetic_state(n, seed=n), S.sbox_target(sbox, n %% 8), S.mux_mask(fixed), [b for b, _ in fixed])\n"
        "    whole = eng.filter7_part(0, 1)\n"
        "    parts = np.sort(np.concatenate([eng.filter7_part(p, 3) for p in range(3)]))[:100000]\n"
        "    r5 = sb.search_5lut(eng, S.synthetic_state(n, seed=n), S.sbox_target(sbox, n %% 8), S.mux_mask(fixed), [b for b, _ in fixed],\n"
        "                        sb.Xorshift1024(np.random.RandomState(n).bytes(128)))\n"
        "    out.append([len(whole), hashlib.sha1(whole.tobytes()).hexdigest(), hashlib.sha1(parts.tobytes()).hexdigest(),\n"
        "                whole[:2000].tolist() if n == 130 and fixed[0][0] == 1 else [], [int(r5.found)] + [int(x) for x in r5.ret]])\n"
        "print(json.dumps(out))\n" % (S.ROOT, os.path.join(S.ROOT, "tests")))
    outs = {}
    for mode in ("0", "1", "2"):
        env = dict(os.environ, SBG_HEAD=mode)
        res = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True,
                             check=True)
        outs[mode] = json.loads(res.stdout.strip().splitlines()[-1])
    assert outs["0"] == outs["1"] == outs["2"]
    lens = [c[0] for c in outs["1"]]
    assert lens[0] == lens[1] == lens[3] == lens[4] == 100000 and 0 < lens[2] < 100000
    assert all(c[1] == c[2] for c in outs["1"])
    n, fixed = 130, [(1, 1), (2, 0), (4, 1), (7, 1)]
    want, _ = S.oracle_filter7(S.synthetic_state(n, seed=n), S.sbox_target(S.rijndael_sbox(), n % 8),
                               S.mux_mask(fixed), [b for b, _ in fixed], cap=2000)
    assert [sb.lut.unpack_tuple7(p) for p in outs["1"][3][3]] == want.tolist()
    # search_5lut on the same states (n = 130: fused kernel, with and without its chunked head)
    # against the oracle where that is quick (dense states: an early match)
    for idx, (n, fixed) in ((3, (130, [(1, 1), (2, 0), (4, 1), (7, 1)])),):
        o_rng = S.OrcRng.from_seed(np.random.RandomState(n).bytes(128))
        found, ret, _ = S.oracle_search(5, S.synthetic_state(n, seed=n),
                                        S.sbox_target(S.rijndael_sbox(), n % 8), S.mux_mask(fixed),
                                        [b for b, _ in fixed], o_rng)
        assert outs["1"][idx][4] == [int(found)] + [int(x) for x in ret]


def _max_size_case():
    rs = np.random.RandomState(500)
    tabs = S.synthetic_state(500, seed=500)
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, 6, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    # (gate 0 must not be excluded: the CPU oracle, like the reference, would step through all
    # C(499,6) tuples that start with it one by one)
    return rs, tabs, S.sbox_target(S.rijndael_sbox(), 2), mask, [5]


def test_maximum_size_state(engine):
    """MAX_GATES = 500 (state.h:26): 16-word gate vectors, 9-bit packed gate numbers, the 100,000
    cap reached inside the first prefixes.  Very sparse mask, so most tuples are feasible and both the
    oracle (asked for the first 3,000 entries only) and the GPU stop early."""
    rs, tabs, tgt, mask, inb = _max_size_case()
    want, _ = S.oracle_filter7(tabs, tgt, mask, inb, cap=3000)
    assert len(want) == 3000
    engine.load(tabs, tgt, mask, inb)
    got = engine.filter7_part(0, 1)
    assert len(got) == 100000 and np.all(got[1:] > got[:-1])
    assert [sb.lut.unpack_tuple7(p) for p in got[:3000]] == want.tolist()
    for which in (5, 7):
        seed = rs.bytes(128)
        o_rng = S.OrcRng.from_seed(seed)
        found, ret, _ = S.oracle_search(which, tabs, tgt, mask, inb, o_rng)
        g_rng = Xorshift1024(seed)
        res = _run_gpu(engine, (which, tabs, tgt, mask, inb), g_rng)
        assert (res.found, res.ret, g_rng.draws) == (found, ret, o_rng.draws)
        assert found
