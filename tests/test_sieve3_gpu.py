"""GPU: phase 1's pair sieve read from the per-3-gate-prefix table (k_sieve3) gives the same 7-LUT
lists as phase 1 without the sieve (SBG_SIEVE=0) and as the CPU oracle.  The sieve runs forced on
(SBG_SIEVE=2) so that every table width is covered: n = 8 ... 60, masks of 1, 2, 4 and 8 words (random
masks with a padded last word, mux masks), excluded input bits incl. gate 0; a single chain (weighted
tickets), sharded parts, a batch of chains (concurrent tickets of two prefixes), a 4,096-entry ticket
table (several launches, the table built by the first), a small hit buffer (the overflow retry
reuses the table), and one handle whose problems shrink and grow n (the table grows)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import _support as S
import test_filter_windows_gpu as W

pytestmark = pytest.mark.gpu


def _engine(sieve):
    import sboxgates_b200 as sb
    old = os.environ.get("SBG_SIEVE")
    os.environ["SBG_SIEVE"] = sieve
    try:
        return sb.LutEngine(0)
    finally:
        if old is None:
            os.environ.pop("SBG_SIEVE", None)
        else:
            os.environ["SBG_SIEVE"] = old


@pytest.fixture(scope="module")
def engines():
    on, off = _engine("2"), _engine("0")
    yield on, off
    on.close()
    off.close()


def _mask(spec, seed):
    return W._random_mask(spec, seed) if isinstance(spec, int) else S.mux_mask(spec)


# (n, mux-fixed (bit, value) pairs or the size of a random mask, excluded input bits, oracle entries
# compared or None = all).  Random masks of 20 / 45 / 100 / 200 positions: 1 / 2 / 4 / 8 words, the
# last one partly padding.
CASES = [
    (8, [], [], None),
    (9, [(3, 1)], [3], None),
    (14, 20, [0], None),
    (24, 45, [], None),
    (27, 100, [1, 2], None),
    (33, 200, [0], None),
    (40, [], [], None),
    (40, [(2, 0)], [2], None),
    (44, 100, [5], None),
    (52, [(0, 1), (6, 0)], [0, 6], None),
    (56, [(3, 0), (4, 1), (5, 1)], [], 3000),
    (60, [(1, 0)], [1], None),
    (60, [(2, 1), (4, 0), (7, 1)], [2, 4, 7], None),
]


def _states():
    sbox = S.rijndael_sbox()
    return [(n, S.synthetic_state(n, seed=9800 + i), S.sbox_target(sbox, (n + i) % 8),
             _mask(spec, 9900 + i), inb, cmp) for i, (n, spec, inb, cmp) in enumerate(CASES)]


def test_sieve3_lists_match_unsieved_and_oracle(engines):
    on, off = engines
    for n, tabs, tgt, mask, inb, cmp in _states():
        on.load(tabs, tgt, mask, inb)
        off.load(tabs, tgt, mask, inb)
        got, ref = on.filter7_part(0, 1), off.filter7_part(0, 1)
        assert np.array_equal(got, ref), (n, inb, len(got), len(ref))
        want = S.oracle_filter7(tabs, tgt, mask, inb, cap=cmp or W.CAP)[0]
        if cmp is not None:
            assert len(want) == cmp and len(got) >= cmp, (n, inb, len(got))
            got = got[:cmp]
        assert np.array_equal(got, W._pack(want)), (n, inb)


@pytest.mark.parametrize("nparts", [2, 3])
def test_sieve3_sharded_parts_match(engines, nparts):
    on, off = engines
    for n, tabs, tgt, mask, inb, _ in _states()[5:]:
        on.load(tabs, tgt, mask, inb)
        off.load(tabs, tgt, mask, inb)
        for part in range(nparts):
            got, ref = on.filter7_part(part, nparts), off.filter7_part(part, nparts)
            assert np.array_equal(got, ref), (n, nparts, part, len(got), len(ref))


def test_sieve3_batch_equals_single_calls(engines):
    """Chains sharing the device (two prefixes per ticket) == the same searches one at a time, with
    and without the sieve."""
    on, off = engines
    rs = np.random.RandomState(9950)
    states = _states()[3:11]
    jobs = []
    for slot, (n, tabs, tgt, mask, inb, _) in enumerate(states):
        on.stage(slot, tabs, tgt, mask, inb)
        off.stage(slot, tabs, tgt, mask, inb)
        jobs.append(dict(slot=slot, order5=bytes(rs.permutation(256).astype(np.uint8)),
                         outer=bytes(rs.permutation(256).astype(np.uint8)),
                         middle=bytes(rs.permutation(256).astype(np.uint8))))
    res = on.search_batch(jobs)
    for eng in (on, off):
        for j, r in zip(jobs, res):
            eng.use(j["slot"])
            r5 = eng.search5(j["order5"])
            assert (r.r5.found, r.r5.key, r.r5.tuples_feasible) == (r5.found, r5.key, r5.tuples_feasible)
            if not r5.found:
                r7 = eng.search7(j["outer"], j["middle"])
                assert (r.r7.found, r.r7.key, r.r7.tuples_feasible, list(r.r7.gates)) \
                    == (r7.found, r7.key, r7.tuples_feasible, list(r7.gates))
                if r7.tuples_feasible < W.CAP:
                    assert r.r7.tuples_swept == r7.tuples_swept


def test_sieve3_table_follows_n_on_one_handle(engines):
    """n shrinks, then grows past what the table was allocated for: every list stays exact."""
    on, off = engines
    sbox = S.rijndael_sbox()
    for i, (n, fixed) in enumerate([(30, [(1, 1)]), (12, []), (58, [(0, 0), (7, 1)]), (20, [(5, 0)]),
                                    (60, [(3, 1), (6, 0)])]):
        tabs, tgt, mask = S.synthetic_state(n, seed=9960 + i), S.sbox_target(sbox, i), S.mux_mask(fixed)
        inb = [b for b, _ in fixed]
        on.load(tabs, tgt, mask, inb)
        off.load(tabs, tgt, mask, inb)
        assert np.array_equal(on.filter7_part(0, 1), off.filter7_part(0, 1)), n


def _run(env_extra):
    code = (
        "import sys, hashlib, json, numpy as np; sys.path[:0]=[%r, %r]\n"
        "import _support as S, sboxgates_b200 as sb\n"
        "eng = sb.LutEngine(0); sbox = S.rijndael_sbox(); out = []\n"
        "for n, fixed in [(34, [(0,1)]), (44, [(2,1),(3,0)]), (48, [(0,1),(5,0),(3,1)]), (60, [(1,1)])]:\n"
        "    eng.load(S.synthetic_state(n, seed=n + 7), S.sbox_target(sbox, n %% 8), S.mux_mask(fixed), [b for b, _ in fixed])\n"
        "    whole = eng.filter7_part(0, 1)\n"
        "    parts = np.sort(np.concatenate([eng.filter7_part(p, 3) for p in range(3)]))[:100000]\n"
        "    r = eng.search7(bytes(range(256)), bytes(range(255, -1, -1)))\n"
        "    out.append([len(whole), hashlib.sha1(whole.tobytes()).hexdigest(), hashlib.sha1(parts.tobytes()).hexdigest(), int(r.key & 0xffffffffffff), int(r.tuples_feasible)])\n"
        "print(json.dumps(out))\n" % (S.ROOT, os.path.join(S.ROOT, "tests")))
    env = dict(os.environ)
    env.update(env_extra)
    res = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True,
                         check=True)
    return res.stdout.strip().splitlines()[-1]


def test_sieve3_segments_and_overflow_retry_reuse_the_table():
    """A 4,096-entry ticket table (several launches per sweep) and a small hit buffer (the retry)
    with the sieve forced on give the lists of one unsieved launch."""
    ref = _run({"SBG_SIEVE": "0"})
    assert _run({"SBG_SIEVE": "2", "SBG_TICKET_TABLE": "4096"}) == ref
    assert _run({"SBG_SIEVE": "2", "SBG_HITS_CAP": "200000"}) == ref
    rows = json.loads(ref)
    assert all(r[1] == r[2] for r in rows) and any(r[0] == 100000 for r in rows)
    assert any(0 < r[0] < 100000 for r in rows)
