"""GPU: phase 1 of search_7lut with the pair-separation sieve (forced on for every mask size with
SBG_SIEVE=2; by default it runs above 32 masked positions) gives the same lists as without it
(SBG_SIEVE=0) and as the CPU oracle.  The sieve only rules out last gates
before the exact cell loop of the shifted-window filter, so nothing about the list may change: not
its entries, not their order, not the cap.  Cases: the window cases of test_filter_windows_gpu
(n = 12 ... 63, mux masks of depth 0-3, random masks, excluded input bits incl. gate 0, the sparse
state whose list is capped), states that take the chunked head (n >= 48, at most 64 positions),
a single chain (weighted tickets), sharded parts and batched searches."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import _support as S
import test_filter_windows_gpu as W

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    """(sieve, no sieve, no sieve with shifted windows above n = 60, sieve with them)."""
    import sboxgates_b200 as sb
    out = []
    old = {k: os.environ.get(k) for k in ("SBG_SIEVE", "SBG_SHIFT")}
    try:
        for sieve, shift in (("2", None), ("0", None), ("0", "1"), ("2", "1")):
            os.environ["SBG_SIEVE"] = sieve
            if shift is None:
                os.environ.pop("SBG_SHIFT", None)
            else:
                os.environ["SBG_SHIFT"] = shift
            out.append(sb.LutEngine(0))
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    yield out
    for e in out:
        e.close()


def _head_states():
    """n >= 48 under 64 and 32 positions: the sweep starts with (prefix, chunk) tickets."""
    sbox = S.rijndael_sbox()
    return [(48, S.synthetic_state(48, seed=8401), S.sbox_target(sbox, 1),
             S.mux_mask([(0, 1), (5, 0)]), [0, 5], 3000),
            (56, S.synthetic_state(56, seed=8402), S.sbox_target(sbox, 6),
             S.mux_mask([(2, 0), (3, 1), (7, 0)]), [2, 3, 7], 3000),
            (60, S.synthetic_state(60, seed=8403), S.sbox_target(sbox, 4),
             S.mux_mask([(1, 1), (6, 1)]), [], 1000)]


def test_sieve_lists_match_unsieved_and_oracle(engines):
    on, off, off_sh, on_sh = engines
    states = W._states() + _head_states()
    with ThreadPoolExecutor(max_workers=max(1, min(8, os.cpu_count() or 1))) as pool:
        wants = list(pool.map(lambda s: S.oracle_filter7(s[1], s[2], s[3], s[4],
                                                         cap=s[5] or W.CAP)[0], states))
    capped = 0
    for (n, tabs, tgt, mask, inb, cmp), want in zip(states, wants):
        pairs = [(on, off)] + ([(on_sh, off_sh)] if n > 60 else [])
        for a, b in pairs:
            a.load(tabs, tgt, mask, inb)
            b.load(tabs, tgt, mask, inb)
            got, ref = a.filter7_part(0, 1), b.filter7_part(0, 1)
            assert np.array_equal(got, ref), (n, inb, len(got), len(ref))
            if cmp is None:
                assert len(got) == len(want), (n, inb, len(got), len(want))
            else:
                assert len(want) == cmp and len(got) >= cmp, (n, inb, len(got))
                got = got[:cmp]
            assert np.array_equal(got, W._pack(want)), (n, inb)
            capped += len(got) == W.CAP
    assert capped >= 1


@pytest.mark.parametrize("n,fixed,inb", [(40, [], [3]), (40, [(1, 0), (6, 1)], [1, 6]),
                                         (33, [(0, 0), (2, 1), (4, 0)], [0, 2, 4])])
def test_sieve_sharded_parts_match(engines, n, fixed, inb):
    on, off = engines[0], engines[1]
    tabs = S.synthetic_state(n, seed=8500 + n + len(fixed))
    tgt = S.sbox_target(S.rijndael_sbox(), len(fixed))
    mask = S.mux_mask(fixed)
    for e in (on, off):
        e.load(tabs, tgt, mask, inb)
    for part in range(3):
        got, ref = on.filter7_part(part, 3), off.filter7_part(part, 3)
        assert np.array_equal(got, ref), (n, part, len(got), len(ref))


def test_sieve_batch_equals_unsieved_single_calls(engines):
    """Batched searches (chains sharing the device) with the sieve == one at a time without it."""
    on, off = engines[0], engines[1]
    sbox = S.rijndael_sbox()
    rs = np.random.RandomState(8600)
    jobs, states = [], []
    for slot in range(8):
        n = int(rs.choice([24, 33, 40, 47]))
        tabs = S.synthetic_state(n, seed=8600 + slot)
        fixed = [(int(b), int(rs.randint(0, 2))) for b in rs.choice(8, slot % 4, replace=False)]
        mask, inb = S.mux_mask(fixed), [b for b, _ in fixed]
        tgt = S.sbox_target(sbox, slot % 8)
        on.stage(slot, tabs, tgt, mask, inb)
        off.stage(slot, tabs, tgt, mask, inb)
        jobs.append(dict(slot=slot, order5=bytes(rs.permutation(256).astype(np.uint8)),
                         outer=bytes(rs.permutation(256).astype(np.uint8)),
                         middle=bytes(rs.permutation(256).astype(np.uint8))))
    res = on.search_batch(jobs)
    for j, r in zip(jobs, res):
        off.use(j["slot"])
        r5 = off.search5(j["order5"])
        assert (r.r5.found, r.r5.key, r.r5.tuples_feasible) == (r5.found, r5.key, r5.tuples_feasible)
        if not r5.found:
            r7 = off.search7(j["outer"], j["middle"])
            assert (r.r7.found, r.r7.key, r.r7.tuples_feasible, list(r.r7.gates), r.r7.func_inner) \
                == (r7.found, r7.key, r7.tuples_feasible, list(r7.gates), r7.func_inner)
            if r7.tuples_feasible < W.CAP:   # a capped sweep stops where the schedule left it
                assert r.r7.tuples_swept == r7.tuples_swept
