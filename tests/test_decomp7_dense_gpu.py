"""GPU: search_7lut's phase 2 (k_decomp7) against the CPU oracle on dense lists -- states of 40
and 64 gates under masks of 32 and 64 positions, where most list entries pass stage 1 and the stage-2
work per entry is largest.  Windows of the phase-1 list with and without a match, lists of
stale-cache tuples (gate 0 allowed), with the stage-1 filter on and off (SBG_DECOMP_FILTER)."""
import numpy as np
import pytest

import _support as S
import sboxgates_b200 as sb
from sboxgates_b200.lut import pack_tuple7, unpack_tuple7
from sboxgates_b200.rng import Xorshift1024

pytestmark = pytest.mark.gpu

NONE = 2**64 - 1
CASES = [(40, [(0, 1), (3, 0), (5, 1)]), (40, [(1, 0), (6, 1)]),
         (64, [(2, 1), (4, 0), (7, 1)]), (64, [(0, 0), (5, 1)])]
WINDOW = 24


def _stale_list(rs, n):
    """Pairs (0, g1-4, .., g1-1, g1, g2) < (0, g1, g2, ...): every second entry reuses the outer
    tables of the one before it for its rows 0-3 (the reference's truncated cache key)."""
    out = []
    for g1 in range(5, n - 6, 5):
        g2 = g1 + 1
        rest = sorted(int(x) for x in rs.choice(np.arange(g2 + 1, n), 4, replace=False))
        out.append(pack_tuple7([0, g1 - 4, g1 - 3, g1 - 2, g1 - 1, g1, g2]))
        out.append(pack_tuple7([0, g1, g2] + rest))
    return np.array(sorted(out), dtype=np.uint64)


def _cases(rs):
    """(tables, target, mask, lists); half the targets are planted 7-LUT circuits (dense lists with
    many matches), half S-box bits (hardly any)."""
    sbox = S.rijndael_sbox()
    eng = sb.LutEngine(0)
    try:
        for i, (n, fixed) in enumerate(CASES):
            tabs = S.synthetic_state(n, seed=4000 + n + len(fixed))
            if i % 2 == 0:
                g = [int(x) for x in rs.choice(n, 7, replace=False)]
                t_outer = S.lut_table(0x96, tabs[g[0]], tabs[g[1]], tabs[g[2]])
                t_mid = S.lut_table(0xE8, tabs[g[3]], tabs[g[4]], tabs[g[5]])
                tgt = S.lut_table(0xCA, t_outer, t_mid, tabs[g[6]])
            else:
                tgt = S.sbox_target(sbox, (n + len(fixed)) % 8)
            mask = S.mux_mask(fixed)
            eng.load(tabs, tgt, mask, [])
            lst = eng.filter7_part(0, 1)
            assert len(lst) >= 4 * WINDOW, (n, fixed, len(lst))
            starts = [0] + sorted(int(a) for a in rs.choice(len(lst) - WINDOW, 2, replace=False))
            yield tabs, tgt, mask, [lst[a:a + WINDOW] for a in starts] + [_stale_list(rs, n)]
    finally:
        eng.close()


def test_decomp7_keys_match_the_oracle_on_dense_lists(monkeypatch):
    rs = np.random.RandomState(2026)
    runs = []
    for tabs, tgt, mask, lists in _cases(rs):
        for w in lists:
            outer, middle = sb.shuffled_orders7(Xorshift1024(rs.bytes(128)))
            tuples = np.array([unpack_tuple7(p) for p in w], dtype=np.uint16)
            want = S.oracle_decomp7_key(tabs, tgt, mask, tuples, outer, middle)
            runs.append((tabs, tgt, mask, w, outer, middle, want))
    with_match = sum(r[-1] != NONE for r in runs)
    assert 0 < with_match < len(runs), (with_match, len(runs))
    for decomp_filter in ("1", "0"):
        monkeypatch.setenv("SBG_DECOMP_FILTER", decomp_filter)
        eng = sb.LutEngine(0)
        try:
            for i, (tabs, tgt, mask, w, outer, middle, want) in enumerate(runs):
                eng.load(tabs, tgt, mask, [])
                eng.set_list7(w)
                got = eng.decomp7_part(0, 1, outer, middle)
                assert got == want, (i, decomp_filter, hex(got), hex(want))
        finally:
            eng.close()
