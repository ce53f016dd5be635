"""GPU: search_7lut's phase-1 list against the CPU oracle at the sizes where the shifted-window
filter (n <= 60) starts each chunk's windows at the lowest candidate gate of its lanes.  Depending on
how many candidate gates a window spans, a position's four parts share one register (quad windows,
at most 7 gates), two registers (packed, at most 15) or take one register each (up to 31 gates);
n = 12 ... 63 and mux masks of depth 0-3, with and without excluded input bits, meet all three, as
well as windows that start below gate 8, where the excluded bits are cut out."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import _support as S

pytestmark = pytest.mark.gpu

CAP = 100000

# (n, mux-fixed (bit, value) pairs or the size of a random mask, excluded input bits, oracle entries
# compared or None = all).  The oracle walks the combinations one by one, so the largest states are
# compared on the first entries of their lists; the last case is a sparse mask whose list reaches
# the 100,000 cap.  Random masks of 33, 65, 129 and 200 positions leave their last 32-bit word
# partly padding.
CASES = [
    (12, [], [], None),
    (12, [(1, 1)], [1], None),
    (12, [(0, 0), (4, 1)], [], None),
    (12, [(2, 1), (5, 0), (7, 1)], [2, 5, 7], None),
    (20, [], [3], None),
    (20, [(6, 0)], [], None),
    (20, [(0, 1), (3, 0)], [0, 3], None),
    (20, [(1, 0), (2, 1), (4, 0)], [], None),
    (31, [], [0, 6], None),
    (31, [(3, 1)], [3], None),
    (31, [(1, 1), (2, 0), (6, 1)], [], None),
    (32, [], [], None),
    (32, [(4, 0), (7, 1)], [4, 7], None),
    (32, [(0, 1), (5, 1), (6, 0)], [0, 5, 6], None),
    (40, [], [1], None),
    (40, [(5, 1)], [], None),
    (40, [(1, 0), (6, 1)], [1, 6], None),
    (40, [(0, 0), (3, 1), (7, 0)], [0, 3, 7], None),
    (47, [(2, 1), (4, 0), (5, 1)], [2, 4, 5], None),
    (47, [(1, 1), (7, 0)], [], 300),
    (63, [(0, 1), (3, 0), (5, 1)], [0, 3, 5], None),
    (63, [(4, 0), (6, 1), (7, 1)], [], None),
    (31, 33, [0], None),
    (31, 65, [], None),
    (32, 129, [0, 4], None),
    (40, 200, [], None),
    (47, 33, [], 2000),
]


def _pack(lst):
    """(count, 7) gate numbers -> the library's packed 63-bit form (9 bits per gate)."""
    out = np.zeros(len(lst), dtype=np.uint64)
    for i in range(7):
        out |= lst[:, i].astype(np.uint64) << np.uint64(9 * (6 - i))
    return out


def _random_mask(positions, seed):
    rs = np.random.RandomState(seed)
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, positions, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def _sparse_cap_case():
    """n = 63 under 12 random positions: most combinations are feasible, the list is capped."""
    return (63, S.synthetic_state(63, seed=6300), S.sbox_target(S.rijndael_sbox(), 5),
            _random_mask(12, 63), [2])


def _states():
    sbox = S.rijndael_sbox()
    out = []
    for i, (n, fixed, inb, cmp) in enumerate(CASES):
        mask = _random_mask(fixed, 8200 + i) if isinstance(fixed, int) else S.mux_mask(fixed)
        out.append((n, S.synthetic_state(n, seed=8100 + i), S.sbox_target(sbox, i % 8), mask, inb,
                    cmp))
    n, tabs, tgt, mask, inb = _sparse_cap_case()
    out.append((n, tabs, tgt, mask, inb, None))
    return out


def test_filter7_windows_match_oracle(engine, monkeypatch):
    """Above n = 60 the library uses aligned two-word windows; SBG_SHIFT=1 keeps the shifted ones,
    whose chunks then need a second window where they start at or below gate n - 32."""
    import sboxgates_b200 as sb
    states = _states()
    # the oracle's calls release the interpreter lock: the slow states run side by side
    with ThreadPoolExecutor(max_workers=max(1, min(8, os.cpu_count() or 1))) as pool:
        wants = list(pool.map(lambda s: S.oracle_filter7(s[1], s[2], s[3], s[4],
                                                         cap=s[5] or CAP)[0], states))
    monkeypatch.setenv("SBG_SHIFT", "1")
    shifted = sb.LutEngine(0)
    capped = 0
    try:
        for (n, tabs, tgt, mask, inb, cmp), want in zip(states, wants):
            for eng in (engine, shifted) if n > 60 else (engine,):
                eng.load(tabs, tgt, mask, inb)
                got = eng.filter7_part(0, 1)
                if cmp is None:
                    assert len(got) == len(want), (n, inb, len(got), len(want))
                else:
                    assert len(want) == cmp and len(got) >= cmp, (n, inb, len(got))
                    got = got[:cmp]
                assert np.array_equal(got, _pack(want)), (n, inb, eng is shifted)
                capped += len(got) == CAP
    finally:
        shifted.close()
    assert capped >= 1
