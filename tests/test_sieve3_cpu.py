"""CPU: phase 1's pair sieve built once per 3-gate prefix (k_sieve3) and used by every 4-gate
prefix that starts with it (k_filter7_pm, shifted windows), restated in Python.

The entry of a 3-gate prefix (a, b, c) holds up to 64 (target 1, target 0) pairs inside the mixed
cells of (a, b, c) -- each masked position of a mixed cell, in order, paired with the first position
of the other target in its cell, the cell's first target-0 position left out -- as S[u] = the gates
separating pair u, and sep[x] = the pairs gate x separates for c < x <= n - 2, pairs past the last
one counted as separated.  A 4-gate prefix (a, b, c, d) and lane pair (e, f) intersect the candidate
last gates g with S[u] for every pair that none of d, e and f separates.  Checked: every stored pair
agrees on a, b and c and has different targets, sep is the transpose of S, and against brute force
the use never removes a feasible g -- 32 to 256 positions, excluded input bits, 3-gate prefixes
without a mixed cell, and a gate d that separates every stored pair."""
import random

import numpy as np
import pytest

import _support as S
import test_filter_sieve_cpu as F

PAIRS = 64
ALL = (1 << PAIRS) - 1


def _cells(pos, abc):
    out = []
    for bits, _ in pos:
        c = 0
        for g in abc:
            c = (c << 1) | ((bits >> g) & 1)
        out.append(c)
    return out


def _entry(pos, abc, n):
    """(pairs as (p, q) position indices, S, sep) of the 3-gate prefix abc."""
    cell = _cells(pos, abc)
    first = {}
    for i, (_, t) in enumerate(pos):
        first.setdefault((cell[i], t), i)
    mixed = {c for c, t in first if (c, 1 - t) in first}
    pairs = []
    for i, (_, t) in enumerate(pos):
        if cell[i] not in mixed or (not t and i == first[(cell[i], 0)]):
            continue
        if len(pairs) < PAIRS:
            pairs.append((i, first[(cell[i], 1 - t)]))
    S_ = [pos[p][0] ^ pos[q][0] for p, q in pairs]   # = ~(xr[p] ^ xr[q]) over the gate bits
    unused = ALL & ~((1 << len(S_)) - 1)
    sep = {x: sum(((s >> x) & 1) << u for u, s in enumerate(S_)) | unused
           for x in range(abc[2] + 1, n - 1)}
    return pairs, S_, sep


def _use(S_, sep, d, e, f, cand):
    left = ALL & ~(sep[d] | sep[e] | sep[f])
    u = 0
    while left and cand:
        if left & 1:
            cand &= S_[u]
        left >>= 1
        u += 1
    return cand


def _check_state(n, tables, target, mask, inbits, prefixes3, rng, per_prefix=3):
    pos = F._positions(tables, target, mask, n)
    excl = sum(1 << b for b in inbits)
    for abc in prefixes3:
        pairs, S_, sep = _entry(pos, abc, n)
        cell = _cells(pos, abc)
        for (p, q), s in zip(pairs, S_):
            assert cell[p] == cell[q] and pos[p][1] != pos[q][1]
            assert (s >> n) == 0 and all(((s >> g) & 1) == 0 for g in abc)
        for x, word in sep.items():
            for u in range(PAIRS):
                assert (word >> u) & 1 == (((S_[u] >> x) & 1) if u < len(S_) else 1)
        ds = [d for d in range(abc[2] + 1, n - 3) if not (excl >> d) & 1]
        for d in rng.sample(ds, min(per_prefix, len(ds))):
            pre = list(abc) + [d]
            for e in range(d + 1, n - 2):
                for f in range(e + 1, n - 1):
                    if (excl >> e) & 1 or (excl >> f) & 1:
                        continue
                    cand = ((1 << n) - 1) & ~((1 << (f + 1)) - 1) & ~excl
                    got = _use(S_, sep, d, e, f, cand)
                    want = 0
                    for g in range(f + 1, n):
                        if (cand >> g) & 1 and F._feasible(pos, pre + [e, f, g]):
                            want |= 1 << g
                    assert got & want == want, (pre, e, f, bin(got), bin(want))


def _random_prefixes3(n, inbits, count, rng):
    excl = set(inbits)
    allowed = [g for g in range(n - 4) if g not in excl]
    return [tuple(sorted(rng.sample(allowed, 3))) for _ in range(count)]


@pytest.mark.parametrize("positions,n,inbits", [(256, 16, []), (200, 18, [2]), (128, 16, [0, 5]),
                                                (64, 20, [1]), (33, 18, []), (32, 22, [3, 6])])
def test_sieve3_never_removes_a_feasible_gate(positions, n, inbits):
    rs = np.random.RandomState(positions * 137 + n)
    rng = random.Random(positions + n)
    tables = S.synthetic_state(n, seed=9400 + positions)
    target = S.sbox_target(S.rijndael_sbox(), positions % 8)
    mask = F._random_mask(positions, rs)
    _check_state(n, tables, target, mask, inbits, _random_prefixes3(n, inbits, 5, rng), rng)


def test_sieve3_keeps_64_pairs_spread_over_the_cells():
    """Under a full mask every cell of a 3-gate prefix is mixed and has far more than 64 pairs: the
    entry is full, and since positions are taken in order its pairs come from every cell."""
    n = 16
    tables = S.synthetic_state(n, seed=9501)
    target = S.sbox_target(S.rijndael_sbox(), 2)
    mask = F._random_mask(256, np.random.RandomState(1))
    pos = F._positions(tables, target, mask, n)
    pairs, S_, sep = _entry(pos, (0, 1, 2), n)
    assert len(S_) == PAIRS
    assert len({_cells(pos, (0, 1, 2))[p] for p, _ in pairs}) == 8
    _check_state(n, tables, target, mask, [], [(0, 1, 2), (3, 7, 9)], random.Random(2))


def test_sieve3_prefix_without_mixed_cells_passes_everything():
    """8 positions over which input bits 0-2 vary: (0, 1, 2) puts one position in each cell, so the
    entry has no pair and every sep word is all-ones."""
    n = 14
    tables = S.synthetic_state(n, seed=9601)
    target = S.sbox_target(S.rijndael_sbox(), 5)
    mask = S.mux_mask([(3, 0), (4, 1), (5, 0), (6, 1), (7, 0)])
    pos = F._positions(tables, target, mask, n)
    pairs, S_, sep = _entry(pos, (0, 1, 2), n)
    assert pairs == [] and all(w == ALL for w in sep.values())
    cand = ((1 << n) - 1) & ~((1 << 6) - 1)
    assert _use(S_, sep, 3, 4, 5, cand) == cand
    _check_state(n, tables, target, mask, [], [(0, 1, 2)], random.Random(3), per_prefix=8)


def test_sieve3_gate_d_separating_every_pair():
    """Gate d equal to the target separates every (target 1, target 0) pair: the 4-gate prefixes
    (a, b, c, d) keep every candidate, as they must (every tuple with d is feasible)."""
    n = 14
    d = 9
    tables = S.synthetic_state(n, seed=9701)
    target = S.sbox_target(S.rijndael_sbox(), 1)
    tables = np.array(tables, dtype=np.uint64)
    tables[d] = target
    mask = F._random_mask(128, np.random.RandomState(4))
    pos = F._positions(tables, target, mask, n)
    abc = (0, 3, 5)
    _, S_, sep = _entry(pos, abc, n)
    assert len(S_) > 0 and sep[d] == ALL
    for e in range(d + 1, n - 2):
        for f in range(e + 1, n - 1):
            cand = ((1 << n) - 1) & ~((1 << (f + 1)) - 1)
            assert _use(S_, sep, d, e, f, cand) == cand
    _check_state(n, tables, target, mask, [], [abc], random.Random(5), per_prefix=4)
