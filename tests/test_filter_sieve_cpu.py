"""CPU: the pair-separation sieve of phase 1 (k_filter7_pm, shifted windows), restated in Python.

A 7-tuple is feasible iff no masked target-1 position and target-0 position agree on all seven gates.
Per 4-gate prefix the kernel takes up to 64 (target 1, target 0) pairs inside the prefix's mixed
cells -- each position paired with the first position of the other target in its cell -- and a
lane with pair (e,f) intersects its candidate last gates g with the gates separating each chosen
pair that e and f leave unseparated.  That may only remove infeasible g, and it removes all of them
when the chosen pairs are all the prefix's within-cell pairs (every mixed cell has a single
position of one target, at most 64 pairs).  Checked against brute force (and the CPU oracle's
check_n_lut_possible on a sample) for 32 to 256 positions, excluded input bits and prefixes
without a mixed cell."""
import random

import numpy as np
import pytest

import _support as S

PAIRS = 64


def _positions(tables, target, mask, n):
    """Masked positions in order: (gate bits, target bit)."""
    out = []
    for p in range(256):
        if (int(mask[p >> 6]) >> (p & 63)) & 1:
            bits = 0
            for g in range(n):
                bits |= ((int(tables[g][p >> 6]) >> (p & 63)) & 1) << g
            out.append((bits, (int(target[p >> 6]) >> (p & 63)) & 1))
    return out


def _sieve_pairs(pos, pre):
    """The kernel's choice: (S list, whether the pairs are all the prefix's within-cell pairs).
    Every position of a mixed cell, in order, is paired with the first position of the other
    target in its cell -- except the cell's first target-0 position, whose pair the first target-1
    position has -- up to 64 pairs."""
    cell = []
    for bits, _ in pos:
        c = 0
        for g in pre:
            c = (c << 1) | ((bits >> g) & 1)
        cell.append(c)
    first = {}   # (cell, target) -> first position
    count = {}
    for i, (_, t) in enumerate(pos):
        first.setdefault((cell[i], t), i)
        count[(cell[i], t)] = count.get((cell[i], t), 0) + 1
    mixed = {c for c, t in first if (c, 1 - t) in first}
    S_, chosen = [], 0
    for i, (bits, t) in enumerate(pos):
        if cell[i] not in mixed or (not t and i == first[(cell[i], 0)]):
            continue
        chosen += 1
        if len(S_) < PAIRS:
            q = first[(cell[i], 1 - t)]
            S_.append(bits ^ pos[q][0])   # = ~(xr[p] ^ xr[q]): xr is complemented where the target is 0
    # these are all the within-cell pairs iff every mixed cell has a single position of one target
    every = all(min(count[(c, 0)], count[(c, 1)]) == 1 for c in mixed)
    return S_, every and chosen <= PAIRS


def _sieve(S_, e, f, cand):
    for s in S_:
        if cand == 0:
            break
        if not ((s >> e) & 1 or (s >> f) & 1):
            cand &= s
    return cand


def _feasible(pos, gates):
    ones, zeros = set(), set()
    for bits, t in pos:
        key = tuple((bits >> g) & 1 for g in gates)
        (ones if t else zeros).add(key)
    return not (ones & zeros)


def _random_mask(positions, rs):
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, positions, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def _check_state(n, tables, target, mask, inbits, prefixes, rng, oracle_sample=0):
    pos = _positions(tables, target, mask, n)
    excl = sum(1 << b for b in inbits)
    allowed = [g for g in range(n - 3) if not (excl >> g) & 1]
    exact_prefixes = 0
    checked = 0
    for pre in prefixes(allowed, rng):
        S_, exact = _sieve_pairs(pos, pre)
        last = pre[-1]
        for e in range(last + 1, n - 2):
            for f in range(e + 1, n - 1):
                if (excl >> e) & 1 or (excl >> f) & 1:
                    continue
                cand = ((1 << n) - 1) & ~((1 << (f + 1)) - 1) & ~excl
                got = _sieve(S_, e, f, cand)
                want = 0
                for g in range(f + 1, n):
                    if (cand >> g) & 1 and _feasible(pos, list(pre) + [e, f, g]):
                        want |= 1 << g
                assert got & want == want, (pre, e, f, bin(got), bin(want))
                if exact:
                    assert got == want, (pre, e, f, bin(got), bin(want))
                if checked < oracle_sample:   # the brute force is check_n_lut_possible(7)
                    g = rng.choice(range(f + 1, n))
                    assert _feasible(pos, list(pre) + [e, f, g]) == S.oracle_check(
                        7, target, mask, [tables[x] for x in list(pre) + [e, f, g]])
                    checked += 1
        exact_prefixes += exact
    return exact_prefixes


def _random_prefixes(count):
    def gen(allowed, rng):
        for _ in range(count):
            yield sorted(rng.sample(allowed, 4))
    return gen


@pytest.mark.parametrize("positions,n,inbits", [(256, 16, []), (200, 18, [2]), (128, 16, [0, 5]),
                                                (64, 20, [1]), (33, 18, []), (32, 22, [3, 6])])
def test_sieve_never_removes_a_feasible_gate(positions, n, inbits):
    rs = np.random.RandomState(positions * 131 + n)
    tables = S.synthetic_state(n, seed=9100 + positions)
    target = S.sbox_target(S.rijndael_sbox(), positions % 8)
    mask = _random_mask(positions, rs)
    _check_state(n, tables, target, mask, inbits, _random_prefixes(6), random.Random(positions),
                 oracle_sample=20)


def test_sieve_is_exact_when_all_pairs_fit():
    """A mux mask of depth 4 leaves 16 positions, about one per cell: in many prefixes every mixed
    cell has a single position of one target, and the sieve alone is exact."""
    n = 20
    tables = S.synthetic_state(n, seed=9201)
    target = S.sbox_target(S.rijndael_sbox(), 3)
    mask = S.mux_mask([(1, 0), (4, 1), (6, 1), (7, 0)])
    exact = _check_state(n, tables, target, mask, [1, 4, 6, 7], _random_prefixes(12), random.Random(7))
    assert exact >= 3


def test_sieve_passes_prefixes_without_mixed_cells():
    """16 positions over which input bits 0-3 vary: prefix (0,1,2,3) splits them into one position
    per cell, so no cell is mixed and the sieve keeps every candidate."""
    n = 14
    tables = S.synthetic_state(n, seed=9301)
    target = S.sbox_target(S.rijndael_sbox(), 0)
    mask = S.mux_mask([(4, 0), (5, 1), (6, 0), (7, 1)])
    pos = _positions(tables, target, mask, n)
    S_, exact = _sieve_pairs(pos, (0, 1, 2, 3))
    assert S_ == [] and exact
    cand = ((1 << n) - 1) & ~((1 << 6) - 1)
    assert _sieve(S_, 4, 5, cand) == cand
    _check_state(n, tables, target, mask, [], lambda allowed, rng: [(0, 1, 2, 3)], random.Random(1))
