"""Test-side closed forms of enumerated records for states in which every candidate matches: masks
of 0 or 1 positions.  check_n_lut_possible cannot fail there (no cell can hold a masked 1 next to a
masked 0), so the match at any rank follows from the rank alone:
  3-LUT: the rank-th position triple i < k < m of the gate order (lexicographic);
  5-LUT: rank = c * 2560 + k * 256 + pos, c = the c-th 5-combination of the gates inbits allows;
  7-LUT: rank = ((idx * 70 + k) * 256 + po) * 256 + pm over the list of the first `cap`
         7-combinations (all of them feasible).
func_inner / inner_seen: 0 / 0 without a masked position; with one masked position p, the cell c
the LUT inputs select at p is seen, and is a 1 iff the target is 1 at p.

TEST INFRASTRUCTURE -- nothing under sboxgates_b200/ imports this module.
"""
from math import comb

import numpy as np

W5 = 10 * 256            # matches per allowed 5-combination
W7 = 70 * 256 * 256      # matches per 7-LUT list entry


def unrank(elems, t, r):
    """The r-th t-subset (lexicographic) of the ascending list elems.  The subsets whose first
    element has index x0 .. X number comb(n - x0, left) - comb(n - X - 1, left), so each element
    is found by bisection."""
    out, x0, n = [], 0, len(elems)
    for left in range(t, 0, -1):
        base = comb(n - x0, left)
        lo, hi = x0, n - left
        while lo < hi:
            mid = (lo + hi) // 2
            if r < base - comb(n - mid - 1, left):
                hi = mid
            else:
                lo = mid + 1
        r -= base - comb(n - lo, left)
        out.append(elems[lo])
        x0 = lo + 1
    return out


def rank_of(n, combo):
    """Lexicographic rank of an ascending t-subset of 0..n-1."""
    r, prev, t = 0, -1, len(combo)
    for i, g in enumerate(combo):
        for x in range(prev + 1, g):
            r += comb(n - x - 1, t - i - 1)
        prev = g
    return r


def masked_position(mask):
    """The single masked position of a 1-position mask, None for the empty mask."""
    bits = [p for p in range(256) if (int(mask[p >> 6]) >> (p & 63)) & 1]
    assert len(bits) <= 1, "closed forms hold for masks of 0 or 1 positions"
    return bits[0] if bits else None


def _bit(words, p):
    return (int(words[p >> 6]) >> (p & 63)) & 1


def _inner(tabs, target, p, cell_of):
    """(func_inner, inner_seen) given a function of one gate's bit at p -> the inner cell."""
    if p is None:
        return 0, 0
    c = cell_of(lambda g: _bit(tabs[g], p))
    return (_bit(target, p) << c), 1 << c


def _lut_bit(func, a, b, c):
    return (func >> (a << 2 | b << 1 | c)) & 1


def total3(n):
    return comb(n, 3)


def total5(n, inbits):
    return comb(len([g for g in range(n) if g not in inbits]), 5) * W5


def total7(n, cap):
    return min(cap, comb(n, 7)) * W7


def record3(rank, tabs, target, mask, order):
    """(key, gates[7], func_outer, func_middle, func_inner, inner_seen, width) of the 3-LUT match at
    `rank`."""
    n = len(tabs)
    i, k, m = unrank(list(range(n)), 3, rank)
    g = [int(order[i]), int(order[k]), int(order[m])]
    fi, seen = _inner(tabs, target, masked_position(mask),
                      lambda b: b(g[0]) << 2 | b(g[1]) << 1 | b(g[2]))
    return (i << 18 | k << 9 | m, g + [0] * 4, 0, 0, fi, seen, 3)


def record5(rank, tabs, target, mask, inbits, order, rows5):
    n = len(tabs)
    allowed = [g for g in range(n) if g not in inbits]
    c, rest = divmod(rank, W5)
    k, pos = divmod(rest, 256)
    combo = unrank(allowed, 5, c)
    g = [combo[rows5[k][i]] for i in range(5)]
    fo = order[pos]
    fi, seen = _inner(tabs, target, masked_position(mask),
                      lambda b: _lut_bit(fo, b(g[0]), b(g[1]), b(g[2])) << 2 | b(g[3]) << 1
                      | b(g[4]))
    return (rank_of(n, combo) << 12 | k << 8 | pos, g + [0, 0], fo, 0, fi, seen, 5)


def record7(rank, tabs, target, mask, outer, middle, rows7, cap):
    n = len(tabs)
    idx, rest = divmod(rank, W7)
    assert idx < min(cap, comb(n, 7))
    k, rest = divmod(rest, 65536)
    po, pm = divmod(rest, 256)
    combo = unrank(list(range(n)), 7, idx)
    g = [combo[rows7[k][i]] for i in range(7)]
    fo, fm = outer[po], middle[pm]
    fi, seen = _inner(tabs, target, masked_position(mask),
                      lambda b: _lut_bit(fo, b(g[0]), b(g[1]), b(g[2])) << 2
                      | _lut_bit(fm, b(g[3]), b(g[4]), b(g[5])) << 1 | b(g[6]))
    return (idx << 23 | k << 16 | po << 8 | pm, g, fo, fm, fi, seen, 7)


def as_tuple(rec):
    """A MATCH_DTYPE record in the closed forms' shape (pad bytes must be 0)."""
    assert not any(int(x) for x in rec["pad"])
    return (int(rec["key"]), [int(x) for x in rec["gates"]], int(rec["func_outer"]),
            int(rec["func_middle"]), int(rec["func_inner"]), int(rec["inner_seen"]),
            int(rec["width"]))


def one_position_mask(p):
    mask = np.zeros(4, dtype=np.uint64)
    mask[p >> 6] = np.uint64(1) << np.uint64(p & 63)
    return mask
