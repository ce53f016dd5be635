"""Test-side reference of the whole-space 7-LUT enumeration (sbg_enum7_all), built from the CPU
oracle alone: the feasible 7-combinations of the whole space (orc_filter7_range over all of C(n,7),
inbits applied), their keys from orc_enum7 as if they were one uncapped list, and the list index of
each key replaced by the combination's rank among all C(n,7).  Records come from
_enum_reference.build_records over the table of every combination, so they are indexed by rank.

Deal blocks follow the whole-space tickets: a ticket is the 6-gate prefix (a..f) of the
combination, numbered in lexicographic order among the 6-subsets of 0..n-2, and kDeal consecutive
prefixes form a block.

TEST INFRASTRUCTURE -- nothing under sboxgates_b200/ imports this module.
"""
from math import comb

import numpy as np

import _enum_reference as R
import _enum_support as E

LOW23 = np.uint64((1 << 23) - 1)


def lex_ranks(combos, m):
    """Lexicographic rank of each sorted t-subset (rows of `combos`) of 0..m-1:
    C(m, t) - 1 - sum_i C(m - 1 - c_i, t - i)."""
    c = np.asarray(combos, dtype=np.int64).reshape(len(combos), -1)
    t = c.shape[1]
    table = np.array([[comb(v, r) for r in range(t + 1)] for v in range(m + 1)], dtype=np.int64)
    out = np.full(len(c), comb(m, t) - 1, dtype=np.int64)
    for i in range(t):
        out -= table[m - 1 - c[:, i], t - i]
    return out


def feasible_tuples(tables, target, mask, inbits):
    """The feasible 7-combinations of the whole space, in rank order ((count, 7) uint16)."""
    return E.filter7_range(tables, target, mask, inbits, 0, comb(len(tables), 7))


def list_to_whole(keys, tuples, n):
    """Keys over the list `tuples` (high field = list index) -> whole-space keys (high field =
    the combination's rank)."""
    keys = np.asarray(keys, dtype=np.uint64)
    if len(keys) == 0:
        return keys
    ranks = lex_ranks(tuples, n).astype(np.uint64)
    return (ranks[(keys >> np.uint64(23)).astype(np.int64)] << np.uint64(23)) | (keys & LOW23)


class WholeReference(R.Reference):
    """R.Reference of sbg_enum7_all: same fields and select(); feasible is the number of feasible
    combinations (under a depth filter: those with an ordering within the bound), and items /
    blocks / shares follow the 6-gate prefix tickets."""

    def __init__(self, tables, target, mask, inbits, orders, tuples=None, keys=None):
        n = len(tables)
        self.feasible_list = feasible_tuples(tables, target, mask, inbits) if tuples is None \
            else tuples
        if keys is None:
            _, keys, _ = R.oracle_keys(7, tables, target, mask, inbits, orders,
                                       tuples=self.feasible_list)
            assert keys is not None, "more than %d matches" % R.CAP
        self.list_keys = keys
        super().__init__(7, tables, target, mask, inbits, orders, tuples=R._combs(n, 7),
                         keys=list_to_whole(keys, self.feasible_list, n),
                         feasible=len(self.feasible_list))
        self.items = prefix_items(self.keys, n)
        self.select()

    def select(self, depth=None, bound=None, outer=None, middle=None, inner=None, grouping=None,
               functions=False):
        super().select(depth, bound, outer, middle, inner, grouping, functions)
        self.blocks = self.items[self.idx] // R.KDEAL
        return self

    def _feasible(self, depth, bound, depth_ok):
        if depth is None:
            return len(self.feasible_list)
        d = np.asarray(depth, dtype=np.int64)[self.feasible_list.astype(np.int64)]
        return int(E.bound_admits(d, bound, 7).sum())

    def nblocks(self):
        return -(-comb(self.n - 1, 6) // R.KDEAL)

    def group_sizes(self, depth=None, bound=None, outer=None, middle=None, inner=None,
                    grouping=None, functions=False):
        """The number of filtered matches in the group of each of recs (grouped settings)."""
        ok = np.ones(len(self.all), dtype=bool)
        if depth is not None:
            ok &= E.record_depths(self.all, depth) <= bound
        if functions:
            ok &= R.function_ok(self.all, outer, middle, inner)
        ids = R.group_ids(self.all["key"][ok], 7, grouping)
        uniq, counts = np.unique(ids, return_counts=True)
        return counts[np.searchsorted(uniq, R.group_ids(self.recs["key"], 7, grouping))] \
            .astype(np.uint64)


def prefix_items(keys, n):
    """The whole-space ticket (6-gate prefix number) of each whole-space key."""
    keys = np.asarray(keys, dtype=np.uint64)
    if len(keys) == 0:
        return np.zeros(0, dtype=np.int64)
    combos = R._combs(n, 7)[(keys >> np.uint64(23)).astype(np.int64)]
    return lex_ranks(combos[:, :6], n - 1)
