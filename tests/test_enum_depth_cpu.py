"""CPU: the host side of the depth filter -- graph.gate_depths against the golden graphs' XML,
match_depth on hand-worked records, shallowest_matches over a stand-in engine, the argument checks
that need no device, and the header's constants and declarations.  Also the host reference the GPU
tests filter with (tests/_enum_support.py): record_depths against match_depth, the pruning shortcuts
against the minimum over every ordering row, and the brute-force feasible count against the CPU
oracle."""
import ctypes as C
import glob
import os
import re
import xml.etree.ElementTree as ET

import numpy as np
import pytest

import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import graph, native

GRAPHS = sorted(glob.glob(os.path.join(S.GOLDEN, "graphs", "*.xml")))


def _xml_depths(path):
    """Depths straight from the XML, by memoised recursion over the <input gate=...> references."""
    gates = [el for el in ET.parse(path).getroot() if el.tag == "gate"]
    memo = {}

    def depth(i):
        if i not in memo:
            ins = [int(x.get("gate")) for x in gates[i] if x.tag == "input"]
            memo[i] = 0 if gates[i].get("type") == "IN" else 1 + max(depth(j) for j in ins)
        return memo[i]
    return [depth(i) for i in range(len(gates))]


def test_golden_graphs_exist():
    assert len(GRAPHS) >= 3


@pytest.mark.parametrize("path", GRAPHS, ids=os.path.basename)
def test_gate_depths_match_the_xml(path):
    d = graph.gate_depths(graph.load_graph(path))
    assert d.dtype == np.uint16
    assert [int(x) for x in d] == _xml_depths(path)
    assert int(d.max()) >= 2


def _rec(width, gates):
    r = np.zeros(1, dtype=sb.MATCH_DTYPE)[0]
    r["width"] = width
    r["gates"][:width] = gates
    return r


def test_match_depth_by_hand():
    depth = [0, 1, 2, 3, 4, 5, 6, 7, 0, 0]
    # width 3: 1 + max(D)
    assert sb.match_depth(_rec(3, [0, 8, 9]), depth) == 1
    assert sb.match_depth(_rec(3, [2, 7, 1]), depth) == 8
    # width 5: 1 + max(1 + max(a, b, c), d, e)
    assert sb.match_depth(_rec(5, [0, 1, 2, 8, 9]), depth) == 4      # outer 1 + 2, inner 3 + 1
    assert sb.match_depth(_rec(5, [0, 8, 9, 7, 1]), depth) == 8      # the deep gate feeds the inner
    assert sb.match_depth(_rec(5, [7, 8, 9, 0, 1]), depth) == 9      # ... or the outer LUT
    # width 7: 1 + max(1 + max(a, b, c), 1 + max(d, e, f), g)
    assert sb.match_depth(_rec(7, [0, 8, 9, 1, 2, 3, 4]), depth) == 5
    assert sb.match_depth(_rec(7, [0, 8, 9, 1, 2, 3, 7]), depth) == 8
    assert sb.match_depth(_rec(7, [0, 8, 9, 7, 2, 3, 1]), depth) == 9
    with pytest.raises(ValueError):
        sb.match_depth(_rec(0, []), depth)


class _StandIn:
    """An engine over a fixed list of records (in key order) that filters them as the library
    does: the matches of depth <= max_depth, and their histogram."""

    def __init__(self, recs):
        self.recs = recs
        self.filter = None
        self.calls = []

    def set_depth_filter(self, depth, max_depth):
        self.filter = (np.asarray(depth), int(max_depth))

    def _run(self, k):
        depth, bound = self.filter
        d = np.array([sb.match_depth(r, depth) for r in self.recs], dtype=np.int64)
        keep = self.recs[d <= bound]
        self.hist = np.bincount(d[d <= bound]).astype(np.uint64) if keep.size else \
            np.zeros(0, dtype=np.uint64)
        self.calls.append(bound)
        return sb.Enumeration(len(keep), 0, keep[:k])

    def enumerate5(self, order, k, count=True):
        return self._run(k)

    def depth_counts(self):
        nz = np.flatnonzero(self.hist)
        return self.hist[:nz[-1] + 1] if nz.size else self.hist[:0]


def test_shallowest_matches_over_a_stand_in():
    recs = np.zeros(5, dtype=sb.MATCH_DTYPE)
    gates = [[0, 1, 2, 3, 4], [0, 1, 2, 3, 5], [1, 2, 3, 4, 5], [0, 1, 5, 3, 4], [2, 3, 4, 0, 1]]
    for i, g in enumerate(gates):
        recs[i]["key"] = i
        recs[i]["width"] = 5
        recs[i]["gates"][:5] = g
    depth = [0, 0, 0, 0, 0, 4]
    eng = _StandIn(recs)
    dmin, count, got = sb.shallowest_matches(eng, 5, (bytes(range(256)),), depth, 10)
    assert (dmin, count) == (2, 2) and list(got["key"]) == [0, 4]
    assert eng.calls == [sb.SBG_DEPTH_BINS - 1, 2]
    dmin, count, got = sb.shallowest_matches(eng, 5, (bytes(range(256)),), depth, 1)
    assert (dmin, count, list(got["key"])) == (2, 2, [0])
    eng = _StandIn(recs[:0])
    assert sb.shallowest_matches(eng, 5, (bytes(range(256)),), depth, 10)[:2] == (None, 0)
    with pytest.raises(ValueError):
        sb.shallowest_matches(eng, 4, (), depth, 10)


def test_depth_filter_argument_checks():
    eng = sb.LutEngine.__new__(sb.LutEngine)   # no device: the checks run before the library
    for bad in ([], [[1, 2]], [0.5, 1.0], [0, -1], [0, native.SBG_MAX_DEPTH + 1],
                np.zeros(native.SBG_MAX_GATES + 1, dtype=np.uint16)):
        with pytest.raises(ValueError):
            eng.set_depth_filter(bad, 3)
    for bound in (-1, 2**32):
        with pytest.raises(ValueError):
            eng.set_depth_filter([0, 1, 2], bound)


def test_header_declares_the_depth_filter():
    with open(os.path.join(S.ROOT, "include", "sboxgates_b200.h")) as f:
        header = f.read()
    consts = dict(re.findall(r"#define (SBG_MAX_DEPTH|SBG_DEPTH_BINS) (\d+)", header))
    assert int(consts["SBG_MAX_DEPTH"]) == native.SBG_MAX_DEPTH == sb.SBG_MAX_DEPTH == 1020
    assert int(consts["SBG_DEPTH_BINS"]) == native.SBG_DEPTH_BINS == sb.SBG_DEPTH_BINS == 1024
    # the deepest match (a 7-LUT over gates of the largest depth) still has a bin
    assert native.SBG_MAX_DEPTH + 2 < native.SBG_DEPTH_BINS
    assert "int sbg_enum_set_depth(sbg_handle *h, const uint16_t *depth, int n, uint32_t " \
        "max_depth);" in header
    assert "int sbg_enum_depth_counts(sbg_handle *h, uint64_t *out, uint32_t nbins);" in header
    assert native.SIGNATURES["sbg_enum_set_depth"] == (
        C.c_int, [C.c_void_p, C.POINTER(C.c_uint16), C.c_int, C.c_uint32])
    assert native.SIGNATURES["sbg_enum_depth_counts"] == (C.c_int, [C.c_void_p, native.u64p,
                                                                    C.c_uint32])
    # the new entry points appear in the cursor-lifetime list
    lifetime = header[header.index("Cursor lifetime:"):header.index("Without a cursor")]
    assert "sbg_enum_depth_counts" in lifetime and "sbg_enum_set_depth" in lifetime


def _records(width, gates):
    recs = np.zeros(len(gates), dtype=sb.MATCH_DTYPE)
    recs["width"] = width
    recs["gates"][:, :width] = gates
    return recs


@pytest.mark.parametrize("width", [3, 5, 7])
def test_record_depths_equal_match_depth(width):
    rs = np.random.RandomState(width)
    depth = rs.randint(0, native.SBG_MAX_DEPTH + 1, 40)
    depth[:8] = rs.choice([0, 1, native.SBG_MAX_DEPTH], 8)
    recs = _records(width, np.array([rs.choice(40, width, replace=False) for _ in range(500)]))
    got = E.record_depths(recs, depth)
    assert [int(x) for x in got] == [sb.match_depth(r, depth) for r in recs]
    assert E.record_depths(recs[:0], depth).shape == (0,)


@pytest.mark.parametrize("width", [3, 5, 7])
def test_bound_shortcuts_equal_every_ordering(width):
    """The kernels prune a gate set unless no gate has depth >= B and at most two (width 5) or one
    (width 7) have depth B - 1; that must be exactly 'some ordering row has depth <= B', the
    minimum of match_depth over the 10 rows of order5_rows / 70 rows of order7_rows."""
    rows = {3: [[0, 1, 2]], 5: S.order5_rows(), 7: S.order7_rows()}[width]
    assert len(rows) == {3: 1, 5: 10, 7: 70}[width]
    recs = _records(width, np.array(rows))
    rs = np.random.RandomState(50 + width)
    seen = set()
    for i in range(3000):
        hi = 4 if i % 2 else 1022
        d = rs.randint(0, hi + 1, width)
        if i % 3 == 0:   # gates concentrated on the edges of a bound
            b = int(rs.randint(2, 1023))
            d = rs.choice([b - 2, b - 1, b], width)
        best = int(E.record_depths(recs, d).min())
        if width > 3:   # the closed form the pruning rests on
            s = sorted(d, reverse=True)
            assert best == max(2 + int(s[{5: 2, 7: 1}[width]]), 1 + int(s[0]))
        for bound in {0, best - 2, best - 1, best, best + 1, int(rs.randint(0, 1024))}:
            if bound < 0:
                continue
            ok = bool(E.bound_admits(d, bound, width))
            assert ok == (best <= bound), (d, bound, best)
            seen.add((ok, int(np.sum(d == bound - 1))))
    # both sides of the count rule occur: the largest count kept and the smallest dropped
    keep_max = {3: 3, 5: 2, 7: 1}[width]
    assert (True, keep_max) in seen
    if width > 3:
        assert (False, keep_max + 1) in seen


def _feasible_state(n, seed):
    """A seeded state whose target is a planted 5-LUT circuit, under a mux mask of depth 1 - 3."""
    tabs = S.synthetic_state(n, seed=seed)
    rs = np.random.RandomState(seed)
    fixed = [(int(b), int(rs.randint(0, 2))) for b in rs.choice(8, 1 + seed % 3, replace=False)]
    inb = [b for b, _ in fixed]
    g = [int(x) for x in rs.choice([x for x in range(n) if x not in inb], 5, replace=False)]
    tgt = S.lut_table(int(rs.randint(1, 255)), S.lut_table(int(rs.randint(1, 255)), tabs[g[0]],
                      tabs[g[1]], tabs[g[2]]), tabs[g[3]], tabs[g[4]])
    return tabs, tgt, S.mux_mask(fixed), inb


@pytest.mark.parametrize("n,seed", [(12, 3), (16, 4), (18, 5), (20, 6)])
def test_feasible5_brute_force_equals_oracle(n, seed):
    """With the loosest bound the brute force counts what search_5lut's enumeration reports as
    feasible (the CPU oracle); tighter bounds only ever drop combinations."""
    tabs, tgt, mask, inb = _feasible_state(n, seed)
    order = E.orders(seed)[0]
    _, _, feasible = E.oracle_enum5(tabs, tgt, mask, inb, order, 0)
    depth = np.random.RandomState(seed).randint(0, native.SBG_MAX_DEPTH + 1, n)
    assert E.feasible5_under_bound(tabs, tgt, mask, inb, depth, sb.SBG_DEPTH_BINS - 1) == feasible
    assert feasible > 0
    small = np.random.RandomState(seed).randint(0, 4, n)
    got = [E.feasible5_under_bound(tabs, tgt, mask, inb, small, b) for b in range(7)]
    assert got[0] == got[1] == 0 and got[-1] == feasible
    assert got == sorted(got)
