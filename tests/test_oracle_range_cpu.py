"""The rank-range forms of the CPU oracle (tests/enum_oracle.c) against its whole-space forms: over a
partition of the ranks, orc_filter7_range, orc_search5_range, orc_enum5_range and orc_scan3_key must
give what orc_filter_7lut, orc_search5_key, orc_enum5 and a plain loop over the position triples
give.  The large-state GPU checks (test_oracle_large_gpu.py) rest on this."""
import numpy as np

import _enum_support as E
import _support as S

NONE = E.NONE


def _mask(rs, positions):
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, positions, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def _states():
    """n = 9-14 under random masks (1-200 positions) and mux masks, S-box and planted targets."""
    sbox = S.rijndael_sbox()
    rs = np.random.RandomState(4242)
    out = []
    for i, positions in enumerate([1, 3, 7, 12, 33, 65, 100, 200, 256, 128, 64, 32]):
        n = int(rs.choice([9, 10, 12, 14]))
        tabs = S.synthetic_state(n, seed=4300 + i)
        mask = _mask(rs, positions) if positions not in (256, 128, 64, 32) else \
            S.mux_mask([(b, 1) for b in range({256: 0, 128: 1, 64: 2, 32: 3}[positions])])
        if i % 3 == 0:
            g = [int(x) for x in rs.choice(n, 5, replace=False)]
            tgt = S.lut_table(int(rs.randint(1, 255)), S.lut_table(int(rs.randint(1, 255)),
                              tabs[g[0]], tabs[g[1]], tabs[g[2]]), tabs[g[3]], tabs[g[4]])
        elif i % 3 == 1:
            g = [int(x) for x in rs.choice(n, 3, replace=False)]
            tgt = S.lut_table(int(rs.randint(1, 255)), tabs[g[0]], tabs[g[1]], tabs[g[2]])
        else:
            tgt = S.sbox_target(sbox, i % 8)
        inb = [0] if i % 2 else [int(rs.randint(1, 8)), 0] if i % 4 == 0 else []
        out.append((tabs, tgt, mask, inb))
    return out


def _cuts(total, rs):
    """A random partition of [0, total) given as its piece size; 1 and total are included."""
    return [1, total, max(1, int(rs.randint(1, max(2, total // 3))))]


def test_filter7_range_is_the_phase1_list():
    rs = np.random.RandomState(1)
    nonempty = 0
    for i, (tabs, tgt, mask, inb) in enumerate(_states()):
        n = tabs.shape[0]
        want, _ = S.oracle_filter7(tabs, tgt, mask, inb)
        total = S.oracle_lib().orc_n_choose_k(n, 7)
        for size in _cuts(total, rs):
            got = E.filter7_range(tabs, tgt, mask, inb, 0, total, piece=size)
            assert np.array_equal(got, want), (i, size)
        bad, first = E.check7_list(tabs, tgt, mask, want)
        assert bad == 0 and first == -1, i
        nonempty += len(want) > 0
        # the slice of the list between two ranks
        lo, hi = sorted(int(x) for x in rs.randint(0, total + 1, 2))
        ranks = np.array([E.comb_rank(n, 7, t) for t in want], dtype=np.int64)
        got = E.filter7_range(tabs, tgt, mask, inb, lo, hi)
        assert np.array_equal(got, want[(ranks >= lo) & (ranks < hi)]), (i, lo, hi)
    assert nonempty >= 6


def test_check7_list_finds_infeasible_entries():
    tabs, tgt, mask, inb = _states()[4]
    lst, _ = S.oracle_filter7(tabs, tgt, mask, inb)
    every = np.array([E.nth_comb(tabs.shape[0], 7, r) for r in range(120)], dtype=np.uint16)
    want = [i for i, t in enumerate(every) if not S.oracle_check(7, tgt, mask, [tabs[g] for g in t])]
    assert len(want) > 0
    assert E.check7_list(tabs, tgt, mask, every) == (len(want), want[0])


def test_search5_and_enum5_ranges_are_the_whole_space_oracle():
    rs = np.random.RandomState(2)
    found = 0
    for i, (tabs, tgt, mask, inb) in enumerate(_states()):
        order = E.orders(i)[0]
        total = S.oracle_lib().orc_n_choose_k(tabs.shape[0], 5)
        want_key = S.oracle_search5_key(tabs, tgt, mask, inb, order)
        want = E.oracle_enum5(tabs, tgt, mask, inb, order, 50)
        for size in _cuts(total, rs):
            assert E.search5_range(tabs, tgt, mask, inb, order, 0, total, size) == want_key, (i, size)
            assert E.enum5_range(tabs, tgt, mask, inb, order, 50, piece=size) == want, (i, size)
        assert (want[1][0] if want[1] else NONE) == want_key
        found += want_key != NONE
    assert found >= 4


def test_scan3_key_is_the_first_triple_of_the_gate_order():
    """The loop of lut.c:501-523 (test_gpu_node._reference_node) restated in Python."""
    rs = np.random.RandomState(3)
    hits = 0
    for i, (tabs, tgt, mask, _) in enumerate(_states()):
        n = tabs.shape[0]
        order = [int(x) for x in rs.permutation(n)]
        want = NONE
        for a in range(n):
            for b in range(a + 1, n):
                for c in range(b + 1, n):
                    if want == NONE and S.oracle_check(3, tgt, mask, [tabs[order[a]], tabs[order[b]],
                                                                      tabs[order[c]]]):
                        want = a << 18 | b << 9 | c
        for size in _cuts(n * (n - 1) * (n - 2) // 6, rs):
            assert E.scan3_key(tabs, tgt, mask, order, piece=size) == want, (i, size)
        hits += want != NONE
    assert hits >= 4
