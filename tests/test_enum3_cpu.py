"""The 3-LUT enumeration without a GPU: the oracle's orc_enum3_range against orc_scan3_key and a
plain numpy count over all position triples, and the Python decoding of 3-LUT records
(decode_key3, match_to_lut3; match_to_ret refuses them)."""
import itertools

import numpy as np
import pytest

import _enum3_support as E3
import _enum_support as E
import _support as S
import sboxgates_b200 as sb

NONE = E.NONE


def _mask(rs, positions):
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, positions, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
    return mask


def _states():
    """n = 8-20 under random masks of 0-200 positions and mux masks; planted 3-LUT, 5-input and
    S-box targets."""
    sbox = S.rijndael_sbox()
    rs = np.random.RandomState(3303)
    out = []
    for i, positions in enumerate([0, 1, 3, 7, 12, 33, 65, 100, 200, 256, 128, 64, 32]):
        n = int(rs.choice([8, 11, 14, 17, 20]))
        tabs = S.synthetic_state(n, seed=3400 + i)
        mask = _mask(rs, positions) if positions not in (256, 128, 64, 32) else \
            S.mux_mask([(b, 1) for b in range({256: 0, 128: 1, 64: 2, 32: 3}[positions])])
        if i % 3 == 0:
            g = [int(x) for x in rs.choice(n, 3, replace=False)]
            tgt = S.lut_table(int(rs.randint(1, 255)), tabs[g[0]], tabs[g[1]], tabs[g[2]])
        elif i % 3 == 1:
            g = [int(x) for x in rs.choice(n, 5, replace=False)]
            tgt = S.lut_table(int(rs.randint(1, 255)), S.lut_table(int(rs.randint(1, 255)),
                              tabs[g[0]], tabs[g[1]], tabs[g[2]]), tabs[g[3]], tabs[g[4]])
        else:
            tgt = S.sbox_target(sbox, i % 8)
        order = [int(x) for x in rs.permutation(n)]
        out.append((tabs, tgt, mask, order))
    return out


def _bits(words):
    """(4,) uint64 -> (256,) 0/1, position p = bit p & 63 of word p >> 6."""
    w = np.asarray(words, dtype=np.uint64)
    return ((w[:, None] >> np.arange(64, dtype=np.uint64)[None, :]) & np.uint64(1)).reshape(256)


def _numpy_keys(tabs, tgt, mask, order):
    """Keys of every position triple whose cells hold no masked 1 next to a masked 0: a plain
    numpy restatement of check_n_lut_possible(3, ...) (lut.c:34-66)."""
    n = len(tabs)
    pos = np.nonzero(_bits(mask))[0]
    t = _bits(tgt)[pos].astype(bool)
    g = np.stack([_bits(tabs[order[p]])[pos] for p in range(n)]).astype(np.int64)   # by position
    trips = np.array(list(itertools.combinations(range(n), 3)), dtype=np.int64).reshape(-1, 3)
    cell = 4 * g[trips[:, 0]] + 2 * g[trips[:, 1]] + g[trips[:, 2]]     # (triples, positions)
    onehot = np.left_shift(1, cell)
    ones = np.bitwise_or.reduce(np.where(t[None, :], onehot, 0), axis=1)    # 0 without positions
    zeros = np.bitwise_or.reduce(np.where(~t[None, :], onehot, 0), axis=1)
    ok = (ones & zeros) == 0
    return [int(a) << 18 | int(b) << 9 | int(c) for (a, b, c), y in zip(trips, ok) if y]


def _cuts(total, rs):
    return [1, total, max(1, int(rs.randint(1, max(2, total // 3))))]


def test_enum3_range_first_key_is_scan3_key():
    rs = np.random.RandomState(5)
    hits = 0
    for i, (tabs, tgt, mask, order) in enumerate(_states()):
        n = len(tabs)
        for size in _cuts(n * (n - 1) * (n - 2) // 6, rs):
            want = E.scan3_key(tabs, tgt, mask, order, piece=size)
            total, keys = E3.enum3_range(tabs, tgt, mask, order, 3, piece=size)
            assert (keys[0] if keys else NONE) == want, (i, size)
            assert len(keys) == min(total, 3) and keys == sorted(set(keys)), (i, size)
        hits += total > 0
    assert hits >= 8


def test_enum3_range_totals_are_a_plain_count():
    rs = np.random.RandomState(6)
    zero_mask = 0
    for i, (tabs, tgt, mask, order) in enumerate(_states()):
        n = len(tabs)
        want = _numpy_keys(tabs, tgt, mask, order)
        all_triples = n * (n - 1) * (n - 2) // 6
        for size in _cuts(all_triples, rs):
            total, keys = E3.enum3_range(tabs, tgt, mask, order, len(want) + 1, piece=size)
            assert total == len(want) and keys == want, (i, size, total, len(want))
        # a slice of ranks holds the matches whose triples have those ranks
        lo, hi = sorted(int(x) for x in rs.randint(0, all_triples + 1, 2))
        ranks = {k: E.comb_rank(n, 3, [k >> 18, (k >> 9) & 0x1FF, k & 0x1FF]) for k in want}
        sub = [k for k in want if lo <= ranks[k] < hi]
        assert E3.enum3_range(tabs, tgt, mask, order, len(sub) + 1, lo, hi) == (len(sub), sub), i
        if not int(np.bitwise_or.reduce(mask)):
            assert len(want) == all_triples   # no masked position: every triple realises the target
            zero_mask += 1
    assert zero_mask == 1


def _match(width, key, gates, fo, fm, fi, seen):
    m = np.zeros(1, dtype=sb.MATCH_DTYPE)[0]
    m["key"], m["func_outer"], m["func_middle"] = key, fo, fm
    m["func_inner"], m["inner_seen"], m["width"] = fi, seen, width
    m["gates"][:len(gates)] = gates
    return m


def test_decode_key3():
    assert sb.decode_key3((499 << 18) | (300 << 9) | 257) == (499, 300, 257)
    assert sb.decode_key3((0 << 18) | (1 << 9) | 2) == (0, 1, 2)


def test_match_to_lut3_fills_like_lut_search():
    """The add_lut call of a 3-LUT match: the solved bits, plus one draw for the don't-care cells
    iff a cell is unseen -- what lut_search does with sbg_node_result::func3 / seen3."""
    seed = bytes(range(128))
    for seen in (0xFF, 0x5A, 0x00):
        fi = 0x96 & seen
        a, b = sb.Xorshift1024(seed), sb.Xorshift1024(seed)
        want = fi
        if seen != 0xFF:
            want |= (~seen & 0xFF) & (a.next() & 0xFF)
        got = sb.match_to_lut3(_match(3, (2 << 18) | (5 << 9) | 9, [11, 4, 7], 0, 0, fi, seen), b)
        assert got == (want, 11, 4, 7)
        assert a.draws == b.draws == (0 if seen == 0xFF else 1)
    with pytest.raises(ValueError):
        sb.match_to_lut3(_match(5, 0, [3, 9, 4, 1, 7], 0x96, 0, 0x12, 0xFF), sb.Xorshift1024(seed))


def test_match_to_ret_rejects_width3():
    rng = sb.Xorshift1024(bytes(range(128)))
    with pytest.raises(ValueError):
        sb.match_to_ret(_match(3, 0, [0, 1, 2], 0, 0, 0x80, 0xFF), rng)
    assert rng.draws == 0
