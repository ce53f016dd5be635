"""CPU: the two facts k_decomp7's stage 2 rests on, checked on Python mirrors of the kernel code.

1. An outer function fo and its complement admit the same middle functions: complementing fo swaps
   the merged sets r1 and r0, and middle_cubes answers (r1, r0) and (r0, r1) with the same set.  So
   stage 2 decides one member of each complementary pair of survivors, and the pair's outer position
   is the smaller of the two.
2. Deciding a tuple's (pair, row) entries 32 at a time, in a flat list over all its outer triples,
   gives the same key as deciding each triple's survivors row by row and stopping at the first row
   with a match.
"""
import numpy as np


def compress16x2(r, b, z):
    """Of both 16-bit halves of r, the 8 bits whose index has bit b equal to z, in order."""
    out = 0
    for half in (0, 16):
        i = 0
        for p in range(16):
            if ((p >> b) & 1) == z:
                out |= ((r >> (half + p)) & 1) << (half + i)
                i += 1
    return out


def index_bit_to_top(r, b):
    """Mirror of the CUDA helper: three adjacent index-bit exchanges, each only where b <= its
    lower bit."""
    for lo, d, m in ((0, 1, 0x22222222), (1, 2, 0x0C0C0C0C), (2, 4, 0x00F000F0)):
        t = ((r >> d) ^ r) & (m if b <= lo else 0)
        r = (r ^ t ^ (t << d)) & 0xFFFFFFFF
    return r


def constraints(r1, r0, b):
    """The four inner cells (x, g) of middle_cubes: (A, B) = middle patterns with a masked 1 / 0."""
    out = []
    for ci in range(4):
        ab = compress16x2(r1 if ci & 2 else r0, b, ci & 1)
        out.append((ab & 0xFF, ab >> 16))
    return out


def admitted_brute(r1, r0, b):
    """Middle functions fm that send, in every inner cell with both sets non-empty, A to one value
    and B to the other: fm & (A | B) in {A, B}."""
    cons = [(a, bb) for a, bb in constraints(r1, r0, b) if a and bb]
    return {fm for fm in range(256) if all((fm & (a | bb)) in (a, bb) for a, bb in cons)}


def admitted_cubes(r1, r0, b):
    """middle_cubes + the 16 (c0, c1) checks: the union of the cubes {fm : fm & S == V}."""
    cs, ca, cb = [], [], []
    for a, bb in constraints(r1, r0, b):
        act = a != 0 and bb != 0
        cs.append(a | bb if act else 0)
        ca.append(a if act else 0)
        cb.append(bb if act else 0)
    hs, hv, hok = [], [], []
    for h2 in range(2):
        i = 2 * h2
        hs.append(cs[i] | cs[i + 1])
        ov2 = cs[i] & cs[i + 1]
        hv.append([])
        hok.append([])
        for c in range(4):
            v0 = cb[i] if c & 1 else ca[i]
            v1 = cb[i + 1] if c & 2 else ca[i + 1]
            hok[h2].append(((v0 ^ v1) & ov2) == 0)
            hv[h2].append(v0 | v1)
    S, ov = hs[0] | hs[1], hs[0] & hs[1]
    out = set()
    for c0 in range(4):
        for c1 in range(4):
            if hok[0][c0] and hok[1][c1] and ((hv[0][c0] ^ hv[1][c1]) & ov) == 0:
                V = hv[0][c0] | hv[1][c1]
                out |= {fm for fm in range(256) if fm & S == V}
    return out


def test_index_bit_to_top_keeps_compress16x2s_order():
    rs = np.random.RandomState(1)
    for r in [0, 0xFFFFFFFF, 0x12345678] + [int(x) for x in rs.randint(0, 2**32, 300, dtype=np.uint64)]:
        for b in range(4):
            for z in range(2):
                assert compress16x2(index_bit_to_top(r, b), 3, z) == compress16x2(r, b, z), (r, b, z)


def test_complementary_outer_functions_admit_the_same_middle_functions():
    rs = np.random.RandomState(2)
    nonempty = 0
    for _ in range(400):
        # sparse sets, so that many cells carry both a 1 and a 0 and the sets are neither empty nor full
        r1 = int(rs.randint(0, 2**32, dtype=np.uint64)) & int(rs.randint(0, 2**32, dtype=np.uint64))
        r0 = int(rs.randint(0, 2**32, dtype=np.uint64)) & int(rs.randint(0, 2**32, dtype=np.uint64))
        b = int(rs.randint(0, 4))
        want = admitted_brute(r1, r0, b)
        assert admitted_cubes(r1, r0, b) == want
        assert admitted_brute(r0, r1, b) == want
        assert admitted_cubes(r0, r1, b) == want
        assert admitted_cubes(index_bit_to_top(r0, b), index_bit_to_top(r1, b), 3) == want
        nonempty += 0 < len(want) < 256
    assert nonempty > 50


NONE = 0xFFFFFFFF


def _random_tuple(rs):
    """Triples (j, first ordering k0, rows, survivors, best_pm[row][fo]) of one tuple, in order j;
    survivors closed under complement, best_pm the same for fo and ~fo (fact 1)."""
    rows_of = [4] * 15 + [1] * 10
    rs_perm = rs.permutation(25)
    k0s, k = [], 0
    for j in range(25):
        k0s.append(k)
        k += rows_of[rs_perm[j]]
    out = []
    for j in range(25):
        if rs.rand() < 0.5:
            continue
        nrows = rows_of[rs_perm[j]]
        npairs = int(rs.choice([0, 1, 2, 3, 7, 20, 64, 128]))
        reps = rs.choice(128, npairs, replace=False)
        surv = sorted(set(int(x) for x in reps) | set(255 - int(x) for x in reps))
        p_match = rs.choice([0.0, 0.002, 0.05])
        pm = [[None] * 256 for _ in range(nrows)]
        for row in range(nrows):
            for fo in range(128):
                v = int(rs.randint(0, 256)) if rs.rand() < p_match else None
                pm[row][fo] = pm[row][255 - fo] = v
        out.append((j, k0s[j], nrows, surv, pm))
    return out


def _key_row_by_row(triples, pos):
    """The former stage 2: per triple, every survivor one lane, rows one after the other; the first
    row with a match decides, then the smallest (po, pm)."""
    for j, k0, nrows, surv, pm in triples:
        if not surv:
            continue
        row_best = [NONE] * nrows
        for row in range(nrows):
            for fo in surv:
                if pm[row][fo] is not None:
                    row_best[row] = min(row_best[row], pos[fo] << 8 | pm[row][fo])
        for row in range(nrows):
            if row_best[row] != NONE:
                return (k0 + row) << 16 | row_best[row]
    return NONE


def _key_flat(triples, pos):
    """Mirror of k_decomp7's loop: one entry per (pair, row), full 32-entry passes as the list fills,
    the partial pass carried over, stop after the first pass with a match (plus the entries left)."""
    pmin = [min(pos[fo], pos[255 - fo]) for fo in range(128)]
    ent, best, passes = [], NONE, 0

    def run(chunk):
        nonlocal passes
        passes += 1
        cands = [(k << 16 | pmin[fo] << 8 | pm[row][fo]) for k, row, fo, pm in chunk
                 if pm[row][fo] is not None]
        return min(cands, default=NONE)

    for j, k0, nrows, surv, pm in triples:
        reps = [fo for fo in surv if fo < 128]
        if not reps:
            continue
        for fo in reps:
            for row in range(nrows):
                ent.append((k0 + row, row, fo, pm))
        if len(ent) < 32:
            continue
        full = len(ent) & ~31
        for p0 in range(0, full, 32):
            best = min(best, run(ent[p0:p0 + 32]))
        if best != NONE:
            ent = ent[full:]
            break
        ent = ent[full:]
    if ent:
        best = min(best, run(ent))
    return best, passes


def test_flat_entry_list_gives_the_row_by_row_key():
    rs = np.random.RandomState(3)
    hits = 0
    for _ in range(600):
        triples = _random_tuple(rs)
        pos = [int(x) for x in rs.permutation(256)]
        want = _key_row_by_row(triples, pos)
        got, _ = _key_flat(triples, pos)
        assert got == want
        hits += want != NONE
    assert 100 < hits < 590
