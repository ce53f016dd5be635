"""CPU model of phase 1's pair-separation sieve (k_filter7_pm, shifted windows) on bench.py's states.

For sampled 4-gate prefixes of the 8 states of a bench step (n gates, step seed 1003 by default) it
counts, per chunk of 32 (e,f) pairs:
  * positions: what the exact cell loop visits without the sieve -- whole mixed cells in cell order,
    until no lane of the chunk has a candidate last gate left;
  * sieve: the slowest lane's sieve iterations (pairs intersected into its candidate set);
  * exact: chunks where some lane still has a candidate after the sieve (they run the cell loop);
and, per prefix, whether the sieve's pairs are all its within-cell (target 1, target 0) pairs (then
the sieve alone is exact).  The -DSBG_COUNT_FILTER build of the library prints the measured
counterparts (F1 line: positions / chunks, sieve / chunks, exact) for whole sweeps.

    python scripts/sieve_model.py [n] [prefixes per state] [step seed]

Counts only: no timing, no GPU.
"""
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

PAIRS = 64


def rows_of(tables, target, mask, n):
    """Compressed positions in order: (row, target bit); row = gate bits, complemented where the
    target is 0 (the device's xr without its target bit)."""
    out = []
    for p in range(256):
        if not (int(mask[p >> 6]) >> (p & 63)) & 1:
            continue
        t = (int(target[p >> 6]) >> (p & 63)) & 1
        row = 0
        for g in range(n):
            row |= ((int(tables[g][p >> 6]) >> (p & 63)) & 1) << g
        out.append((row if t else row ^ ((1 << n) - 1), t))
    return out


def mixed_cells(pos, pre, n):
    """Mixed cells of prefix `pre` in cell order (first gate most significant): lists of positions."""
    full = (1 << n) - 1
    cells = {}
    for i, (row, t) in enumerate(pos):
        vals = row if t else row ^ full
        c = 0
        for g in pre:
            c = (c << 1) | ((vals >> g) & 1)
        cells.setdefault(c, []).append(i)
    return [cells[c] for c in sorted(cells) if len({pos[i][1] for i in cells[c]}) == 2]


def sieve_tables(pos, cells, n):
    """The kernel's pair choice: every position of a mixed cell, in order, with the first position
    of the other target in its cell (the cell's first target-0 position left out: the first
    target-1 position has that pair), up to 64 pairs.  Returns (S list, exact): S[u] = gates that
    separate pair u; exact = the pairs are all the within-cell pairs."""
    full = (1 << n) - 1
    first, cell_of = {}, {}
    for k, cell in enumerate(cells):
        for i in cell:
            cell_of[i] = k
            first.setdefault((k, pos[i][1]), i)
    S, chosen = [], 0
    for i in sorted(cell_of):
        k, t = cell_of[i], pos[i][1]
        if not t and i == first[(k, 0)]:
            continue
        chosen += 1
        if len(S) < PAIRS:
            S.append(~(pos[i][0] ^ pos[first[(k, 1 - t)]][0]) & full)
    single = all(min(sum(pos[i][1] for i in c), sum(1 - pos[i][1] for i in c)) == 1 for c in cells)
    return S, single and chosen <= PAIRS


def sieve(S, e, f, cand):
    """(surviving candidates, iterations) of one lane."""
    its = 0
    for s in S:
        if cand == 0:
            break
        if (s >> e) & 1 or (s >> f) & 1:
            continue
        cand &= s
        its += 1
    return cand, its


def exact_after_cells(pos, cells, e, f, cand, n):
    """The exact loop's candidate set after each mixed cell, in order."""
    full = (1 << n) - 1
    out = []
    for cell in cells:
        for ve in (0, 1):
            for vf in (0, 1):
                part = [i for i in cell
                        if (((pos[i][0] if pos[i][1] else pos[i][0] ^ full) >> e) & 1) == ve
                        and (((pos[i][0] if pos[i][1] else pos[i][0] ^ full) >> f) & 1) == vf]
                if len({pos[i][1] for i in part}) < 2:
                    continue
                a_and, a_or = full, 0
                for i in part:
                    a_and &= pos[i][0]
                    a_or |= pos[i][0]
                cand &= a_and | (~a_or & full)
        out.append(cand)
    return out


def model_state(st, n, samples, rs):
    pos = rows_of(st["tables"], st["target"], st["mask"], n)
    excl = 0
    for b in st["inbits"]:
        excl |= 1 << b
    acc = dict(chunks=0, positions=0, sieve=0, exact=0, lanes=0, lanes_left=0, prefixes=0, fit=0)
    allowed = [g for g in range(n - 3) if not (excl >> g) & 1]
    for _ in range(samples):
        pre = sorted(rs.sample(allowed, 4))
        last = pre[-1]
        pairs = [(e, f) for e in range(last + 1, n - 1) for f in range(e + 1, n - 1)]
        if not pairs:
            continue
        cells = mixed_cells(pos, pre, n)
        S, fit = sieve_tables(pos, cells, n)
        acc["prefixes"] += 1
        acc["fit"] += fit
        for q0 in range(0, len(pairs), 32):
            lanes = []
            for e, f in pairs[q0:q0 + 32]:
                if (excl >> e) & 1 or (excl >> f) & 1:
                    continue
                cand = ((1 << n) - 1) & ~((1 << (f + 1)) - 1) & ~excl
                lanes.append((e, f, cand))
            if not lanes:
                continue
            acc["chunks"] += 1
            worst, left = 0, 0
            seqs = []
            for e, f, cand in lanes:
                c2, its = sieve(S, e, f, cand)
                seq = exact_after_cells(pos, cells, e, f, cand, n)
                final = seq[-1] if seq else cand
                assert c2 & final == final, "the sieve removed a feasible g"
                if fit:
                    assert c2 == final, "the sieve is exact when its pairs are all the within-cell pairs"
                worst = max(worst, its)
                left += c2 != 0
                seqs.append(seq)
            acc["sieve"] += worst
            acc["exact"] += left != 0
            acc["lanes"] += len(lanes)
            acc["lanes_left"] += left
            for k, cell in enumerate(cells):   # whole cells until no lane has a candidate left
                acc["positions"] += len(cell)
                if all(s[k] == 0 for s in seqs):
                    break
    return acc


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 40
    samples = int(sys.argv[2]) if len(sys.argv) > 2 else 150
    seed = int(sys.argv[3]) if len(sys.argv) > 3 else 1003
    rs = random.Random(seed)
    by_m = {}
    for st in bench.build_batch(n, 8, seed):
        m = sum(bin(int(w)).count("1") for w in st["mask"])
        a = model_state(st, n, samples, rs)
        tot = by_m.setdefault(m, dict.fromkeys(a, 0))
        for k, v in a.items():
            tot[k] += v
    print("n = %d, step seed %d, %d sampled prefixes per state" % (n, seed, samples))
    print("%9s %18s %20s %20s %16s %14s" % ("positions", "cell loop pos/chunk", "sieve its/chunk",
                                           "lanes left (%)", "exact chunks (%)", "exact alone (%)"))
    for m in sorted(by_m, reverse=True):
        t = by_m[m]
        c = max(t["chunks"], 1)
        print("%9d %18.1f %20.1f %20.3f %16.2f %14.0f" % (
            m, t["positions"] / c, t["sieve"] / c, 100.0 * t["lanes_left"] / max(t["lanes"], 1),
            100.0 * t["exact"] / c, 100.0 * t["fit"] / max(t["prefixes"], 1)))


if __name__ == "__main__":
    main()
