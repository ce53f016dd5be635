"""Cost of global ranks across shares (sbg_enum_block_sums / sbg_enum_set_global), on one GPU.

P LutEngine handles on the same device stand in for the P shares of a sharded enumeration: handle q
counts part q of P.  The script times, per share, with CUDA events (median of --reps runs after one
warm-up):
  count        the share's count (max_matches = 0)
  globalize    its sbg_enum_block_sums plus sbg_enum_set_global (the rows gathered on the host)
  page_mid     a global 4,096-match page at rank total / 2 (sbg_enum_fetch on the global cursor)
  page_last    the global page that ends at the last rank
  pick4096     a global pick of 4,096 uniform ranks (sbg_enum_pick on the global cursor)
and prints the slowest share's time of each, next to one whole-share handle (part 0 of 1) doing the
same count, fetches and pick.  States, as in DESIGN.md section 9: bench.py's n = 40 state under 32
positions, and states under the empty mask (3-LUT at n = 500, 5-LUT at n = 40 and 64, 7-LUT at
n = 40).

The shares run one after another on one GPU, so the slowest share is what one of P GPUs would
spend, apart from the collectives; what P GPUs gain over one is not measured here.

    python scripts/enum_global_time.py [--parts 4] [--reps 3]
"""
import argparse
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import sboxgates_b200 as sb  # noqa: E402


def event_ms(fn):
    """CUDA-event time (ms) of fn() on the current stream, and fn()'s result."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def count_call(eng, width, order, part, nparts):
    if width == 3:
        return eng.enumerate3(order, 0, True, part, nparts)
    if width == 5:
        return eng.enumerate5(order, 0, True, part, nparts)
    return eng.enumerate7(order[0], order[1], 0, True, part, nparts)


def one_rep(whole, shares, width, order, seed):
    """One timed run of every step; returns (whole's times, per-share times, total)."""
    P = len(shares)
    ms_c, e = event_ms(lambda: count_call(whole, width, order, 0, 1))
    total = e.total
    ranks = np.random.default_rng(seed).choice(total, min(4096, total), replace=False)
    mid, last = total // 2, max(0, total - 4096)
    w = [ms_c, event_ms(lambda: whole.fetch_matches(mid, 4096))[0],
         event_ms(lambda: whole.fetch_matches(last, 4096))[0],
         event_ms(lambda: whole.pick_matches(ranks))[0]]
    counts, glob = [], [0.0] * P
    for q, eng in enumerate(shares):
        counts.append(event_ms(lambda: count_call(eng, width, order, q, P))[0])
    nb = [eng.enum_block_count() for eng in shares]
    sums = np.zeros((P, max(max(nb), 1)), dtype=np.uint64)
    for q, eng in enumerate(shares):
        glob[q], row = event_ms(eng.enum_block_sums)
        sums[q, :nb[q]] = row
    for q, eng in enumerate(shares):
        ms, t = event_ms(lambda: eng.enum_set_global(sums, nb))
        assert t == total, (t, total)
        glob[q] += ms
    per = [counts, glob]
    for fn in (lambda e: e.fetch_matches(mid, 4096), lambda e: e.fetch_matches(last, 4096),
               lambda e: e.pick_matches(ranks)):
        per.append([event_ms(lambda: fn(eng))[0] for eng in shares])
    return w, per, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    stream = torch.cuda.current_stream().cuda_stream
    whole = sb.LutEngine(0, stream=stream)
    shares = [sb.LutEngine(0, stream=stream) for _ in range(args.parts)]
    print("%s, %d SMs, power limit %s W; %d shares on one GPU" % (
        torch.cuda.get_device_name(0), torch.cuda.get_device_properties(0).multi_processor_count,
        bench.power_limit_w(0), args.parts))
    st = bench.build_batch(40, 4, args.seed)[3]
    go40 = np.random.RandomState(1000 * args.seed + 3).permutation(40)
    rs = np.random.RandomState(args.seed)
    empty = np.zeros(4, dtype=np.uint64)
    cases = [("n=40 mask 32 (bench)", st["tables"], st["target"], st["mask"], st["inbits"],
              [(3, go40), (5, st["order5"]), (7, (st["outer"], st["middle"]))])]
    for n, widths in ((500, (3,)), (40, (5, 7)), (64, (5,))):
        tables = bench._state(n, 1000 + n)
        orders = {3: rs.permutation(n), 5: st["order5"], 7: (st["outer"], st["middle"])}
        cases.append(("n=%d empty mask" % n, tables, st["target"], empty, [],
                      [(w, orders[w]) for w in widths]))
    cols = ("count", "page_mid", "page_last", "pick4096")
    print("%-22s %5s %15s | whole: %s | slowest share: %s" % (
        "state", "width", "total", " ".join("%9s" % c for c in cols),
        " ".join("%9s" % c for c in ("count", "globalize") + cols[1:])))
    for label, tables, target, mask, inbits, runs in cases:
        for eng in [whole] + shares:
            eng.load(tables, target, mask, inbits)
        for width, order in runs:
            reps = [one_rep(whole, shares, width, order, args.seed) for _ in range(args.reps + 1)][1:]
            total = reps[0][2]
            w = [statistics.median(r[0][i] for r in reps) for i in range(4)]
            s = [statistics.median(max(r[1][i]) for r in reps) for i in range(5)]
            print("%-22s %5d %15d |        %s |                %s" % (
                label, width, total, " ".join("%9.3f" % x for x in w),
                " ".join("%9.3f" % x for x in s)), flush=True)
    for eng in [whole] + shares:
        eng.close()


if __name__ == "__main__":
    main()
