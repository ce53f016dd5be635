"""Cost of enumeration next to the first-match searches, on bench.py's synthetic states.

For each state (n = 40: masks of mux depth 0..3, i.e. the full mask and 128 / 64 / 32 positions;
n = 64 likewise; a seeded shuffled gate order per state) it times with CUDA events, median of
--reps runs after one warm-up:
  scan3               lut_search's 3-LUT scan alone (search_node with SBG_DO_SCAN3 only)
  count3  / first3    its full enumeration (count only) and count-free with max_matches = 1
  search5 / search7   the first-match searches (search7 includes phase 1)
  count5  / count7    full enumeration, count only (max_matches = 0); count7 on the list search7
                      left installed, i.e. phase 2 only
  first5  / first7    count-free enumeration with max_matches = 1 (a first-match search)
and prints one line per state plus the totals.

A second table times the cursor calls after a count, per width: the count itself (max_matches =
0), a 4,096-match page at the middle rank (sbg_enum_fetch), the page that ends at the last rank,
and a pick of 4,096 uniform ranks (sbg_enum_pick).  States: bench.py's n = 40 state under 32
positions, and states under the empty mask, where every candidate matches (3-LUT at n = 500, 5-LUT
at n = 40 and 64, 7-LUT at n = 40: totals of 2.1e7 to 4.6e11).

    python scripts/enum_time.py [--n 40 64] [--reps 3] [--no-main] [--no-fetch]
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


def timed(fn, reps):
    """Median CUDA-event time (ms) of fn() on the current stream, and fn()'s last result."""
    fn()
    times, out = [], None
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[40, 64])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--no-main", action="store_true", help="skip the first table")
    ap.add_argument("--no-fetch", action="store_true", help="skip the fetch / pick table")
    args = ap.parse_args()
    eng = sb.LutEngine(0, stream=torch.cuda.current_stream().cuda_stream)
    print("%s, %d SMs, power limit %s W" % (
        torch.cuda.get_device_name(0), torch.cuda.get_device_properties(0).multi_processor_count,
        bench.power_limit_w(0)))
    if not args.no_main:
        print("%4s %5s %4s | %8s %7s %7s %7s | %10s %9s %9s %9s | %11s %7s %9s %9s %9s" % (
            "n", "mask", "inb", "matches3", "scan3", "count3", "first3", "matches5", "search5",
            "count5", "first5", "matches7", "list", "search7", "count7", "first7"))
    for n in ([] if args.no_main else args.n):
        for j, st in enumerate(bench.build_batch(n, 4, args.seed)):
            eng.load(st["tables"], st["target"], st["mask"], st["inbits"])
            gate_order = np.random.RandomState(1000 * args.seed + j).permutation(n)
            ms_s3, r3 = timed(lambda: eng.search_node(0, gate_order=gate_order), args.reps)
            ms_c3, e3 = timed(lambda: eng.enumerate3(gate_order, 0), args.reps)
            ms_f3, f3 = timed(lambda: eng.enumerate3(gate_order, 1, count=False), args.reps)
            assert (list(f3.matches["key"]) or [sb.lut.SBG_KEY_NONE])[0] == r3.key3
            ms_s5, r5 = timed(lambda: eng.search5(st["order5"]), args.reps)
            ms_c5, e5 = timed(lambda: eng.enumerate5(st["order5"], 0), args.reps)
            ms_f5, f5 = timed(lambda: eng.enumerate5(st["order5"], 1, count=False), args.reps)
            assert (list(f5.matches["key"]) or [sb.lut.SBG_KEY_NONE])[0] == r5.key
            ms_s7, r7 = timed(lambda: eng.search7(st["outer"], st["middle"]), args.reps)
            ms_c7, e7 = timed(lambda: eng.enumerate7(st["outer"], st["middle"], 0), args.reps)
            ms_f7, f7 = timed(lambda: eng.enumerate7(st["outer"], st["middle"], 1, count=False),
                              args.reps)
            positions = sum(bin(int(w)).count("1") for w in st["mask"])
            print("%4d %5d %4s | %8d %7.3f %7.3f %7.3f | %10d %9.3f %9.3f %9.3f | %11d %7d %9.3f "
                  "%9.3f %9.3f" % (
                      n, positions, ",".join(map(str, st["inbits"])) or "-", e3.total, ms_s3,
                      ms_c3, ms_f3, e5.total, ms_s5, ms_c5, ms_f5, e7.total, e7.feasible, ms_s7,
                      ms_c7, ms_f7), flush=True)
    if not args.no_fetch:
        fetch_table(eng, args.reps, args.seed)
    eng.close()


def fetch_table(eng, reps, seed):
    """Count, then a middle page, the last page and a uniform pick on the count's cursor."""
    print("%-22s %5s | %15s %9s | %9s %9s %9s" % ("state", "width", "total", "count", "page_mid",
                                                  "page_last", "pick4096"))
    st = bench.build_batch(40, 4, seed)[3]
    go40 = np.random.RandomState(1000 * seed + 3).permutation(40)
    rs = np.random.RandomState(seed)
    empty = np.zeros(4, dtype=np.uint64)
    cases = [("n=40 mask 32 (bench)", st["tables"], st["target"], st["mask"], st["inbits"],
              [(3, go40), (5, st["order5"]), (7, (st["outer"], st["middle"]))])]
    for n, widths in ((500, (3,)), (40, (5, 7)), (64, (5,))):
        tables = bench._state(n, 1000 + n)
        orders = {3: rs.permutation(n), 5: st["order5"], 7: (st["outer"], st["middle"])}
        cases.append(("n=%d empty mask" % n, tables, st["target"], empty, [],
                      [(w, orders[w]) for w in widths]))
    for label, tables, target, mask, inbits, runs in cases:
        eng.load(tables, target, mask, inbits)
        for width, order in runs:
            if width == 3:
                count = lambda: eng.enumerate3(order, 0)   # noqa: E731
            elif width == 5:
                count = lambda: eng.enumerate5(order, 0)   # noqa: E731
            else:
                count = lambda: eng.enumerate7(order[0], order[1], 0)   # noqa: E731
            ms_c, e = timed(count, reps)
            total = e.total
            ranks = np.random.default_rng(seed).choice(total, min(4096, total), replace=False)
            ms_mid, _ = timed(lambda: eng.fetch_matches(total // 2, 4096), reps)
            ms_last, _ = timed(lambda: eng.fetch_matches(max(0, total - 4096), 4096), reps)
            ms_pick, _ = timed(lambda: eng.pick_matches(ranks), reps)
            print("%-22s %5d | %15d %9.3f | %9.3f %9.3f %9.3f" % (
                label, width, total, ms_c, ms_mid, ms_last, ms_pick), flush=True)


if __name__ == "__main__":
    main()
